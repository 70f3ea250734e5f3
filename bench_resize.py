#!/usr/bin/env python
"""bench_resize.py — the CLIs' LANCZOS resizes on the GPU (forward_u8 with a geometry) against PIL on the host.

    python bench_resize.py                    # cyclegan-turbo fp16 (config #3 weights), 1280x720 and 1920x1080, batch 1 and 16

For each frame size and batch, resize_512x512 in and back to the frame size out (src/inference_unpaired.py:40-45,53):
  - device time of the resample launches per image (Engine.profile: CUDA events around every launch of the plan);
  - img/s of CycleGAN_Turbo.forward_u8(frames, resize=(512, 512), out_size=frame) — uint8 frames in and out of host memory;
  - img/s of the host pipeline it replaces: PIL resize -> forward_u8 -> PIL resize, with PIL on one thread and on a pool
    of os.cpu_count() threads (PIL releases the GIL while resizing).
The card's name and power limit are read in the same run and printed with the numbers.  Prints one JSON line at the end.
"""
import argparse
import json
import os
import sys
import time
import warnings
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
from bench_gemm import card  # noqa: E402  (puts the package on sys.path)


def pil_resize_batch(frames, hw, pool):
    from PIL import Image

    def one(a):
        return np.asarray(Image.fromarray(a, "RGB").resize((hw[1], hw[0]), Image.LANCZOS))
    return np.stack(list(pool.map(one, frames)) if pool else [one(a) for a in frames])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5, help="profile repetitions (device time of the resample launches)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_resize.py needs a CUDA device")
    from _host import build_text_stack
    from cyclegan_turbo import CycleGAN_Turbo
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = CycleGAN_Turbo(synthetic_caption="driving in the night", synthetic_direction="a2b",
                           text_stack=build_text_stack(1024))
    m.eval(); m.half()
    c = card()
    print(f"card: {c.get('name')}  power limit {c.get('power.limit')}  SM clock {c.get('clocks.sm')} (max {c.get('clocks.max.sm')})"
          f"  host threads {os.cpu_count()}")
    pool = ThreadPoolExecutor(os.cpu_count())
    rows = []
    for H, W in ((720, 1280), (1080, 1920)):
        for B in (1, 16):
            rng = np.random.default_rng(B)
            frames = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
            src = torch.from_numpy(frames).pin_memory()
            eps = torch.randn(B, 4, 64, 64, device="cuda", dtype=torch.float16)

            def device_step():
                return m.forward_u8(src, eps=eps, resize=(512, 512), out_size=(H, W)).cpu()

            def host_step(p):
                x = torch.from_numpy(pil_resize_batch(frames, (512, 512), p))
                y = m.forward_u8(x, eps=eps).cpu().numpy()
                return pil_resize_batch(y, (H, W), p)

            def rate(fn):
                for _ in range(args.warmup):
                    fn()
                torch.cuda.synchronize()
                t = time.perf_counter()
                for _ in range(args.steps):
                    fn()
                torch.cuda.synchronize()
                return B * args.steps / (time.perf_counter() - t)

            same = np.array_equal(device_step().numpy(), host_step(pool))
            dev = rate(device_step)
            prof = m._engine.profile(reps=args.reps)   # the plan of the last forward: the geometry one
            rs_ms = sum(p["ms"] for p in prof if p["kind"].startswith("resample"))
            rs_gb = sum(p["bytes"] for p in prof if p["kind"].startswith("resample")) / 1e9
            step_ms = sum(p["ms"] for p in prof)
            host1 = rate(lambda: host_step(None))
            hostn = rate(lambda: host_step(pool))
            r = {"frame": f"{W}x{H}", "batch": B, "bit_equal": bool(same),
                 "resample_ms_per_image": rs_ms / B, "resample_GB_per_step": rs_gb, "resample_share_of_launch_time": rs_ms / step_ms,
                 "device_img_s": dev, "host_1thread_img_s": host1, "host_pool_img_s": hostn}
            rows.append(r)
            print(f"{W}x{H} batch {B:>2}: resample {rs_ms / B * 1e3:7.1f} us/image ({rs_gb * 1e3:.1f} MB/step, "
                  f"{rs_ms / step_ms:.2%} of the step's launch time) | img/s device {dev:6.1f}  host PIL 1 thread {host1:6.1f}  "
                  f"host PIL {os.cpu_count()} threads {hostn:6.1f} | bit-equal {same}", flush=True)
    pool.shutdown()
    print(json.dumps({"model": "cyclegan fp16", "card": c, "rows": rows}), flush=True)


if __name__ == "__main__":
    main()
