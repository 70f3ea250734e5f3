#!/usr/bin/env python
"""bench_ragged.py — a stream of uploads of mixed sizes through one ragged forward per batch, against one forward per image.

    python bench_ragged.py [--rounds 3] [--batches 6] [--batch 8] [--json OUT]

CycleGAN-Turbo fp16 at SD-Turbo width, inference_unpaired.py's resize_512x512 in and the resize back to each upload's size
out, all on the GPU.  Uploads are drawn (seeded) from the 24 frame sizes of bench_plans.py, between 640x480 and 1920x1080.

  - ragged:    CycleGAN_Turbo.forward_u8_batch on batches of `--batch` uploads (one plan per batch size, any mix of sizes);
  - per image: CycleGAN_Turbo.forward_u8(upload[None], resize=(512, 512), out_size=upload size), one plan per upload size
               under the wrappers' limit of 16 plans, so the stream keeps rebuilding evicted plans.

Each path has its own model (same seed, same weights) so neither evicts the other's plans.  The two run alternately, round
by round, on the same uploads and eps.  Reported per path: img/s between device events around a round, plan builds and
evictions in the timed rounds (i2it_memory_stats_get), and for the ragged path the device time of the resample_*_ragged
launches (i2it_profile).  The outputs of both paths are compared byte for byte.  The card's name and power limit are read in
the same run and printed with the numbers.  Prints one JSON line at the end.
"""
import argparse
import json
import os
import sys
import warnings

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
from bench_plans import card, frame_sizes  # noqa: E402  (puts the package on sys.path)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="timed rounds per path, alternating")
    ap.add_argument("--batches", type=int, default=6, help="batches per round")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5, help="profile repetitions of the ragged plan")
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_ragged.py needs a CUDA device")
    from _host import build_text_stack
    from cyclegan_turbo import CycleGAN_Turbo
    info = card()
    print("card", json.dumps(info), flush=True)
    text_stack = build_text_stack(1024)
    models = {}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for k in ("ragged", "per_image"):
            m = CycleGAN_Turbo(synthetic_caption="driving in the night", synthetic_direction="a2b", text_stack=text_stack)
            m.eval(); m.half()
            models[k] = m
    sizes = frame_sizes()
    g = torch.Generator(device="cuda").manual_seed(0)
    frames = {hw: torch.randint(0, 256, hw + (3,), device="cuda", dtype=torch.uint8, generator=g) for hw in sizes}
    pick = torch.Generator().manual_seed(1)
    stream = [[sizes[int(i)] for i in torch.randint(0, len(sizes), (args.batch,), generator=pick)] for _ in range(args.batches)]
    eps = [torch.randn(args.batch, 4, 64, 64, device="cuda", generator=g).half() for _ in stream]
    n_img = args.batch * args.batches

    def run(path):
        m = models[path]
        outs = []
        for b, e in zip(stream, eps):
            imgs = [frames[hw] for hw in b]
            if path == "ragged":
                outs += m.forward_u8_batch(imgs, eps=e)
            else:
                outs += [m.forward_u8(x[None], eps=e[i:i + 1], resize=(512, 512), out_size=hw)[0]
                         for i, (x, hw) in enumerate(zip(imgs, b))]
        return outs

    def timed(path):
        eng = models[path]._get_engine()
        s0 = eng.memory_stats()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0.record()
        run(path)
        t1.record()
        torch.cuda.synchronize()
        s1 = eng.memory_stats()
        return {"img_s": n_img / (t0.elapsed_time(t1) / 1e3), "plan_builds": s1["plan_builds"] - s0["plan_builds"],
                "plan_evictions": s1["plan_evictions"] - s0["plan_evictions"]}

    # warm-up and check: one full stream per path (plans, graphs, prompt), outputs compared byte for byte
    ref, got = run("per_image"), run("ragged")
    torch.cuda.synchronize()
    equal = all(torch.equal(a, b) for a, b in zip(ref, got)) and len(ref) == len(got) == n_img
    del ref, got
    print("byte_equal", equal, flush=True)
    rows = {"ragged": [], "per_image": []}
    for r in range(args.rounds):
        for path in (("ragged", "per_image") if r % 2 == 0 else ("per_image", "ragged")):
            row = timed(path)
            rows[path].append(row)
            print("round", r, path, json.dumps(row), flush=True)
    eng = models["ragged"]._get_engine()
    models["ragged"].forward_u8_batch([frames[hw] for hw in stream[0]], eps=eps[0])
    prof = eng.profile(reps=args.reps)
    rs_ms = sum(p["ms"] for p in prof if p["kind"] in ("resample_h_ragged", "resample_v_ragged"))
    step_ms = sum(p["ms"] for p in prof)
    best = {k: max(x["img_s"] for x in v) for k, v in rows.items()}
    res = {"model": "cyclegan-turbo fp16, SD-Turbo width, resize_512x512 in, input size out", "card": info,
           "batch": args.batch, "uploads_per_round": n_img, "byte_equal": equal, "rounds": rows, "best_img_s": best,
           "ragged_resample_ms_per_batch": rs_ms, "ragged_resample_share_of_launch_time": rs_ms / step_ms,
           "ragged_speedup": best["ragged"] / best["per_image"]}
    print(f"ragged {best['ragged']:.1f} img/s vs per image {best['per_image']:.1f} img/s ({res['ragged_speedup']:.2f}x); "
          f"resample_*_ragged {rs_ms:.3f} ms per batch of {args.batch} ({rs_ms / step_ms:.2%} of the launch time); "
          f"byte-equal {equal}", flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        json.dump(res, open(args.json, "w"), indent=1)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
