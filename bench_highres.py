"""High-resolution measurements: ms per image of the pix2pix forward from 512^2 to 12 MP, the plan's footprint, and the VAE
attention (one head of 512) fused against the unfused path.

    python bench_highres.py [--reps 5] [--out DIR]

Prints one JSON document (and writes DIR/highres.json when --out is given).  Needs an H100; bf16, batch 1, random-init
SD-Turbo-shaped weights.  Each resolution gets a fresh engine, so one plan's workspace is resident at a time.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "img2img-turbo_b200"))

SIZES = [(512, 512), (720, 1280), (1080, 1920), (1440, 2560), (2160, 3840), (3024, 4032)]   # (H, W)
ATTN_N = [14400, 16384, 32400]


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as e:          # the numbers below still stand; the card line says why it is missing
        return f"nvidia-smi unavailable: {e}"


def forward_times(sd, reps):
    import i2it
    import weights as W
    dt = torch.bfloat16
    rows = []
    for H, Wd in SIZES:
        e = i2it.Engine(dt, i2it.PIX2PIX, cfg=W.SD_TURBO)
        e.load_state_dict(sd)
        e.set_adapter_scale("default", 1.0)
        e.set_adapter_scale("vae_skip", 2.0)
        e.finalize(1.0, 1.0, 1.0, -1.0)
        g = torch.Generator().manual_seed(1)
        x = (torch.rand(1, 1, H, Wd, generator=g) < 0.08).float().expand(-1, 3, -1, -1).contiguous().to(dt).cuda()
        text = torch.randn(1, 77, 1024, generator=g).to(dt).cuda()
        eps = torch.randn(1, 4, H // 8, Wd // 8, generator=g).to(dt).cuda()
        out = torch.empty_like(x)
        torch.cuda.synchronize()
        free0, _ = torch.cuda.mem_get_info()
        e.forward(x, text, eps, out=out)               # builds the plan
        e.forward(x, text, eps, out=out)               # warm-up
        torch.cuda.synchronize()
        free1, _ = torch.cuda.mem_get_info()
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            e.forward(x, text, eps, out=out)
            b.record()
            b.synchronize()
            ts.append(a.elapsed_time(b))
        plan = [o["kind"] for o in e.profile(1)]
        rows.append({"H": H, "W": Wd, "ms_per_image": sorted(ts)[len(ts) // 2], "ms_min": min(ts), "ms_max": max(ts),
                     "workspace_GiB": e.workspace_bytes(1, H, Wd) / 2**30, "memgetinfo_drop_GiB": (free0 - free1) / 2**30,
                     "vae_attention": "fused" if "flash_attn512" in plan else "unfused",
                     "finite": bool(torch.isfinite(out.float()).all())})
        print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
        e.close()
        del e
        torch.cuda.empty_cache()
    return rows


def attention_times(rounds):
    """Kernel time of one op_attention call (every kernel it launches, from torch.profiler), fused vs I2IT_NO_FLASH=1,
    alternating the two variants."""
    import i2it
    from torch.profiler import ProfilerActivity, profile
    dt = torch.bfloat16
    engines = {}
    for name, off in (("fused", False), ("unfused", True)):
        if off:
            os.environ["I2IT_NO_FLASH"] = "1"
        engines[name] = i2it.Engine(dt, use_cuda_graph=False)
        os.environ.pop("I2IT_NO_FLASH", None)
    rows = []
    for N in ATTN_N:
        g = torch.Generator(device="cuda").manual_seed(0)
        q = torch.randn(1, N, 512, device="cuda", generator=g).to(dt)
        k = torch.randn(1, N, 512, device="cuda", generator=g).to(dt)
        vt = torch.randn(1, 512, (N + 7) // 8 * 8, device="cuda", generator=g).to(dt)
        res = {"fused": [], "unfused": []}
        for name in res:
            engines[name].op_attention(q, k, vt, 1)     # warm-up
        for _ in range(rounds):
            for name in res:
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    engines[name].op_attention(q, k, vt, 1)
                    torch.cuda.synchronize()
                us = sum(ev.device_time for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA
                         and "memcpy" not in ev.name.lower() and "memset" not in ev.name.lower())
                res[name].append(us / 1e3)
        flops = 4.0 * N * N * 512
        row = {"N": N, "minimal_GFLOP": flops / 1e9}
        for name, ts in res.items():
            row[f"{name}_ms"] = ts
            row[f"{name}_TFLOPs_at_median"] = flops / (sorted(ts)[len(ts) // 2] * 1e-3) / 1e12
        rows.append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--skip-forward", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_highres.py needs a CUDA device (H100)")
    import weights as W
    t0 = time.time()
    res = {"card": card(), "dtype": "bf16", "batch": 1}
    res["attention_d512"] = attention_times(a.rounds)
    if not a.skip_forward:
        sd = W.make_state_dict("pix2pix", W.SD_TURBO, seed=0)
        res["forward"] = forward_times(sd, a.reps)
    res["card_after"] = card()
    res["wall_s"] = time.time() - t0
    js = json.dumps(res, indent=1)
    print(js)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "highres.json"), "w") as f:
            f.write(js)


if __name__ == "__main__":
    main()
