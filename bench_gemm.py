#!/usr/bin/env python
"""bench_gemm.py — where the tapgemm time of one step goes, per launch kind.

    python bench_gemm.py                      # config #2: pix2pix-turbo edge_to_image bf16, batch 8, 512x512
    python bench_gemm.py --model cyclegan     # config #3: cyclegan-turbo fp16, batch 16

Every launch of one step is timed in isolation with CUDA events (Engine.profile); the table sums the tapgemm launches by
kind (ms, TFLOP/s on the algorithmic FLOPs, launch count, share of the step's summed launch time) and lists the slowest
BN / shape groups.  The card's name, power limit and SM clocks are read in the same run and printed with the numbers.
Prints one JSON line at the end.
"""
import argparse
import json
import os
import subprocess
import sys
import warnings

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (puts the package on sys.path)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={q}",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        vals = [v.strip() for v in r.stdout.strip().split(",")]
        return dict(zip(q.split(","), vals))
    except (OSError, subprocess.SubprocessError) as ex:
        return {"name": torch.cuda.get_device_name(), "error": str(ex)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="pix2pix", choices=["pix2pix", "cyclegan"])
    ap.add_argument("--reps", type=int, default=3, help="timed repetitions of every launch (median per launch)")
    ap.add_argument("--top", type=int, default=12, help="shape groups listed")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_gemm.py needs a CUDA device")
    from _host import build_text_stack
    dt = torch.bfloat16 if args.model == "pix2pix" else torch.float16
    B = 8 if args.model == "pix2pix" else 16
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        text_stack = build_text_stack(1024)
    wl = bench.Workload(args.model, False, dt, B, 512, 0, text_stack)
    for _ in range(3):
        wl.step()
    torch.cuda.synchronize()
    before = card()
    prof = wl.eng.profile(reps=args.reps)
    after = card()

    total_ms = sum(p["ms"] for p in prof)
    kinds, shapes = {}, {}
    for p in prof:
        if not p["kind"].startswith("tapgemm"):
            continue
        k = kinds.setdefault(p["kind"], {"ms": 0.0, "flops": 0.0, "n": 0})
        k["ms"] += p["ms"]; k["flops"] += p["flops"]; k["n"] += 1
        s = shapes.setdefault((p["kind"], p.get("shape", "")), {"ms": 0.0, "flops": 0.0, "n": 0})
        s["ms"] += p["ms"]; s["flops"] += p["flops"]; s["n"] += 1
    tg_ms = sum(v["ms"] for v in kinds.values())
    tg_fl = sum(v["flops"] for v in kinds.values())

    def tfs(v):
        return v["flops"] / (v["ms"] * 1e-3) / 1e12 if v["ms"] > 0 else 0.0

    print(f"card: {before.get('name')}  power limit {before.get('power.limit')}  SM clock {before.get('clocks.sm')} -> "
          f"{after.get('clocks.sm')} (max {before.get('clocks.max.sm')})")
    print(f"{args.model} {str(dt).split('.')[-1]} batch {B}: {len(prof)} launches, {total_ms:.2f} ms summed; "
          f"tapgemm {sum(v['n'] for v in kinds.values())} launches, {tg_ms:.2f} ms ({tg_ms / total_ms:.1%}), {tfs({'ms': tg_ms, 'flops': tg_fl}):.0f} TFLOP/s")
    print(f"{'kind':<24}{'ms':>10}{'TFLOP/s':>10}{'launches':>10}{'share':>9}")
    for k, v in sorted(kinds.items(), key=lambda kv: -kv[1]["ms"]):
        print(f"{k:<24}{v['ms']:>10.3f}{tfs(v):>10.0f}{v['n']:>10}{v['ms'] / total_ms:>9.1%}")
    print(f"slowest shape groups (ms summed over launches):")
    for (k, s), v in sorted(shapes.items(), key=lambda kv: -kv[1]["ms"])[:args.top]:
        print(f"  {v['ms']:8.3f} ms {tfs(v):5.0f} TFLOP/s x{v['n']:<3} {k} {s}")
    line = {"model": args.model, "card": before, "card_after": after, "step_launch_ms": total_ms, "tapgemm_ms": tg_ms,
            "tapgemm_tflops": tfs({"ms": tg_ms, "flops": tg_fl}), "tapgemm_share": tg_ms / total_ms,
            "by_kind": {k: {"ms": round(v["ms"], 4), "tflops": round(tfs(v), 1), "launches": v["n"],
                            "share": round(v["ms"] / total_ms, 4)} for k, v in kinds.items()}}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
