#!/usr/bin/env python
"""bench_variations.py — n variations of one control image: one variations forward against the plain forward on the image
repeated n times (DESIGN.md section 8).

    python bench_variations.py [--steps 10] [--warmup 3] [--ns 1,2,4,8,16] [--json OUT]

Workload: BASELINE config #4's model (pix2pix-turbo with a TwinConv conv_in, stochastic, r = 0.4), bf16, 512x512, random-init
weights, one sketch-like control image, the prompt's K/V cached (set_text).  For each n both calls get the same eps, noise map
and prompt; the variations forward encodes the image once (batch 1) instead of n times.  Per n:

  * device-event img/s of both, timed alternately (plain, variations) for 3 rounds after warm-up, each round `--steps` steps
    with an L2 flush between steps (bench.py's timing);
  * the per-step device time of the launches of the vae_encode range (input packing through the latent sample), from
    i2it_profile (CUDA events around each launch, so no PDL overlap: a per-launch sum, not a share of the graph's time);
  * arena_bytes of each plan built alone (release_plans first, so the arena holds that one plan);
  * that the two outputs are byte-equal (an assert).

By FLOP count the variations forward does (n*3351 + 1117) / (n*4468) of the repeated batch's work (0.78 at n = 8).  That
estimate (`flop_estimate`, its inverse) is arithmetic; the encoder runs below the step's average rate, so the measured gain
can exceed it.  The card name and power limit are printed with the numbers: both are part of them.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "img2img-turbo_b200"))
sys.path.insert(0, ROOT)

GiB = float(1 << 30)


def encode_ms(profile):
    """Device ms of the vae_encode launches: everything up to and including the latent sample, the plan's first launch
    without a kind name."""
    k = [p["kind"] for p in profile].index("misc")
    return sum(p["ms"] for p in profile[: k + 1]), k + 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ns", default="1,2,4,8,16")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default="", help="also write the table here")
    args = ap.parse_args()
    from bench import Workload, synthetic_inputs, timed
    from bench_plans import card
    from _host import build_text_stack
    info = card()
    print("card", json.dumps(info), flush=True)
    S, dt, r = 512, torch.bfloat16, 0.4
    w = Workload("pix2pix", True, dt, 1, S, 0, build_text_stack(1024))      # binds the prompt: its K/V are cached
    eng = w.eng
    x1 = w.c_t[:1].contiguous()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")   # > 50 MB L2, zeroed between timed steps
    rows = []
    for n in (int(v) for v in args.ns.split(",")):
        _, _, eps, noise = synthetic_inputs(n, S, 1024, dt, "cuda", kind="sketch")
        xr = x1.expand(n, -1, -1, -1).contiguous()
        out_p = torch.empty(n, 3, S, S, device="cuda", dtype=dt)
        out_v = torch.empty_like(out_p)
        plain = lambda: eng.forward(xr, None, eps, noise_map=noise, r=r, out=out_p)
        var = lambda: eng.forward_variations(x1, None, eps, noise_map=noise, r=r, out=out_v)
        plain()
        var()
        torch.cuda.synchronize()
        assert torch.equal(out_p, out_v), f"n={n}: the variations forward differs from the repeated batch"
        ms = {"plain": [], "variations": []}
        for _ in range(args.rounds):
            for name, fn in (("plain", plain), ("variations", var)):
                ms[name].append(timed(fn, args.steps, args.warmup, 1, None, flush)[0])
        row = {"n": n, "equal": True}
        for name, fn in (("plain", plain), ("variations", var)):
            med = statistics.median(ms[name])
            row[name] = {"img_s": n / (med / 1e3), "ms_per_step": med, "rounds_ms": ms[name]}
            fn()
            enc, launches = encode_ms(eng.profile(3))
            row[name].update({"vae_encode_ms": enc, "vae_encode_launches": launches})
        row["speedup"] = row["variations"]["img_s"] / row["plain"]["img_s"]
        row["flop_estimate"] = (n * 4468) / (n * 3351 + 1117)
        rows.append(row)
        print("variations", json.dumps(row), flush=True)
    for row in rows:                       # each plan alone in the arena
        n = row["n"]
        _, _, eps, noise = synthetic_inputs(n, S, 1024, dt, "cuda", kind="sketch")
        xr = x1.expand(n, -1, -1, -1).contiguous()
        for name in ("plain", "variations"):
            eng.release_plans()
            if name == "plain":
                eng.forward(xr, None, eps, noise_map=noise, r=r)
            else:
                eng.forward_variations(x1, None, eps, noise_map=noise, r=r)
            torch.cuda.synchronize()
            row[name]["arena_gib"] = eng.memory_stats()["arena_bytes"] / GiB
        print("arena", json.dumps({"n": n, "plain_gib": row["plain"]["arena_gib"],
                                   "variations_gib": row["variations"]["arena_gib"]}), flush=True)
    eng.release_plans()
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        json.dump({"card": info, "rows": rows}, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
