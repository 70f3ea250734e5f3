#!/usr/bin/env python
"""bench_mixed.py — CycleGAN batches that mix both directions: one mixed forward per batch against two single-direction forwards.

    python bench_mixed.py [--requests 48] [--rounds 3] [--iters 10] [--json OUT]

CycleGAN-Turbo fp16 at SD-Turbo size, 512x512 NCHW inputs, one prompt.  A seeded stream of `--requests` requests, each with a
random direction, is served in batches of 2 and of 8:

  - mixed: one CycleGAN_Turbo.forward(x, direction=[...]) per batch (one plan per batch size for every mix);
  - split: each batch split into its a2b and its b2a images, one single-direction forward per non-empty part (every
           sub-batch size of both directions is warmed first, so neither arm builds a plan while it is timed).

Each arm has its own model (same seed, same weights), so neither evicts the other's plans; the arms alternate, round by
round, on the same inputs and eps.  The selection's own cost: an all-a2b batch of 8 and of 16 through the mixed plan against
the single-direction plan, alternating for `--rounds` rounds of `--iters` forwards each.  Times are device events around
each timed block.  Every output of the compared arms is checked byte for byte.  The card's name and power limit are read in
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
from bench_plans import card  # noqa: E402  (puts the package on sys.path)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=48)
    ap.add_argument("--rounds", type=int, default=3, help="timed rounds per arm, alternating")
    ap.add_argument("--iters", type=int, default=10, help="forwards per round of the selection-cost comparison")
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_mixed.py needs a CUDA device")
    from _host import build_text_stack
    from cyclegan_turbo import CycleGAN_Turbo
    info = card()
    print("card", json.dumps(info), flush=True)
    text_stack = build_text_stack(1024)
    models = {}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for k in ("mixed", "split"):
            m = CycleGAN_Turbo(synthetic_caption="driving in the night", synthetic_direction="a2b", text_stack=text_stack)
            m.eval(); m.half()
            models[k] = m
    H = W = 512
    g = torch.Generator(device="cuda").manual_seed(0)
    n = args.requests
    xs = (torch.rand(n, 3, H, W, device="cuda", generator=g) * 2 - 1).half()
    eps = torch.randn(n, 4, H // 8, W // 8, device="cuda", generator=g).half()
    pick = torch.Generator().manual_seed(1)
    dirs = ["a2b" if int(v) == 0 else "b2a" for v in torch.randint(0, 2, (n,), generator=pick)]

    def run(arm, bs):
        m = models[arm]
        outs = []
        for s in range(0, n, bs):
            x, e, d = xs[s:s + bs], eps[s:s + bs], dirs[s:s + bs]
            if arm == "mixed":
                outs.append(m.forward(x, direction=d, eps=e))
                continue
            y = torch.empty_like(x)
            for dd in ("a2b", "b2a"):
                idx = [i for i, v in enumerate(d) if v == dd]
                if idx:
                    sel = torch.tensor(idx, device="cuda")
                    y[sel] = m.forward(x[sel], direction=dd, eps=e[sel])
            outs.append(y)
        return torch.cat(outs)

    def timed(arm, bs):
        eng = models[arm]._get_engine()
        s0 = eng.memory_stats()["plan_builds"]
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0.record()
        run(arm, bs)
        t1.record()
        torch.cuda.synchronize()
        return {"img_s": n / (t0.elapsed_time(t1) / 1e3), "plan_builds": eng.memory_stats()["plan_builds"] - s0}

    res = {"model": "cyclegan-turbo fp16, SD-Turbo, 512x512", "card": info, "requests": n,
           "a2b_share": dirs.count("a2b") / n, "stream": {}}
    equal_all = True
    for bs in (2, 8):
        for k in range(1, bs + 1):          # warm every sub-batch size of both directions on the split arm
            for dd in ("a2b", "b2a"):
                models["split"].forward(xs[:k], direction=dd, eps=eps[:k])
        ref, got = run("split", bs), run("mixed", bs)
        torch.cuda.synchronize()
        equal = torch.equal(ref, got)
        equal_all &= equal
        del ref, got
        rows = {"mixed": [], "split": []}
        for r in range(args.rounds):
            for arm in (("mixed", "split") if r % 2 == 0 else ("split", "mixed")):
                row = timed(arm, bs)
                rows[arm].append(row)
                print("batch", bs, "round", r, arm, json.dumps(row), flush=True)
        best = {k: max(x["img_s"] for x in v) for k, v in rows.items()}
        res["stream"][bs] = {"rounds": rows, "best_img_s": best, "speedup": best["mixed"] / best["split"], "byte_equal": equal}
        print(f"batch {bs}: mixed {best['mixed']:.1f} img/s vs split {best['split']:.1f} img/s "
              f"({best['mixed'] / best['split']:.3f}x), byte-equal {equal}", flush=True)

    # the selection's own cost: all-a2b batches through the mixed plan and through the single-direction plan
    m = models["mixed"]
    res["selection"] = {}
    for bs in (8, 16):
        x, e = xs[:bs], eps[:bs]
        a = m.forward(x, direction="a2b", eps=e)
        b = m.forward(x, direction=["a2b"] * bs, eps=e)
        equal = torch.equal(a, b)
        equal_all &= equal
        ms = {"single": [], "mixed": []}
        for r in range(args.rounds):
            for arm in (("single", "mixed") if r % 2 == 0 else ("mixed", "single")):
                d = "a2b" if arm == "single" else ["a2b"] * bs
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                t0.record()
                for _ in range(args.iters):
                    m.forward(x, direction=d, eps=e)
                t1.record()
                torch.cuda.synchronize()
                ms[arm].append(t0.elapsed_time(t1) / args.iters)
        best = {k: min(v) for k, v in ms.items()}
        res["selection"][bs] = {"ms_per_forward": ms, "best_ms": best, "mixed_over_single": best["mixed"] / best["single"],
                                "byte_equal": equal}
        print(f"all-a2b batch {bs}: mixed plan {best['mixed']:.2f} ms vs single-direction plan {best['single']:.2f} ms "
              f"({best['mixed'] / best['single']:.4f}x), byte-equal {equal}", flush=True)
    res["byte_equal"] = equal_all
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        json.dump(res, open(args.json, "w"), indent=1)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
