#!/usr/bin/env python
"""bench_refold.py — what a change of the fold inputs costs: a new r for stochastic pix2pix, and a new checkpoint for a live
CycleGAN-Turbo model, through i2it_finalize_weights (every plan rebuilt) against i2it_refold_weights (weights rewritten in
place, plans and CUDA graphs kept).  DESIGN.md section 8.

    python bench_refold.py [--requests 48] [--rounds 3] [--json OUT]

Sketch-demo stream: Pix2Pix-Turbo with a TwinConv conv_in at SD-Turbo width, bf16, 512x512, batch 1, the prompt's K/V cached
(set_text).  Each request draws r from {0.2, 0.4, 0.6, 0.8, 1.0} (seeded); when r differs from the last request's, the weights
are folded again and the prompt re-bound, as the wrapper does.  The two paths run the same stream alternately for --rounds
rounds on one engine.  Per path: median and p90 host-synchronised latency per request, the fold call's time, plan builds and
graph captures, and, for the refold, the algorithmic bytes its jobs read and write and prep_jobs_kernel's device time
(torch.profiler, a separate pass) with its share of the data sheet's 3.35 TB/s.  The two paths' outputs must be byte-equal.

Checkpoint switch: CycleGAN-Turbo at SD-Turbo width, fp16, with three resident plans (batch 1 and batch 8 at 512x512, and a
uint8 720x1280 upload resized to 512x512 and back).  Two seeded checkpoints of the same structure (the three UNet adapters and
every VAE tensor of both directions) are loaded in turn; each load is timed from the load call to the first output of each
resident shape, through a new engine (the wrapper's path for a checkpoint of other keys) and in place.  Every output must equal
a fresh model of that checkpoint, byte for byte.  The card name and power limit are printed with the numbers.
"""
import argparse
import json
import os
import random
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "img2img-turbo_b200"))
sys.path.insert(0, ROOT)

HBM_BPS = 3.35e12      # H100 SXM data sheet


def pct(v, q):
    v = sorted(v)
    return v[min(len(v) - 1, int(round(q * (len(v) - 1))))]


def sketch_stream(args):
    from bench import Workload
    from _host import build_text_stack
    S, dt = 512, torch.bfloat16
    w = Workload("pix2pix", True, dt, 1, S, 0, build_text_stack(1024))
    eng, text = w.eng, w.model._encode_text(w.prompt)
    rs = random.Random(7)
    stream = [rs.choice([0.2, 0.4, 0.6, 0.8, 1.0]) for _ in range(args.requests)]
    out = torch.empty(1, 3, S, S, device="cuda", dtype=dt)
    state = {"r": None}

    def run(path, record=None):
        lat, fold_ms, nbytes = [], [], []
        s0, c0 = eng.memory_stats()["plan_builds"], eng.graph_captures()
        for i, r in enumerate(stream):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if r != state["r"]:
                t1 = time.perf_counter()
                (eng.finalize if path == "finalize" else eng.refold)(r, r, r, r)
                fold_ms.append((time.perf_counter() - t1) * 1e3)
                if path == "refold":
                    nbytes.append(eng._debug_refold_info()["bytes"])
                eng.set_text(text)
                state["r"] = r
            eng.forward(w.c_t, None, w.eps, noise_map=w.noise, r=r, out=out)
            torch.cuda.synchronize()
            lat.append((time.perf_counter() - t0) * 1e3)
            if record is not None:
                record.append(out.cpu())
        return {"lat": lat, "fold_ms": fold_ms, "bytes": nbytes,
                "plan_builds": eng.memory_stats()["plan_builds"] - s0, "graph_captures": eng.graph_captures() - c0}

    outs = {"finalize": [], "refold": []}
    runs = {"finalize": [], "refold": []}
    for rnd in range(args.rounds):
        for path in ("finalize", "refold"):
            runs[path].append(run(path, outs[path] if rnd == 0 else None))
    equal = all(torch.equal(a, b) for a, b in zip(outs["finalize"], outs["refold"]))
    assert equal, "the finalize and refold paths' outputs differ"
    res = {"requests": args.requests, "folds_per_stream": len(runs["refold"][0]["fold_ms"]), "outputs_equal": equal}
    for path in ("finalize", "refold"):
        lat = [v for x in runs[path] for v in x["lat"]]
        fold = [v for x in runs[path] for v in x["fold_ms"]]
        res[path] = {"median_ms": statistics.median(lat), "p90_ms": pct(lat, 0.9),
                     "fold_call_median_ms": statistics.median(fold),
                     "plan_builds_per_stream": [x["plan_builds"] for x in runs[path]],
                     "graph_captures_per_stream": [x["graph_captures"] for x in runs[path]]}
    res["refold"]["bytes_median"] = statistics.median([v for x in runs["refold"] for v in x["bytes"]])
    # prep_jobs_kernel device time over a few refolds, in a pass of its own
    from torch.profiler import ProfilerActivity, profile
    seq = [0.2, 0.6, 1.0, 0.4, 0.8, 0.2]
    nb = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for r in seq:
            eng.refold(r, r, r, r)
            nb.append(eng._debug_refold_info()["bytes"])
    us, n = 0.0, 0
    for ev in prof.key_averages():
        if "prep_jobs_kernel" in ev.key:
            us += getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
            n += ev.count
    if n:
        kms = us / 1e3 / n
        res["refold"].update({"prep_jobs_kernel_ms": kms, "prep_jobs_bytes": statistics.median(nb),
                              "prep_jobs_hbm_share": statistics.median(nb) / (kms / 1e3) / HBM_BPS})
    eng.set_text(text)
    w.model.release_plans()
    return res


def cyclegan_ckpt(model, seed):
    """A checkpoint in train_cyclegan_turbo.py's format with the model's structure and seeded values: new LoRA tensors for the
    three UNet adapters, every VAE tensor of both directions perturbed."""
    g = torch.Generator().manual_seed(seed)
    ck = {"rank_unet": 8, "rank_vae": 4, "sd_encoder": {}, "sd_decoder": {}, "sd_other": {}, "sd_vae_enc": {},
          "sd_vae_dec": {}}
    for k, v in model._sd.items():
        if k.startswith("unet.") and ".lora_" in k:
            for part, a in (("sd_encoder", "default_encoder"), ("sd_decoder", "default_decoder"), ("sd_other", "default_others")):
                if f".{a}." in k:
                    ck[part][k[len("unet."):].replace(f".{a}.", ".")] = torch.randn(v.shape, generator=g) * 0.02
        elif k.startswith(("vae.", "vae_b2a.")):
            part = "sd_vae_enc" if ".encoder." in k or k.split(".")[1] == "quant_conv" else "sd_vae_dec"
            ck[part][k] = v + torch.randn(v.shape, generator=g) * 0.01
    return ck


def checkpoint_switch(args):
    from cyclegan_turbo import CycleGAN_Turbo
    from _host import build_text_stack
    stack = build_text_stack(1024)

    def model():
        m = CycleGAN_Turbo(synthetic_caption="driving in the night", synthetic_direction="a2b", text_stack=stack)
        m.eval()
        return m.half()

    g = torch.Generator().manual_seed(3)
    x1 = (torch.rand(1, 3, 512, 512, generator=g) * 2 - 1).half().cuda()
    x8 = (torch.rand(8, 3, 512, 512, generator=g) * 2 - 1).half().cuda()
    e1 = torch.randn(1, 4, 64, 64, generator=g).half().cuda()
    e8 = torch.randn(8, 4, 64, 64, generator=g).half().cuda()
    u8 = torch.randint(0, 256, (1, 720, 1280, 3), generator=g, dtype=torch.uint8).cuda()
    shapes = {"batch1": lambda m: m(x1, eps=e1), "batch8": lambda m: m(x8, eps=e8),
              "resize_512x512": lambda m: m.forward_u8(u8, eps=e1, resize=(512, 512), out_size=(720, 1280))}
    m = model()
    cks = [cyclegan_ckpt(m, 1), cyclegan_ckpt(m, 2)]
    refs = []
    for ck in cks:
        f = model()
        f.load_ckpt_from_state_dict(ck)
        refs.append({k: fn(f).cpu() for k, fn in shapes.items()})
        f._get_engine().close()
        del f
    torch.cuda.empty_cache()
    for fn in shapes.values():
        fn(m)
    torch.cuda.synchronize()
    times = {"new_engine": [], "in_place": []}
    equal = True
    i = 0
    for _ in range(args.rounds):
        for path in ("new_engine", "in_place"):
            ck = cks[i % 2]
            torch.cuda.synchronize()
            if path == "new_engine":
                m._loaded = None          # no record of the registered tensors: the wrapper builds a new engine
            t0 = time.perf_counter()
            m.load_ckpt_from_state_dict(ck)
            row = {}
            for k, fn in shapes.items():
                y = fn(m)
                torch.cuda.synchronize()
                row[k] = (time.perf_counter() - t0) * 1e3
                equal = equal and torch.equal(y.cpu(), refs[i % 2][k])
            times[path].append(row)
            i += 1
    assert equal, "an output after a checkpoint switch differs from a fresh model of that checkpoint"
    res = {"outputs_equal": equal}
    for path, rows in times.items():
        res[path] = {k: statistics.median(r[k] for r in rows) for k in shapes}
        res[path]["rounds_ms"] = rows
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=48)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default="", help="also write the results here")
    args = ap.parse_args()
    from bench_plans import card
    info = card()
    print("card", json.dumps(info), flush=True)
    sk = sketch_stream(args)
    print("sketch_stream", json.dumps(sk), flush=True)
    torch.cuda.empty_cache()
    cs = checkpoint_switch(args)
    print("checkpoint_switch", json.dumps(cs), flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        json.dump({"card": info, "sketch_stream": sk, "checkpoint_switch": cs}, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
