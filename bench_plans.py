#!/usr/bin/env python
"""bench_plans.py — memory and time of the forward-plan cache on one GPU (DESIGN.md section 8).

    python bench_plans.py [--steps 10] [--warmup 3] [--json OUT]

Every forward plan of a handle keeps its transient buffers in one shared arena (the largest resident plan's need) plus a
few small persistent buffers of its own; plans beyond the handle's limit are evicted least recently run.  Three tables:

  1. BASELINE config #5: CycleGAN fp16 512x512 on one handle, per-GPU batch 1, 2, 4, 8, 16, 32 in that order.  Device-event
     img/s, the arena and cudaMemGetInfo's free memory after each batch, and the running sum of the batches' workspace_bytes
     (what one handle held before the arena: a workspace per plan).
  2. A stream of sizes: pix2pix bf16 forward_u8 with resize=paired_geometry over 24 distinct frame sizes between 640x480 and
     1920x1080, batch 1, two passes through the wrappers' default limit (16 plans).  First call per size (plan build, graph
     capture and run), the second pass (evictions force rebuilds), the replay rate, and the peak arena + persistent bytes
     against the summed workspaces.
  3. Plan build cost: host time of a plan build plus its first graph capture and run, synchronised, at 512x512 batch 8 and
     3840x2160 batch 1 (each call a rebuild: the handle keeps one plan), next to the replay time.

The card name and its power limit are printed with the tables: both are part of the numbers.
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
sys.path.insert(0, ROOT)

GiB = float(1 << 30)


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit,power.max_limit",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout.strip()
        limit, max_limit = (float(v) for v in q.split(","))
    except Exception:
        limit = max_limit = None
    return {"name": name, "memory_gib": torch.cuda.get_device_properties(0).total_memory / GiB,
            "power_limit_w": limit, "power_max_limit_w": max_limit}


def free_gib():
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0] / GiB


def config5(steps, warmup, text_stack, flush):
    from bench import Workload, timed
    w = Workload("cyclegan", False, torch.float16, 1, 512, 0, text_stack)
    eng = w.eng
    rows, held = [], 0
    for b in (1, 2, 4, 8, 16, 32):
        row = {"batch": b}
        try:
            w.set_batch(b)
            ms, _ = timed(w.step, steps, warmup, 1, None, flush)
            ws = eng.workspace_bytes(b, 512, 512)
            held += ws
            s = eng.memory_stats()
            row.update({"img_s": b / (ms / 1e3), "ms_per_step": ms, "workspace_gib": ws / GiB,
                        "arena_gib": s["arena_bytes"] / GiB, "plan_persistent_gib": s["plan_bytes"] / GiB,
                        "sum_workspaces_gib": held / GiB, "free_gib": free_gib(), "plans": s["plans"],
                        "finite": bool(torch.isfinite(w.out.float()).all().item())})
        except Exception as ex:          # reported, not hidden: a failing point must not take the other tables with it
            row["error"] = f"{type(ex).__name__}: {ex}"[:300]
        rows.append(row)
        print("config5", json.dumps(row), flush=True)
    del w, eng
    torch.cuda.empty_cache()
    return rows


def frame_sizes(n=24):
    """n distinct (H, W) between 480x640 and 1080x1920, none a multiple of 8 on both sides (the paired CLI resizes each)."""
    out = []
    for i in range(n):
        h = 480 + round(i * 600 / (n - 1))
        w = 640 + round(i * 1280 / (n - 1))
        out.append((h - (1 if h % 8 == 0 and 0 < i < n - 1 else 0), w - (3 if w % 8 == 0 and 0 < i < n - 1 else 0)))
    assert len(set(out)) == n
    return out


def size_stream(text_stack):
    from _host import paired_geometry
    from pix2pix_turbo import Pix2Pix_Turbo
    m = Pix2Pix_Turbo(text_stack=text_stack)
    m.set_eval()
    m.to(torch.bfloat16)
    prompt = "a synthetic benchmark prompt"
    g = torch.Generator(device="cuda").manual_seed(0)
    sizes = frame_sizes()
    frames = {hw: torch.randint(0, 256, (1,) + hw + (3,), device="cuda", dtype=torch.uint8, generator=g) for hw in sizes}
    m.forward_u8(frames[sizes[0]], prompt, resize=paired_geometry(*sizes[0]))     # engine, weights, prompt: not per size
    m.release_plans()
    eng = m._get_engine()
    first, replay, second, summed, peak = [], [], [], 0, 0

    def call(hw):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.forward_u8(frames[hw], prompt, resize=paired_geometry(*hw))
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    for hw in sizes:
        first.append(call(hw))
        replay.append(call(hw))
        rs = paired_geometry(*hw)
        summed += eng.workspace_bytes(1, rs[0], rs[1])
        s = eng.memory_stats()
        peak = max(peak, s["arena_bytes"] + s["plan_bytes"])
    s1 = eng.memory_stats()
    for hw in sizes:
        second.append(call(hw))
    s2 = eng.memory_stats()
    res = {"sizes": [list(hw) for hw in sizes], "first_call_s": first, "replay_s": replay, "second_pass_s": second,
           "first_call_median_s": sorted(first)[len(first) // 2], "second_pass_median_s": sorted(second)[len(second) // 2],
           "replay_img_s": len(replay) / sum(replay),
           "peak_arena_plus_persistent_gib": peak / GiB, "sum_workspaces_gib": summed / GiB,
           "after_pass1": s1, "after_pass2": s2, "free_gib": free_gib()}
    print("stream", json.dumps({k: v for k, v in res.items() if not isinstance(v, list)}), flush=True)
    m.release_plans()
    return m, res


def build_cost(m, text_dim=1024):
    eng = m._get_engine()
    eng.release_plans()
    eng.set_max_plans(1)
    g = torch.Generator(device="cuda").manual_seed(1)
    text = torch.randn(1, 77, text_dim, device="cuda", generator=g).to(torch.bfloat16)
    shapes = {"512x512 b8": (8, 512, 512), "3840x2160 b1": (1, 2160, 3840)}
    io = {k: (torch.rand(B, 3, H, W, device="cuda", generator=g).to(torch.bfloat16),
              torch.randn(B, 4, H // 8, W // 8, device="cuda", generator=g).to(torch.bfloat16),
              torch.empty(B, 3, H, W, device="cuda", dtype=torch.bfloat16)) for k, (B, H, W) in shapes.items()}
    rows = {k: {"build_capture_run_s": [], "replay_s": []} for k in shapes}

    def run(k):
        x, eps, out = io[k]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        eng.forward(x, text, eps, out=out)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    for _ in range(3):
        for k in shapes:                  # one plan at a time: every first call below is a rebuild
            rows[k]["build_capture_run_s"].append(run(k))
            rows[k]["replay_s"].append(run(k))
            rows[k]["arena_gib"] = eng.memory_stats()["arena_bytes"] / GiB
    for k, r in rows.items():
        r["build_capture_s"] = [a - b for a, b in zip(r["build_capture_run_s"], r["replay_s"])]
        print("build", k, json.dumps(r), flush=True)
    eng.set_max_plans(m.MAX_PLANS)
    eng.release_plans()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default="", help="also write the three tables here")
    args = ap.parse_args()
    assert args.steps >= 10, "at least 10 timed steps"
    from _host import build_text_stack
    info = card()
    print("card", json.dumps(info), flush=True)
    text_stack = build_text_stack(1024)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")   # > 50 MB L2, zeroed between timed steps
    res = {"card": info, "config5": config5(args.steps, args.warmup, text_stack, flush)}
    m, res["stream"] = size_stream(text_stack)
    res["build"] = build_cost(m)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        json.dump(res, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
