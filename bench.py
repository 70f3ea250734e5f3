#!/usr/bin/env python
"""bench.py — 512x512 images/s of the one-step image-translation path on N H100s (BASELINE.json metric).

    python bench.py --gpus 1 --steps 10 --warmup 3
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        bench.py --gpus N --steps K --warmup W
    python bench.py --impl reference ...      # the reference's own (CPU) implementation of the path, host cores

One "step" = one forward of the hot path (VAE.encode -> UNet(t=999) -> DDPM x0 -> VAE.decode) over one per-GPU
batch of synthetic 512x512 inputs.  The HEADLINE (`value`, `e2e`, `roofline`) is BASELINE.md config #2: pix2pix-turbo
edge_to_image, bf16, batch 8 per GPU, random-init weights, LoRA folded.  The same JSON line carries a `configs` block with
the other BASELINE configs at the N it was launched with: #3 cyclegan day_to_night fp16 batch 16/GPU, #4 pix2pix
sketch_to_image_stochastic (TwinConv, noise map, gamma = 0.4) bf16 batch 8/GPU, #5 cyclegan clear_to_rainy fp16 per-GPU batch
sweep 1..16.  N > 1 shards images across ranks (weak scaling, no data-path collective) plus ONE NCCL all-gather of the
output latents per step.  Prints one JSON line on rank 0.

  --model/--stochastic/--batch/--dtype pick another headline workload; --configs none|3,4,5 limits the extra block.
  --dump-outputs DIR writes what the last timed step computed (output images and latents, and at N > 1 the all-gathered
  latents; float32 .npy) for comparing builds.  --steps / --warmup apply as given to every GPU timed loop of the line; the
  product arm's `cpu_baseline` is a separate one-image host sample (its size is stated in its `sample` field).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "img2img-turbo_b200"))

FLOPS_PER_IMAGE = 4467.6e9          # SURVEY.md App. B: 2*MAC over every conv / linear / attention at 512x512
CPU_THREADS = os.cpu_count()
WORKLOADS = {
    "2": "pix2pix-turbo edge_to_image bf16 batch=8/GPU 512x512 (BASELINE config #2)",
    "3": "cyclegan-turbo day_to_night (a2b) fp16 batch=16/GPU 512x512 (BASELINE config #3)",
    "4": "pix2pix-turbo sketch_to_image_stochastic (TwinConv, noise map, gamma=0.4) bf16 batch=8/GPU 512x512 (BASELINE config #4)",
    "5": "cyclegan-turbo clear_to_rainy (a2b) fp16 512x512, per-GPU batch sweep (BASELINE config #5)",
}
WORKLOAD = WORKLOADS["2"]


def measured_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return (d.get("bf16_tflops_sustained", 989.0), d.get("bf16_tflops", 989.0), d.get("hbm_gbs", 3350.0),
                "measured (MEASURED_PEAKS.json)")
    return 989.0, 989.0, 3350.0, "NVIDIA H100 SXM data sheet (dense BF16, HBM3; 700 W card)"


class ClockSampler:
    """nvidia-smi clocks + throttle reasons sampled DURING the timed region."""
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.index, self.rows, self.proc = index, [], None

    def start(self):
        """Spawn the sampler and wait for its first row: nvidia-smi's own start-up (NVML init, ~0.5 s) must not fall inside the
        timed region (it was seen to stretch a 10-step region by 25 % when it did)."""
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), f"--query-gpu={self.Q}",
                                          "--format=csv,noheader,nounits", "-lms", "200"], stdout=subprocess.PIPE, text=True)
            threading.Thread(target=self._read, daemon=True).start()
            t0 = time.time()
            while not self.rows and time.time() - t0 < 5.0:
                time.sleep(0.05)
        except Exception:
            self.proc = None

    def mark(self):
        """Rows from here on belong to the timed region."""
        self.first = len(self.rows)

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.25)
        self.proc.terminate()
        self.rows = self.rows[getattr(self, "first", 0):]
        sm = [float(r[0]) for r in self.rows if r and r[0].replace(".", "").isdigit()]
        mx = [float(r[1]) for r in self.rows if len(r) > 1 and r[1].replace(".", "").isdigit()]
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = [n for i, n in enumerate(names) if any(len(r) > 3 + i and r[3 + i].lower().startswith("active") for r in self.rows)]
        pw = [float(r[2]) for r in self.rows if len(r) > 2 and r[2].replace(".", "").isdigit()]
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "power_w_max": max(pw) if pw else None, "power_w_median": statistics.median(pw) if pw else None,
                "samples": len(sm), "reasons": reasons}


def synthetic_inputs(B, size, cross_dim, dtype, device, seed_offset=0, kind="edge"):
    """BASELINE.md inputs: edge = canny-like {0,1} control image (configs 1/2), sketch = (rand < 0.5) (config 4),
    photo = rand*2-1 (configs 3/5); randn text embedding, randn posterior eps, randn noise map (seed 42, config 4)."""
    g = torch.Generator().manual_seed(1 + seed_offset)
    if kind == "photo":
        c_t = torch.rand(B, 3, size, size, generator=g) * 2 - 1
    else:
        c_t = (torch.rand(B, 1, size, size, generator=g) < (0.08 if kind == "edge" else 0.5)).float().expand(-1, 3, -1, -1).contiguous()
    text = torch.randn(1, 77, cross_dim, generator=torch.Generator().manual_seed(2))
    eps = torch.randn(B, 4, size // 8, size // 8, generator=torch.Generator().manual_seed(3 + seed_offset))
    noise = torch.randn(B, 4, size // 8, size // 8, generator=torch.Generator().manual_seed(42 + seed_offset))
    mv = (lambda t: t.to(dtype).to(device)) if device else (lambda t: t.to(dtype))
    return mv(c_t), mv(text), mv(eps), mv(noise)


def cpu_oracle_images_per_s(sd, size, steps, warmup, cross_dim, cfg):
    """The reference's algorithm on the host cores: oracle/ (fp32 restatement of the diffusers path), B=1 per step."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import oracle as O
    c_t, text, eps, _ = synthetic_inputs(1, size, cross_dim, torch.float32, None)
    # pick the host thread count that is actually fastest (oversubscribed many-core hosts are slower with every thread)
    cs, ts, es, _ = synthetic_inputs(1, 128, cross_dim, torch.float32, None)
    best = (1e30, os.cpu_count())
    with torch.no_grad():
        for nt in sorted({os.cpu_count(), 64, 32, 16}):
            if nt > os.cpu_count():
                continue
            torch.set_num_threads(nt)
            O.pix2pix_forward(sd, cs, ts, es, cfg)
            t0 = time.time()
            O.pix2pix_forward(sd, cs, ts, es, cfg)
            best = min(best, (time.time() - t0, nt))
    torch.set_num_threads(best[1])
    global CPU_THREADS
    CPU_THREADS = best[1]
    with torch.no_grad():
        for _ in range(warmup):
            O.pix2pix_forward(sd, c_t, text, eps, cfg)
        t0 = time.time()
        for _ in range(steps):
            O.pix2pix_forward(sd, c_t, text, eps, cfg)
        dt = (time.time() - t0) / steps
    return 1.0 / dt, dt


def run_reference(args):
    """--impl reference: the reference's own CPU implementation of the path.  diffusers/peft are not a dependency of this
    project (DESIGN.md), so this times oracle/ — the restatement of the same algorithm —
    with every host thread.  One step = one image of --size (batch 1); --steps / --warmup are taken as given."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    import weights as W
    sd = W.make_state_dict("pix2pix", W.SD_TURBO, seed=0)
    steps, warmup = args.steps, args.warmup
    ips, sec = cpu_oracle_images_per_s(sd, args.size, steps, warmup, 1024, W.SD_TURBO)
    cores = CPU_THREADS
    line = {"impl": "reference", "metric": "512x512 images/sec", "value": ips, "unit": "images/s", "n_gpus": args.gpus,
            "steps": steps, "warmup": warmup, "ms_per_step": sec * 1e3, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": WORKLOAD, "note": "CPU arm: fp32, batch 1 per step, all host threads"},
            "cpu_baseline": {"value": ips, "unit": "images/s", "cores": cores, "kind": "port",
                             "sample": f"{steps} x one {args.size}x{args.size} image, oracle fp32 (steps/warmup capped at 3/1)"},
            "e2e": {"value": ips, "unit": "images/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line), flush=True)


# ------------------------------------------------------------------------------------------------------------------
# workloads
# ------------------------------------------------------------------------------------------------------------------
class Workload:
    """One BASELINE config on this rank: the model (public reference-compatible API), device-resident inputs and the
    engine-level step (inputs in HBM, text projections cached per prompt)."""

    def __init__(self, kind, stochastic, dt, B, S, rank, text_stack):
        from pix2pix_turbo import Pix2Pix_Turbo
        from cyclegan_turbo import CycleGAN_Turbo
        import i2it
        self.kind, self.stochastic, self.dt, self.B, self.S = kind, stochastic, dt, B, S
        t0 = time.time()
        if kind == "pix2pix":
            # pretrained_name=None, pretrained_path=None -> random init (reference pix2pix_turbo.py:131); the stochastic model
            # carries a TwinConv conv_in with two distinct random weight sets (what sketch_to_image_stochastic loads)
            self.model = Pix2Pix_Turbo(text_stack=text_stack, twin=stochastic)
            self.model.set_eval()
            self.prompt = "a synthetic benchmark prompt"
            self.direction = i2it.A2B
        else:
            self.model = CycleGAN_Turbo(synthetic_caption="driving in the night", synthetic_direction="a2b", text_stack=text_stack)
            self.model.eval()
            self.prompt = self.model.caption
            self.direction = i2it.A2B
        self.model.to(dt)
        self.t_weights = time.time() - t0
        self.rank = rank
        self.r = 0.4
        self.set_batch(B)
        t0 = time.time()
        with torch.no_grad():
            self.out_api = self.call(self.c_t, eps=self.eps)      # builds engine + plan, caches the prompt embedding + K/V
        torch.cuda.synchronize()
        self.t_engine = time.time() - t0
        self.eng = self.model._get_engine()

    def set_batch(self, B):
        S, dt = self.S, self.dt
        kind = "photo" if self.kind == "cyclegan" else ("sketch" if self.stochastic else "edge")
        self.B = B
        self.c_t, _, self.eps, self.noise = synthetic_inputs(B, S, 1024, dt, "cuda", seed_offset=self.rank, kind=kind)
        self.out = torch.empty(B, 3, S, S, device="cuda", dtype=dt)
        self.lat = torch.empty(B, 4, S // 8, S // 8, device="cuda", dtype=dt)

    def call(self, x, **kw):
        """The call a user of the reference makes."""
        if self.kind == "pix2pix":
            if self.stochastic:
                return self.model(x, self.prompt, deterministic=False, r=self.r, noise_map=self.noise, **kw)
            return self.model(x, self.prompt, **kw)
        return self.model(x, **kw)

    def step(self):
        """Engine-level step: inputs resident in HBM, text K/V cached (i2it_set_text ran when the prompt was bound)."""
        self.eng.forward(self.c_t, None, self.eps, noise_map=self.noise if self.stochastic else None,
                         r=self.r if self.stochastic else 1.0, direction=self.direction, out=self.out, out_latent=self.lat)


def make_step(w, world, dist):
    """The timed step of one workload on this rank: the engine-level forward plus, at N > 1, the single collective
    (all-gather of the output latents, 32 KB per image).  Returns (step, finish, description).

    Default: the collective is issued on the compute stream after every step.  I2IT_OVERLAP_GATHER=1 issues it on a SIDE stream
    so that step i+1 computes while the all-gather of step i is in flight (two alternating latent / gather buffers; a step
    waits for the gather that read its buffer two steps back; `finish` joins the side stream into the timed stream before the
    closing event, so all K collectives complete inside the timed region).  The synchronous form is the default."""
    if world == 1:
        return w.step, None, "none"
    B, S, dt = w.B, w.S, w.dt
    if os.environ.get("I2IT_OVERLAP_GATHER") is None:
        gathered = torch.empty(world * B, 4, S // 8, S // 8, device="cuda", dtype=dt)

        w.gathered = gathered

        def step_sync():
            w.step()
            dist.all_gather_into_tensor(gathered, w.lat)              # the single collective: output latents over NVLink
        return step_sync, None, "all_gather_into_tensor(output latents) on the compute stream"
    side = torch.cuda.Stream()
    lats = [w.lat, torch.empty_like(w.lat)]
    gath = [torch.empty(world * B, 4, S // 8, S // 8, device="cuda", dtype=dt) for _ in range(2)]
    gdone = [None, None]
    cnt = [0]

    def step():
        i = cnt[0] & 1
        cur = torch.cuda.current_stream()
        if gdone[i] is not None:
            cur.wait_event(gdone[i])
        w.lat = lats[i]
        w.step()
        ev = torch.cuda.Event()
        ev.record(cur)
        with torch.cuda.stream(side):
            side.wait_event(ev)
            dist.all_gather_into_tensor(gath[i], lats[i])
            w.gathered = gath[i]
            gdone[i] = torch.cuda.Event()
            gdone[i].record(side)
        cnt[0] += 1

    def finish():
        torch.cuda.current_stream().wait_stream(side)
    return step, finish, "all_gather_into_tensor(output latents) on a side stream, overlapped with the next step"


def timed(step_fn, K, Wm, world, dist, flush, finish=None):
    """W warm-up steps, then K steps bracketed by barrier + synchronize, CUDA events, MAX over ranks.  Returns
    (ms_per_step_max_over_ranks, this rank's ms_per_step).  `finish` joins side streams (the overlapped collective) into the
    timed stream before the closing event, so every collective of the K steps completes inside the timed region."""
    for _ in range(Wm):
        flush.zero_()
        step_fn()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(K):
        flush.zero_()                                                  # L2 flush between iterations
        step_fn()
    if finish is not None:
        finish()
    e1.record()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    mine = e0.elapsed_time(e1) / K
    t = torch.tensor([mine], device="cuda")
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.item(), mine


def dump_outputs(out_dir, wl):
    """What the timed step hands its caller, as float32: this rank's output images [B, 3, S, S] and latents [B, 4, S/8, S/8],
    and at N > 1 the all-gathered latents of every rank [N*B, 4, S/8, S/8] (out_latent_gathered).  At most 64 MB in all: a batch
    too large for that is cut to its first images."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    torch.cuda.synchronize()
    gathered = getattr(wl, "gathered", None)
    per_image = 4 * (wl.out[0].numel() + wl.lat[0].numel())
    budget = (64 << 20) - (4 * gathered.numel() if gathered is not None else 0)
    keep = max(1, min(wl.out.shape[0], budget // per_image))
    arrays = [("out", wl.out[:keep]), ("out_latent", wl.lat[:keep])]
    if gathered is not None:
        arrays.append(("out_latent_gathered", gathered))
    for name, t in arrays:
        np.save(os.path.join(out_dir, name + ".npy"), t.float().cpu().numpy())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--batch", type=int, default=None, help="images per GPU per step (default 8 pix2pix / 16 cyclegan)")
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--dtype", default=None, choices=["bf16", "fp16"])
    ap.add_argument("--model", default="pix2pix", choices=["pix2pix", "cyclegan"],
                    help="headline workload: pix2pix = BASELINE config #2 (default); cyclegan = config #3")
    ap.add_argument("--stochastic", action="store_true", help="headline = pix2pix stochastic (TwinConv, noise map, gamma 0.4): config #4")
    ap.add_argument("--configs", default="3,4,5", help="extra BASELINE configs reported in the `configs` block ('none' to skip)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--profile-out", default="", help="write the per-launch timing table (JSON) here")
    ap.add_argument("--dump-outputs", default="", metavar="DIR",
                    help="after the timed steps, write the last step's outputs as DIR/<name>.npy (float32): rank 0's images and "
                         "latents, and at --gpus > 1 the all-gathered latents of every rank")
    args = ap.parse_args()
    if args.steps < 1 or args.warmup < 0:
        ap.error("--steps must be >= 1 and --warmup >= 0")
    if args.impl == "reference":
        return run_reference(args)

    import torch.distributed as dist
    import weights as W
    from _host import build_text_stack

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    if args.stochastic:
        args.model = "pix2pix"
    if args.dtype is None:
        args.dtype = "bf16" if args.model == "pix2pix" else "fp16"
    if args.batch is None:
        args.batch = 8 if args.model == "pix2pix" else 16
    dt = torch.bfloat16 if args.dtype == "bf16" else torch.float16
    B, S, K, Wm = args.batch, args.size, args.steps, args.warmup
    head_id = "4" if args.stochastic else ("2" if args.model == "pix2pix" else "3")
    workload = WORKLOADS[head_id]
    extra = [] if args.configs == "none" else [c for c in args.configs.split(",") if c in ("2", "3", "4", "5") and c != head_id]

    torch.manual_seed(0)
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        text_stack = build_text_stack(1024)
    t_build0 = time.time()
    wl = Workload(args.model, args.stochastic, dt, B, S, rank, text_stack)
    eng = wl.eng
    build_s = {"weights_init_s": round(wl.t_weights, 2), "engine_upload_fold_plan_first_forward_s": round(wl.t_engine, 2),
               "prep_launches": eng.prep_launch_count()}

    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")   # > 50 MB L2
    step, finish, collective = make_step(wl, world, dist)

    sampler = ClockSampler(local)
    sampler.start()                      # before the warm-up: its start-up cost stays out of the timed region
    for _ in range(Wm):
        flush.zero_()
        step()
    torch.cuda.synchronize()
    sampler.mark()
    if finish is not None:
        finish()
    ms_step, ms_mine = timed(step, K, 0, world, dist, flush, finish)
    clocks = sampler.stop()
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, wl)
    value = world * B / (ms_step / 1e3)
    finite = bool(torch.isfinite(wl.out.float()).all().item())

    # ---- multi-GPU: where does the scaling loss come from?  per-rank step time with and without the collective ----
    scaling_diag = None
    if world > 1:
        _, mine_nocoll = timed(wl.step, K, 1, world, dist, flush)
        both = torch.tensor([ms_mine, mine_nocoll], device="cuda")
        allr = torch.empty(world, 2, device="cuda")
        dist.all_gather_into_tensor(allr, both)
        a = allr.cpu()
        scaling_diag = {"per_rank_ms_with_allgather": [round(v, 3) for v in a[:, 0].tolist()],
                        "per_rank_ms_no_collective": [round(v, 3) for v in a[:, 1].tolist()],
                        "note": "independent replicas (no collective) vs lock-step with the per-step all-gather; the step "
                                "time reported is the MAX over ranks"}

    # ---- e2e: the call a user makes (model(c_t, prompt)) with pinned-host input and a device->host read of the result ----
    kind = "photo" if args.model == "cyclegan" else ("sketch" if args.stochastic else "edge")
    host_in = synthetic_inputs(B, S, 1024, dt, None, seed_offset=rank, kind=kind)[0].pin_memory()
    host_out = torch.empty(B, 3, S, S, dtype=dt).pin_memory()
    gathered_img = torch.empty(world * B, 3, S, S, device="cuda", dtype=dt) if world > 1 else None

    def e2e_loop(fn_in, fn_call, fn_out, gather_buf):
        with torch.no_grad():
            for _ in range(Wm):
                fn_out(fn_call(fn_in()))
            torch.cuda.synchronize()
            if world > 1:
                dist.barrier()
            t0 = time.perf_counter()
            for _ in range(K):
                flush.zero_()
                y = fn_call(fn_in())                                     # H2D + randn(eps) + path (the call a user makes)
                if world > 1:
                    dist.all_gather_into_tensor(gather_buf, y)          # sharded users gather the images (dist.sharded_forward)
                fn_out(y)                                                # D2H of the step's result
                torch.cuda.synchronize()
            s = (time.perf_counter() - t0) / K
        te = torch.tensor([s], device="cuda")
        if world > 1:
            dist.all_reduce(te, op=dist.ReduceOp.MAX)
        return world * B / te.item()

    e2e_value = e2e_loop(lambda: host_in.cuda(non_blocking=True), wl.call, lambda y: host_out.copy_(y, non_blocking=True), gathered_img)
    io_bytes = B * 3 * S * S * 2
    # the uint8 HWC boundary (pre/post-processing fused on the GPU): 3 bytes per pixel each way
    u8_in = (torch.rand(B, S, S, 3) * 255).to(torch.uint8).pin_memory()
    u8_out = torch.empty(B, S, S, 3, dtype=torch.uint8).pin_memory()
    gathered_u8 = torch.empty(world * B, S, S, 3, device="cuda", dtype=torch.uint8) if world > 1 else None
    if args.model == "pix2pix":
        if args.stochastic:
            call_u8 = lambda x: wl.model.forward_u8(x, wl.prompt, deterministic=False, r=wl.r, noise_map=wl.noise, sketch=True)
        else:
            call_u8 = lambda x: wl.model.forward_u8(x, wl.prompt)
    else:
        call_u8 = lambda x: wl.model.forward_u8(x)
    e2e_u8_value = e2e_loop(lambda: u8_in.cuda(non_blocking=True), call_u8, lambda y: u8_out.copy_(y, non_blocking=True), gathered_u8)

    # ---- the other BASELINE configs, same N, same timing rules, same --steps / --warmup ----
    configs = {head_id: {"workload": workload, "value": value, "ms_per_step": ms_step, "per_gpu_batch": B, "dtype": args.dtype,
                         "finite": finite}}
    cyc = None
    for cid in extra:
        try:
            if cid in ("3", "5"):
                if cyc is None:
                    cyc = Workload("cyclegan", False, torch.float16, 16, S, rank, text_stack)
                w2 = cyc
            elif cid == "4":
                w2 = Workload("pix2pix", True, torch.bfloat16, 8, S, rank, text_stack)
            else:
                w2 = Workload("pix2pix", False, torch.bfloat16, 8, S, rank, text_stack)
            sweep = [1, 2, 4, 8, 16] if cid == "5" else [w2.B]     # batch 32 does not fit next to the cached plans in 80 GB
            rows = []
            for b in sweep:
                w2.set_batch(b)
                step2, fin2, _ = make_step(w2, world, dist)
                ms2, _ = timed(step2, K, Wm, world, dist, flush, fin2)
                if fin2 is not None:
                    fin2()
                    torch.cuda.synchronize()
                rows.append({"per_gpu_batch": b, "global_batch": world * b, "value": world * b / (ms2 / 1e3), "ms_per_step": ms2,
                             "finite": bool(torch.isfinite(w2.out.float()).all().item()),
                             "step_tensor_frac_of_sustained_peak": (b * FLOPS_PER_IMAGE / (ms2 * 1e-3)) / 1e12 / measured_peaks()[0]})
            entry = {"workload": WORKLOADS[cid], "dtype": "fp16" if w2.dt == torch.float16 else "bf16", "steps": K, "warmup": Wm,
                     "n_gpus": world}
            if cid == "5":
                entry["sweep"] = rows
            else:
                entry.update(rows[0])
            configs[cid] = entry
            if cid == "4":
                del w2
                torch.cuda.empty_cache()
        except Exception as ex:   # a failing extra config must not take the headline line with it; it is reported, not hidden
            configs[cid] = {"workload": WORKLOADS[cid], "error": f"{type(ex).__name__}: {ex}"[:300]}

    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return

    # ---- roofline of the dominant kernel (tapgemm = every conv/linear/attention GEMM), per-launch CUDA events ----
    peak_tf, peak_burst, peak_gbs, peak_src = measured_peaks()
    wl.set_batch(B)
    wl.step()
    torch.cuda.synchronize()
    prof = eng.profile(reps=2)
    if args.profile_out:
        os.makedirs(os.path.dirname(os.path.abspath(args.profile_out)), exist_ok=True)
        json.dump(prof, open(args.profile_out, "w"))
    by_kind = {}
    for p in prof:
        k = by_kind.setdefault(p["kind"], {"ms": 0.0, "flops": 0.0, "bytes": 0.0, "n": 0})
        k["ms"] += p["ms"]; k["flops"] += p["flops"]; k["bytes"] += p["bytes"]; k["n"] += 1
    tg = [p for p in prof if p["kind"].startswith("tapgemm")]
    tg_ms, tg_fl = sum(p["ms"] for p in tg), sum(p["flops"] for p in tg)
    all_ms = sum(p["ms"] for p in prof)
    achieved = tg_fl / (tg_ms * 1e-3) / 1e12 if tg_ms > 0 else 0.0
    gn_ms = sum(v["ms"] for k, v in by_kind.items() if k.startswith("gn_"))
    gn_bytes = sum(v["bytes"] for k, v in by_kind.items() if k.startswith("gn_"))
    roofline = {"bound": "tensor", "kernel": "tapgemm_kernel (wgmma implicit GEMM: conv3x3/1x1/linear/attention; "
                                             "all launches of a step)",
                "achieved": achieved, "peak": peak_burst, "unit": "TFLOP/s", "frac": achieved / peak_burst, "peak_source": peak_src,
                "frac_of_sustained_peak": achieved / peak_tf,
                "launches_per_step": len(tg), "avg_launch_ms": tg_ms / max(1, len(tg)),
                "share_of_step": tg_ms / all_ms if all_ms else None,
                "algorithmic_bytes": sum(p["bytes"] for p in tg),
                "step_tensor_frac": (B * FLOPS_PER_IMAGE / (ms_step * 1e-3)) / 1e12 / peak_tf,
                "step_tensor_frac_note": "whole step in graph replay (long run): images x 4467.6 GFLOP / step time / SUSTAINED peak",
                "by_kind_ms": {k: round(v["ms"], 4) for k, v in sorted(by_kind.items(), key=lambda kv: -kv[1]["ms"])},
                "by_kind_launches": {k: v["n"] for k, v in by_kind.items()},
                "groupnorm": {"ms": round(gn_ms, 4), "bytes": gn_bytes, "gbs": round(gn_bytes / (gn_ms * 1e-3) / 1e9, 1) if gn_ms else None,
                              "peak_gbs": peak_gbs},
                "hbm_kernels_gbs": {k: round(v["bytes"] / (v["ms"] * 1e-3) / 1e9, 1) for k, v in by_kind.items()
                                    if not k.startswith("tapgemm") and v["ms"] > 0 and v["bytes"] > 0}}

    cpu = None
    if not args.no_cpu_baseline and world == 1 and args.model == "pix2pix" and not args.stochastic:
        ips, sec = cpu_oracle_images_per_s(wl.model._sd, S, 1, 0, 1024, W.SD_TURBO)
        cpu = {"value": ips, "unit": "images/s", "cores": CPU_THREADS, "kind": "port",
               "sample": f"1 x one {S}x{S} image (batch 1), oracle fp32 restatement of the diffusers path, {sec:.1f} s"}

    line = {"metric": "512x512 images/sec", "value": value, "unit": "images/s", "n_gpus": world, "steps": K, "warmup": Wm,
            "ms_per_step": ms_step, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": args.dtype,
            "data": "synthetic",
            "config": {"workload": workload, "per_gpu_batch": B, "global_batch": world * B, "size": S,
                       "parallelism": f"dp{world}", "l2": "256 MiB flush write between timed iterations",
                       "collective": ("1 x " + collective + " per step") if world > 1 else "none",
                       "cuda_graph": True, "text": "prompt K/V projected once per prompt (i2it_set_text), not per step"},
            "e2e": {"value": e2e_value, "unit": "images/s", "h2d_bytes_per_step": io_bytes, "d2h_bytes_per_step": io_bytes,
                    "api": "model(c_t, prompt) — the reference's call; pinned host tensor in, pinned host tensor out"},
            "e2e_u8": {"value": e2e_u8_value, "unit": "images/s", "h2d_bytes_per_step": B * S * S * 3, "d2h_bytes_per_step": B * S * S * 3,
                       "api": "model.forward_u8(uint8 HWC) — pre/post-processing fused on the GPU"},
            "gpu_launches": K * eng.launch_count(B, S, S, wl.direction), "clocks": clocks, "finite": finite,
            "engine_build": build_s, "configs": configs, "scaling_diag": scaling_diag,
            "roofline": roofline, "cpu_baseline": cpu}
    print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
