"""-m gpu: the forward-plan cache.  A handle's forward plans share one transient workspace (the arena), which must be
invisible in the outputs; the arena holds the largest plan, not the sum; plans are evicted least recently run and rebuilt
bit-identically; release_plans gives the memory back and keeps the prompt caches."""
import pytest
import torch

pytestmark = pytest.mark.gpu

GRAN = 2 << 20          # cuMemGetAllocationGranularity on H100


def _round(n):
    return (n + GRAN - 1) // GRAN * GRAN


def _engine(kind, dt, sd, cfg, **kw):
    import i2it
    e = i2it.Engine(dt, i2it.CYCLEGAN if kind == "cyclegan" else i2it.PIX2PIX, cfg=cfg, **kw)
    e.load_state_dict(sd)
    if kind == "pix2pix":
        e.set_adapter_scale("default", 1.0)
        e.set_adapter_scale("vae_skip", 2.0)
    else:
        for a in ("default_encoder", "default_decoder", "default_others"):
            e.set_adapter_scale(a, 1.0)
        e.set_adapter_scale("vae_skip", 2.0)
    e.finalize(1.0, 1.0, 1.0, -1.0)
    return e


def _inputs(dt, cross_dim, seed=0):
    """The three forward keys of these tests: A = NCHW batch 2 at 64x64, B = uint8 batch 1 at 64x96, C = uint8 batch 2 resized
    from 100x150 to 64x96, cropped to 64x64 at column 16, and resized back to 100x150."""
    g = torch.Generator().manual_seed(seed)
    text = torch.randn(1, 77, cross_dim, generator=g).to(dt).cuda()
    return {
        "A": dict(x=(torch.rand(2, 3, 64, 64, generator=g) * 2 - 1).to(dt).cuda(),
                  eps=torch.randn(2, 4, 8, 8, generator=g).to(dt).cuda(), text=text),
        "B": dict(u8=torch.randint(0, 256, (1, 64, 96, 3), generator=g, dtype=torch.uint8).cuda(),
                  eps=torch.randn(1, 4, 8, 12, generator=g).to(dt).cuda(), text=text),
        "C": dict(u8=torch.randint(0, 256, (2, 100, 150, 3), generator=g, dtype=torch.uint8).cuda(),
                  eps=torch.randn(2, 4, 8, 8, generator=g).to(dt).cuda(), text=text,
                  geom=dict(resize=(64, 96), crop=(0, 16, 64, 64), out_size=(100, 150))),
    }


def _run(e, inp, direction, mode, cached_text=False):
    text = None if cached_text else inp["text"]
    if "x" in inp:
        return e.forward(inp["x"], text, inp["eps"], direction=direction)
    return e.forward_u8(inp["u8"], mode, text, inp["eps"], direction=direction, **inp.get("geom", {}))


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("kind,graph", [("pix2pix", True), ("pix2pix", False), ("cyclegan", True)],
                         ids=["pix2pix-graph", "pix2pix-eager", "cyclegan-graph"])
def test_aliasing_is_invisible(kind, graph, dt, tiny_sd, tiny_sd_cyc):
    """A, B, C, A, C, B on one handle with the arena filled with 0xFF (NaN in fp16 and bf16) before every forward: each output
    equals a fresh handle that runs only that key.  CycleGAN alternates the two directions (two VAEs) on the one handle."""
    import i2it
    import weights as W
    cfg = W.TINY
    sd = tiny_sd if kind == "pix2pix" else tiny_sd_cyc
    mode = i2it.IN_UNIT if kind == "pix2pix" else i2it.IN_NORMALIZE
    inputs = _inputs(dt, cfg["cross_dim"])
    dirs = [i2it.A2B, i2it.B2A, i2it.A2B, i2it.B2A, i2it.A2B, i2it.B2A] if kind == "cyclegan" else [i2it.A2B] * 6
    order = list(zip("ABCACB", dirs))
    ref = {}
    for name, d in set(order):
        fresh = _engine(kind, dt, sd, cfg, use_cuda_graph=graph)
        ref[(name, d)] = _run(fresh, inputs[name], d, mode).cpu()
        fresh.close()
    e = _engine(kind, dt, sd, cfg, use_cuda_graph=graph)
    for name, d in order:
        e._debug_poison_workspace(0xFF)
        got = _run(e, inputs[name], d, mode)
        torch.cuda.synchronize()
        assert torch.equal(got.cpu(), ref[(name, d)]), (name, d)
    s = e.memory_stats()
    assert s["plans"] == len(set(order)) and s["plan_evictions"] == 0 and s["arena_bytes"] > 0


def test_arena_is_the_max_not_the_sum():
    """CycleGAN fp16 at SD-Turbo width, batches 1, 2, 4 at 512^2 on one handle: the arena is the largest plan's transient need
    rounded to the granularity, below the sum of the plans' workspaces, and the device memory the three builds take is the
    arena growth plus the plans' persistent bytes (slack: graph executables, cudaMalloc rounding of the small persistent
    buffers)."""
    import i2it
    import weights as W
    cfg, dt = W.SD_TURBO, torch.float16
    e = _engine("cyclegan", dt, W.make_state_dict("cyclegan", cfg, seed=0), cfg)
    g = torch.Generator().manual_seed(0)
    text = torch.randn(1, 77, cfg["cross_dim"], generator=g).to(dt).cuda()
    xs = {B: (torch.rand(B, 3, 512, 512, generator=g) * 2 - 1).to(dt).cuda() for B in (1, 2, 4)}
    eps = {B: torch.randn(B, 4, 64, 64, generator=g).to(dt).cuda() for B in (1, 2, 4)}
    outs = {B: torch.empty_like(xs[B]) for B in (1, 2, 4)}
    # a small plan first: weight preparation (engine-level, not workspace) happens at the first build
    e.forward(xs[1][:, :, :64, :64].contiguous(), text, eps[1][:, :, :8, :8].contiguous())
    torch.cuda.synchronize()
    s0 = e.memory_stats()
    free0 = torch.cuda.mem_get_info()[0]
    ws, persistent = {}, {}
    prev = s0["plan_bytes"]
    for B in (1, 2, 4):
        e.forward(xs[B], text, eps[B], out=outs[B])
        torch.cuda.synchronize()
        ws[B] = e.workspace_bytes(B, 512, 512)
        s = e.memory_stats()
        persistent[B] = s["plan_bytes"] - prev
        prev = s["plan_bytes"]
    free1 = torch.cuda.mem_get_info()[0]
    s = e.memory_stats()
    need = max(ws[B] - persistent[B] for B in (1, 2, 4))
    assert s["plans"] == 4 and s["plan_builds"] == 4
    assert s["arena_bytes"] == _round(need), (s, ws, persistent)
    assert s["arena_bytes"] < sum(ws.values())
    slack = 256 << 20
    grown = (s["arena_bytes"] - s0["arena_bytes"]) + (s["plan_bytes"] - s0["plan_bytes"])
    print(f"workspaces {ws} sum {sum(ws.values()) / 2**30:.2f} GiB; arena {s['arena_bytes'] / 2**30:.2f} GiB; "
          f"device memory taken {(free0 - free1) / 2**30:.2f} GiB (arena growth + persistent {grown / 2**30:.2f} GiB)")
    assert free0 - free1 <= grown + slack


def test_lru_eviction(tiny_sd):
    """max_plans = 2, A B C A: four builds, two evictions, the rebuilt A equals the first A bit for bit and prepares no
    weights; building a plan for a new shape (workspace_bytes) evicts, but never the last forward's plan, whose stages stay."""
    import i2it
    import weights as W
    cfg, dt = W.TINY, torch.bfloat16
    inputs = _inputs(dt, cfg["cross_dim"])
    e = _engine("pix2pix", dt, tiny_sd, cfg)
    e.set_max_plans(2)
    a1 = _run(e, inputs["A"], i2it.A2B, i2it.IN_UNIT).cpu()
    preps = e.prep_launch_count()
    _run(e, inputs["B"], i2it.A2B, i2it.IN_UNIT)
    _run(e, inputs["C"], i2it.A2B, i2it.IN_UNIT)
    a2 = _run(e, inputs["A"], i2it.A2B, i2it.IN_UNIT).cpu()
    s = e.memory_stats()
    assert (s["plan_builds"], s["plan_evictions"], s["plans"]) == (4, 2, 2), s
    assert torch.equal(a1, a2)
    assert e.prep_launch_count() == preps

    k = _engine("pix2pix", dt, tiny_sd, cfg, keep_stages=1)
    k.set_max_plans(2)
    _run(k, inputs["A"], i2it.A2B, i2it.IN_UNIT)
    _run(k, inputs["B"], i2it.A2B, i2it.IN_UNIT)
    names = [n for n, _ in k.stage_names()]
    before = {n: k.read_stage(n) for n in names}
    k.workspace_bytes(1, 64, 64)                        # a new plan: the LRU one (A) goes, B stays the last forward's
    s = k.memory_stats()
    assert (s["plans"], s["plan_evictions"]) == (2, 1), s
    assert [n for n, _ in k.stage_names()] == names
    for n in names:
        assert torch.equal(k.read_stage(n), before[n]), n
    with pytest.raises(RuntimeError, match="max_plans"):
        e.set_max_plans(-1)


def test_release_plans_keeps_prompt_caches(tiny_sd):
    """release_plans: no plan, no arena; a text_emb=None forward still uses the earlier set_text projections and equals its
    pre-release output; the text tower still encodes."""
    import i2it
    import weights as W
    from test_gpu_clip import _model, _tokens
    cfg, dt = W.TINY, torch.float16
    clip = _model(cfg["cross_dim"], 2, cfg["cross_dim"] // 64, 2 * cfg["cross_dim"])
    e = i2it.Engine(dt, i2it.PIX2PIX, cfg=cfg, text_heads=cfg["cross_dim"] // 64)
    e.load_state_dict(tiny_sd)
    e.load_state_dict({"text_encoder." + k: v for k, v in clip.state_dict().items()})
    e.set_adapter_scale("default", 1.0)
    e.set_adapter_scale("vae_skip", 2.0)
    e.finalize(1.0, 1.0, 1.0, -1.0)
    tok = _tokens(1)
    emb = e.encode_text(tok, cfg["cross_dim"])
    e.set_text(emb)
    inputs = _inputs(dt, cfg["cross_dim"])
    before = _run(e, inputs["A"], i2it.A2B, i2it.IN_UNIT, cached_text=True).cpu()
    _run(e, inputs["B"], i2it.A2B, i2it.IN_UNIT, cached_text=True)
    assert e.memory_stats()["arena_bytes"] > 0
    e.release_plans()
    s = e.memory_stats()
    assert s["arena_bytes"] == 0 and s["plans"] == 0 and s["plan_bytes"] == 0
    after = _run(e, inputs["A"], i2it.A2B, i2it.IN_UNIT, cached_text=True).cpu()
    assert torch.equal(before, after)
    assert torch.equal(e.encode_text(tok, cfg["cross_dim"]), emb)
    assert e.memory_stats()["plans"] == 1


def test_wrapper_default_limit():
    """Pix2Pix_Turbo (tiny) over 20 image sizes keeps at most 16 plans; the first and last sizes equal a fresh model's output,
    the first one again after its plan was evicted too."""
    import weights as W
    from _host import HashTokenizer
    from pix2pix_turbo import Pix2Pix_Turbo
    from test_gpu_clip import _model
    cfg = W.TINY
    clip = _model(cfg["cross_dim"], 2, cfg["cross_dim"] // 64, 2 * cfg["cross_dim"])

    def model():
        m = Pix2Pix_Turbo(cfg=cfg, text_stack=(HashTokenizer(), clip))
        m.set_eval()
        return m.half()

    sizes = [(64 + 8 * (i % 4), 64 + 8 * (i // 4)) for i in range(20)]
    g = torch.Generator().manual_seed(5)
    xs = [(torch.rand(1, 3, h, w, generator=g) < 0.1).half().cuda() for h, w in sizes]
    eps = [torch.randn(1, 4, h // 8, w // 8, generator=g).half().cuda() for h, w in sizes]
    m = model()
    outs = [m(x, "a house by a lake", eps=ep) for x, ep in zip(xs, eps)]
    s = m._get_engine().memory_stats()
    assert s["plans"] <= 16 and s["plan_builds"] == 20 and s["plan_evictions"] == 4, s
    again = m(xs[0], "a house by a lake", eps=eps[0])
    for i in (0, -1):
        ref = model()(xs[i], "a house by a lake", eps=eps[i])
        assert torch.equal(outs[i], ref), sizes[i]
    assert torch.equal(again, outs[0])
    m.release_plans()
    assert m._get_engine().memory_stats()["arena_bytes"] == 0
