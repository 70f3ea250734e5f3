"""-m gpu: variations of one image (i2it_forward with shared_input).  The VAE encoder runs once at
batch 1 and its moments and skips feed n outputs; image i of a batch is bit-identical to its batch-1 forward, so every case
here compares BIT FOR BIT with the plain forward on the image repeated n times (which the layer audits pin to float64)."""
import pytest
import torch

from test_gpu_plans import _engine

pytestmark = pytest.mark.gpu


def _rep(x, n):
    return x.expand(n, *x.shape[1:]).contiguous()


def _operands(n, H, W, dt, cross, text_batch, stochastic, seed=0):
    g = torch.Generator().manual_seed(seed)
    return dict(x=(torch.rand(1, 3, H, W, generator=g) * 2 - 1).to(dt).cuda(),
                text=torch.randn(text_batch, 77, cross, generator=g).to(dt).cuda(),
                eps=torch.randn(n, 4, H // 8, W // 8, generator=g).to(dt).cuda(),
                noise=torch.randn(n, 4, H // 8, W // 8, generator=g).to(dt).cuda() if stochastic else None)


CASES = {
    # kind, dtype, width config, n, H, W, text (inline text_batch or "cached"), r (None: deterministic), direction
    "pix2pix-bf16-det-odd": ("pix2pix", torch.bfloat16, "tiny", 3, 72, 104, "inline-n", None, "a2b"),
    "pix2pix-fp16-twin-cached": ("twin", torch.float16, "tiny", 4, 64, 64, "cached", 0.4, "a2b"),
    "cyclegan-fp16-b2a": ("cyclegan", torch.float16, "tiny", 2, 64, 64, "inline-1", None, "b2a"),
    "pix2pix-bf16-sdturbo-256": ("pix2pix", torch.bfloat16, "sd", 2, 256, 256, "inline-1", None, "a2b"),
}


@pytest.mark.parametrize("case", list(CASES))
def test_outputs_equal_repeated_batch(case, tiny_sd, tiny_sd_cyc):
    import i2it
    import weights as W
    kind, dt, width, n, H, Wd, text, r, d = CASES[case]
    cfg = W.TINY if width == "tiny" else W.SD_TURBO
    if kind == "twin":
        sd = W.make_state_dict("pix2pix", cfg, seed=0, twin=True, perturb_norm=True)
    elif width == "sd":
        sd = W.make_state_dict(kind, cfg, seed=0)
    else:
        sd = tiny_sd if kind == "pix2pix" else tiny_sd_cyc
    e = _engine("cyclegan" if kind == "cyclegan" else "pix2pix", dt, sd, cfg)
    if r is not None:
        e.finalize(r, r, r, r)
    direction = i2it.B2A if d == "b2a" else i2it.A2B
    op = _operands(n, H, Wd, dt, cfg["cross_dim"], n if text == "inline-n" else 1, r is not None)
    temb = op["text"]
    if text == "cached":
        e.set_text(op["text"])
        temb = None
    rr = 1.0 if r is None else r
    lat_v = torch.empty(n, 4, H // 8, Wd // 8, device="cuda", dtype=dt)
    lat_p = torch.empty_like(lat_v)
    out_v = e.forward_variations(op["x"], temb, op["eps"], op["noise"], rr, direction, out_latent=lat_v)
    out_p = e.forward(_rep(op["x"], n), temb, op["eps"], op["noise"], rr, direction, out_latent=lat_p)
    torch.cuda.synchronize()
    assert out_v.shape == (n, 3, H, Wd) and torch.isfinite(out_v.float()).all()
    assert torch.equal(out_v, out_p) and torch.equal(lat_v, lat_p)
    assert not torch.equal(out_v[0], out_v[1])              # the variations do differ
    if case == "pix2pix-bf16-det-odd":                      # ... and each equals its own batch-1 forward
        for i in range(n):
            one = e.forward(op["x"], op["text"][i:i + 1], op["eps"][i:i + 1].contiguous(), direction=direction)
            assert torch.equal(one[0], out_v[i]), i


@pytest.mark.parametrize("geom", ["none", "sketch", "resize-crop-out"])
def test_u8_paths_equal_repeated_frame(geom, tiny_sd):
    """forward_u8_variations with no geometry, the sketch threshold, and a resize + crop + output resize equals forward_u8 /
    the resize forward on the frame repeated n times."""
    import i2it
    import weights as W
    cfg, dt, n = W.TINY, torch.bfloat16, 3
    e = _engine("pix2pix", dt, tiny_sd, cfg)
    g = torch.Generator().manual_seed(3)
    kw, mode = {}, i2it.IN_UNIT
    if geom == "resize-crop-out":
        frame = torch.randint(0, 256, (1, 100, 150, 3), generator=g, dtype=torch.uint8).cuda()
        kw = dict(resize=(64, 96), crop=(0, 16, 64, 64), out_size=(100, 150))
        H, Wd = 64, 64
    else:
        frame = torch.randint(0, 256, (1, 64, 96, 3), generator=g, dtype=torch.uint8).cuda()
        H, Wd = 64, 96
        mode = i2it.IN_SKETCH if geom == "sketch" else i2it.IN_UNIT
    text = torch.randn(1, 77, cfg["cross_dim"], generator=g).to(dt).cuda()
    eps = torch.randn(n, 4, H // 8, Wd // 8, generator=g).to(dt).cuda()
    lat_v = torch.empty(n, 4, H // 8, Wd // 8, device="cuda", dtype=dt)
    lat_p = torch.empty_like(lat_v)
    got = e.forward_u8_variations(frame, mode, text, eps, out_latent=lat_v, **kw)
    ref = e.forward_u8(_rep(frame, n), mode, text, eps, out_latent=lat_p, **kw)
    torch.cuda.synchronize()
    assert got.shape == ref.shape and got.shape[0] == n
    assert torch.equal(got, ref) and torch.equal(lat_v, lat_p)


REPLICA_OF = {"vae.decoder.skip_conv_1.replica": "skip3", "vae.decoder.skip_conv_2.replica": "skip2",
              "vae.decoder.skip_conv_3.replica": "skip1", "vae.decoder.skip_conv_4.replica": "skip0"}


def test_every_stage_equals_plain_forward(tiny_sd):
    """keep_stages = 2: each stage of the variations forward equals the plain batch-n stage of the same name; encoder stages
    (batch 1) equal image 0 of it; each replica equals its skip broadcast over n.  A wiring error fails on its own layer."""
    import weights as W
    cfg, dt, n = W.TINY, torch.bfloat16, 3
    op = _operands(n, 64, 64, dt, cfg["cross_dim"], 1, False, seed=4)
    ep = _engine("pix2pix", dt, tiny_sd, cfg, keep_stages=2)
    ep.forward(_rep(op["x"], n), op["text"], op["eps"])
    plain = dict(ep.stage_names())
    pstage = {name: ep.read_stage(name) for name in plain}
    ev = _engine("pix2pix", dt, tiny_sd, cfg, keep_stages=2)
    ev.forward_variations(op["x"], op["text"], op["eps"])
    var = dict(ev.stage_names())
    assert set(var) - set(plain) == set(REPLICA_OF), set(var) ^ set(plain)
    assert set(plain) <= set(var)
    batch1 = []
    for name, dims in var.items():
        got = ev.read_stage(name)
        if name in REPLICA_OF:
            skip = ev.read_stage(REPLICA_OF[name])
            assert dims[0] == n and skip.shape[0] == 1, name
            assert torch.equal(got, skip.expand(n, -1, -1, -1)), name
            continue
        ref = pstage[name]
        if dims[0] == 1 and ref.shape[0] == n:
            batch1.append(name)
            ref = ref[:1]
        assert torch.equal(got, ref), name
    assert {"skip0", "skip1", "skip2", "skip3", "enc_mid", "moments", "vae.encoder.conv_in"} <= set(batch1)
    assert "latent" not in batch1 and "vae.decoder.conv_in" not in batch1


def test_launch_list(tiny_sd):
    """i2it_profile: the batch-1 plan's launches through the moments, then the batch-n plan's from the latent sample on, with
    four replication launches inserted, each right before the launch that reads its skip."""
    import weights as W
    cfg, dt, n = W.TINY, torch.bfloat16, 3
    op = _operands(n, 64, 64, dt, cfg["cross_dim"], 1, False, seed=5)
    e = _engine("pix2pix", dt, tiny_sd, cfg)

    def launches():
        return [(p["kind"], p["shape"]) for p in e.profile(1)]

    e.forward(op["x"], op["text"], op["eps"][:1].contiguous())
    p1 = launches()
    e.forward(_rep(op["x"], n), op["text"], op["eps"])
    pn = launches()
    e.forward_variations(op["x"], op["text"], op["eps"])
    pv = launches()
    assert e.launch_count(n, 64, 64) == len(pv) == len(pn) + 4
    k = [kind for kind, _ in p1].index("misc")              # the latent sample: the first shape-less launch
    assert [kind for kind, _ in pn].index("misc") == k
    reps = [i for i, (kind, _) in enumerate(pv) if kind == "replicate"]
    assert len(reps) == 4 and reps[0] > k
    vc = cfg["vae_channels"]                                 # skip i is the input of down block i: skip3 is replicated first
    assert [s for kind, s in pv if kind == "replicate"] == [f"{n}x8x8x{vc[2]}", f"{n}x16x16x{vc[1]}", f"{n}x32x32x{vc[0]}",
                                                            f"{n}x64x64x{vc[0]}"]
    assert [l for l in pv if l[0] != "replicate"] == p1[:k] + pn[k:]
    # mid_block.resnets.1 (norm1, conv1, norm2 before its conv2 reads the skip) and the three upsampler convs
    for i in reps[1:]:
        assert pv[i + 1][0].startswith("tapgemm"), pv[i + 1]
    assert pv[reps[0] + 1][0].startswith("gn"), pv[reps[0] + 1]


def test_arena_sharing_and_eviction(tiny_sd):
    """Variations, plain batch-n and plain batch-1 forwards interleaved on one handle with the arena poisoned before each:
    every output equals a fresh handle's.  With one plan allowed, the variations plan is evicted and rebuilt bit-identically."""
    import weights as W
    cfg, dt, n = W.TINY, torch.float16, 3
    op = _operands(n, 64, 64, dt, cfg["cross_dim"], 1, False, seed=6)
    xr, e1 = _rep(op["x"], n), op["eps"][:1].contiguous()
    runs = {"var": lambda e: e.forward_variations(op["x"], op["text"], op["eps"]),
            "plain": lambda e: e.forward(xr, op["text"], op["eps"]),
            "one": lambda e: e.forward(op["x"], op["text"], e1)}
    ref = {}
    for name, run in runs.items():
        fresh = _engine("pix2pix", dt, tiny_sd, cfg)
        ref[name] = run(fresh).cpu()
        fresh.close()
    assert torch.equal(ref["var"], ref["plain"]) and torch.equal(ref["var"][0], ref["one"][0])
    e = _engine("pix2pix", dt, tiny_sd, cfg)
    for name in ["var", "plain", "one", "var", "one", "plain", "var"]:
        e._debug_poison_workspace(0xFF)
        got = runs[name](e)
        torch.cuda.synchronize()
        assert torch.equal(got.cpu(), ref[name]), name
    s = e.memory_stats()
    assert (s["plans"], s["plan_builds"], s["plan_evictions"]) == (3, 3, 0), s
    e.set_max_plans(1)                                       # keeps the last-run plan: the variations one
    for name in ["one", "var", "plain", "var"]:             # each forward rebuilds its plan and evicts the previous one
        e._debug_poison_workspace(0xFF)
        assert torch.equal(runs[name](e).cpu(), ref[name]), name
    s = e.memory_stats()
    assert (s["plans"], s["plan_builds"], s["plan_evictions"]) == (1, 7, 6), s


def test_variations_rejections_keep_the_handle_usable(tiny_sd):
    """n = 0, a text batch that is neither 1 nor n, a batch-2 image and a crop outside the resized image are refused before
    any launch (no plan is built); the handle then runs a variations forward that equals a fresh handle's."""
    import ctypes as C
    import i2it
    import weights as W
    cfg, dt, n = W.TINY, torch.bfloat16, 3
    op = _operands(n, 64, 64, dt, cfg["cross_dim"], 1, False, seed=7)
    e = _engine("pix2pix", dt, tiny_sd, cfg)
    with pytest.raises(RuntimeError, match="n must be >= 1"):
        e.forward_variations(op["x"], op["text"], op["eps"][:0])
    text2 = torch.cat([op["text"], op["text"]])
    with pytest.raises(ValueError, match="text_emb"):
        e.forward_variations(op["x"], text2, op["eps"])
    out = torch.empty(n, 3, 64, 64, device="cuda", dtype=dt)
    ptr = lambda t: C.c_void_p(t.data_ptr())
    d = i2it.ForwardDesc(batch=n, H=64, W=64, direction=i2it.A2B, shared_input=1, x=ptr(op["x"]), text_emb=ptr(text2),
                         text_batch=2, eps=ptr(op["eps"]), r=1.0, out=ptr(out))
    rc = e.lib.i2it_forward(e._h, C.byref(d), None)
    assert rc != 0 and b"text_batch" in e.lib.i2it_last_error(e._h)
    with pytest.raises(ValueError, match="one image"):
        e.forward_variations(_rep(op["x"], 2), op["text"], op["eps"])
    frame = torch.randint(0, 256, (1, 100, 150, 3), dtype=torch.uint8).cuda()
    with pytest.raises(ValueError, match="one image"):
        e.forward_u8_variations(_rep(frame, 2), i2it.IN_UNIT, op["text"], op["eps"])
    with pytest.raises(RuntimeError, match="crop window"):
        e.forward_u8_variations(frame, i2it.IN_UNIT, op["text"], op["eps"], resize=(64, 96), crop=(8, 40, 64, 64))
    assert e.memory_stats()["plan_builds"] == 0
    got = e.forward_variations(op["x"], op["text"], op["eps"]).cpu()
    fresh = _engine("pix2pix", dt, tiny_sd, cfg)
    assert torch.equal(got, fresh.forward(_rep(op["x"], n), op["text"], op["eps"]).cpu())


def _model(twin):
    import weights as W
    from _host import HashTokenizer
    from pix2pix_turbo import Pix2Pix_Turbo
    from test_gpu_clip import _model as clip_model
    cfg = W.TINY
    clip = clip_model(cfg["cross_dim"], 2, cfg["cross_dim"] // 64, 2 * cfg["cross_dim"])
    m = Pix2Pix_Turbo(cfg=cfg, text_stack=(HashTokenizer(), clip), perturb_norm=True, twin=twin)
    m.set_eval()
    return m.half()


def test_wrappers_equal_forward_on_repeated_image():
    """Pix2Pix_Turbo.variations / variations_u8 with one prompt per variation equal forward / forward_u8 on the repeated image
    (deterministic, and stochastic TwinConv at r = 0.4); repeated calls replay one plan."""
    n = 3
    prompts = ["a house by a lake", "a red car", "a cat on a sofa"]
    g = torch.Generator().manual_seed(8)
    c_t = (torch.rand(1, 3, 64, 64, generator=g) < 0.1).half().cuda()
    eps = torch.randn(n, 4, 8, 8, generator=g).half().cuda()
    noise = torch.randn(n, 4, 8, 8, generator=g).half().cuda()
    frame = torch.randint(0, 256, (1, 64, 64, 3), generator=g, dtype=torch.uint8)

    m = _model(twin=False)
    v = m.variations(c_t, prompts, eps=eps)
    assert torch.equal(v, m(_rep(c_t, n), prompts, eps=eps))
    assert torch.equal(m.variations_u8(frame, prompts, eps=eps, sketch=True),
                       m.forward_u8(_rep(frame, n), prompts, eps=eps, sketch=True))
    builds = m._get_engine().memory_stats()["plan_builds"]
    assert torch.equal(m.variations(c_t, prompts, eps=eps), v)
    assert m._get_engine().memory_stats()["plan_builds"] == builds
    with pytest.raises(ValueError, match="differs"):
        m.variations(c_t, prompts[:2], eps=eps)
    torch.manual_seed(9)
    drawn = m.variations(c_t, "a house", n=2)                 # eps drawn as forward draws it
    torch.manual_seed(9)
    assert drawn.shape[0] == 2 and torch.equal(drawn, m(_rep(c_t, 2), "a house"))

    t = _model(twin=True)
    sv = t.variations(c_t, prompts, deterministic=False, r=0.4, noise_map=noise, eps=eps)
    assert torch.equal(sv, t(_rep(c_t, n), prompts, deterministic=False, r=0.4, noise_map=noise, eps=eps))
    su = t.variations_u8(frame, prompts, deterministic=False, r=0.4, noise_map=noise, eps=eps)
    assert torch.equal(su, t.forward_u8(_rep(frame, n), prompts, deterministic=False, r=0.4, noise_map=noise, eps=eps))
    builds = t._get_engine().memory_stats()["plan_builds"]
    assert torch.equal(t.variations(c_t, prompts, deterministic=False, r=0.4, noise_map=noise, eps=eps), sv)
    assert t._get_engine().memory_stats()["plan_builds"] == builds
