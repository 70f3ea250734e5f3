"""-m gpu: refolding the weights in place (i2it_refold_weights).  A refold writes every prepared weight bit-identically to a
fresh i2it_finalize_weights with the same arguments, keeps the forward plans and their CUDA graphs, allocates nothing, waits
for the work in flight, rebuilds only what changed, and refuses, before any launch, what it cannot do in place."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DTS = [torch.float16, torch.bfloat16]
DT_IDS = ["fp16", "bf16"]


def _engine(dt, sd, fold=(1.0, 1.0, 1.0, -1.0), **kw):
    import i2it
    import weights as W
    e = i2it.Engine(dt, i2it.PIX2PIX, cfg=W.TINY, **kw)
    e.load_state_dict(sd)
    e.set_adapter_scale("default", 1.0)
    e.set_adapter_scale("vae_skip", 2.0)
    if fold is not None:
        e.finalize(*fold)
    return e


def _ops(dt, B=1, seed=0):
    import weights as W
    g = torch.Generator().manual_seed(seed)
    return dict(x=(torch.rand(B, 3, 64, 64, generator=g) * 2 - 1).to(dt).cuda(),
                text=torch.randn(1, 77, W.TINY["cross_dim"], generator=g).to(dt).cuda(),
                eps=torch.randn(B, 4, 8, 8, generator=g).to(dt).cuda(),
                noise=torch.randn(B, 4, 8, 8, generator=g).to(dt).cuda())


def _fwd(e, op, r, text="inline"):
    lat = torch.empty_like(op["eps"])
    out = e.forward(op["x"], op["text"] if text == "inline" else None, op["eps"], op["noise"], r, out_latent=lat)
    return out, lat


def _prepared(e):
    return {k: e.read_prepared(k) for k in e.prepared_keys()}


def _same_prepared(a, b):
    assert sorted(a) == sorted(b)
    for k in a:
        (wa, ba), (wb, bb) = a[k], b[k]
        assert torch.equal(wa.view(torch.int16), wb.view(torch.int16)), k
        assert (ba is None) == (bb is None) and (ba is None or torch.equal(ba.view(torch.int32), bb.view(torch.int32))), k


@pytest.fixture(scope="module")
def twin_sd():
    import weights as W
    return W.make_state_dict("pix2pix", W.TINY, seed=0, twin=True, perturb_norm=True)


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("r2", [0.0, 0.4, 1.0])
def test_twin_refold_bit_identical(dt, r2, twin_sd):
    """A TwinConv handle folded at r = 0.7 and refolded to r2 equals a handle finalized at r2: images, latents and every
    prepared weight, byte for byte."""
    op = _ops(dt)
    e = _engine(dt, twin_sd, (0.7, 0.7, 0.7, 0.7))
    _fwd(e, op, 0.7)
    e.refold(r2, r2, r2, r2)
    got, lat = _fwd(e, op, r2)
    fresh = _engine(dt, twin_sd, (r2, r2, r2, r2))
    ref, ref_lat = _fwd(fresh, op, r2)
    torch.cuda.synchronize()
    assert torch.equal(got.cpu(), ref.cpu()) and torch.equal(lat.cpu(), ref_lat.cpu())
    _same_prepared(_prepared(e), _prepared(fresh))


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
def test_scalars_refold_separately(dt, tiny_sd):
    """A handle without TwinConv: lora_weight_unet, lora_weight_vae and skip_gamma changed one at a time."""
    op = _ops(dt)
    e = _engine(dt, tiny_sd)
    _fwd(e, op, 1.0)
    for fold in [(0.3, 1.0, 1.0, -1.0), (0.3, 0.6, 1.0, -1.0), (0.3, 0.6, 0.5, -1.0)]:
        e.refold(*fold)
        got, lat = _fwd(e, op, 1.0)
        fresh = _engine(dt, tiny_sd, fold)
        ref, ref_lat = _fwd(fresh, op, 1.0)
        torch.cuda.synchronize()
        assert torch.equal(got.cpu(), ref.cpu()) and torch.equal(lat.cpu(), ref_lat.cpu()), fold
        _same_prepared(_prepared(e), _prepared(fresh))
        fresh.close()


def _resident_calls(dt):
    """Five resident plans: batch 1, batch 2, a resize geometry, a variations plan and a ragged plan.  Every call writes into
    the same output tensors, so its graph replays."""
    import i2it
    g = torch.Generator().manual_seed(3)
    b1, b2 = _ops(dt, 1, seed=1), _ops(dt, 2, seed=2)
    u8 = torch.randint(0, 256, (1, 100, 150, 3), generator=g, dtype=torch.uint8).cuda()
    geom = dict(resize=(64, 96), crop=(0, 16, 64, 64), out_size=(100, 150))
    imgs = [torch.randint(0, 256, (80, 60, 3), generator=g, dtype=torch.uint8).cuda(),
            torch.randint(0, 256, (64, 64, 3), generator=g, dtype=torch.uint8).cuda()]
    veps = torch.randn(3, 4, 8, 8, generator=g).to(dt).cuda()
    o1, o2 = torch.empty_like(b1["x"]), torch.empty_like(b2["x"])
    ou8 = torch.empty(1, 100, 150, 3, dtype=torch.uint8, device="cuda")
    ov = torch.empty(3, 3, 64, 64, dtype=dt, device="cuda")
    text = b1["text"]
    return {
        "b1": lambda e: e.forward(b1["x"], text, b1["eps"], out=o1).clone(),
        "b2": lambda e: e.forward(b2["x"], text, b2["eps"], out=o2).clone(),
        "resize": lambda e: e.forward_u8(u8, i2it.IN_UNIT, text, b1["eps"], out=ou8, **geom).clone(),
        "variations": lambda e: e.forward_variations(b1["x"], text, veps, out=ov).clone(),
        "ragged": lambda e: torch.cat([t.flatten() for t in e.forward_u8_ragged(
            imgs, i2it.IN_UNIT, text, b2["eps"], geometries=[dict(resize=(64, 64)), {}])]),
    }


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
def test_plans_and_graphs_survive(dt, tiny_sd):
    calls = _resident_calls(dt)
    e = _engine(dt, tiny_sd)
    for c in calls.values():
        c(e)
    torch.cuda.synchronize()
    builds, captures = e.memory_stats()["plan_builds"], e.graph_captures()
    folds = [(0.5, 0.8, 0.7, -1.0), (1.0, 1.0, 1.0, -1.0), (0.2, 0.4, 0.9, -1.0)]
    for f in folds:
        e.refold(*f)
        got = {k: c(e) for k, c in calls.items()}
        fresh = _engine(dt, tiny_sd, f)
        for k, c in calls.items():
            assert torch.equal(got[k].cpu(), c(fresh).cpu()), (f, k)
        fresh.close()
    torch.cuda.synchronize()
    assert e.memory_stats()["plan_builds"] == builds and e.graph_captures() == captures
    # no growth: the handle's memory after 20 more refolds is what it was after one
    e.refold(0.6, 0.6, 0.6, -1.0)
    torch.cuda.synchronize()
    stats, free = e.memory_stats(), torch.cuda.mem_get_info()[0]
    for i in range(20):
        e.refold(0.1 + 0.04 * i, 0.9 - 0.03 * i, 0.5 + 0.02 * i, -1.0)
    torch.cuda.synchronize()
    assert e.memory_stats() == stats and torch.cuda.mem_get_info()[0] == free
    assert e.memory_stats()["plan_builds"] == builds and e.graph_captures() == captures


def test_refold_drains_first(tiny_sd):
    """forward, refold, forward with no host synchronisation: the first output has the old weights, the second the new."""
    dt = torch.bfloat16
    op = _ops(dt, 2)
    e = _engine(dt, tiny_sd)
    o1, o2 = torch.empty_like(op["x"]), torch.empty_like(op["x"])
    e.forward(op["x"], op["text"], op["eps"], out=o1)          # builds and captures the plan
    torch.cuda.synchronize()
    e.forward(op["x"], op["text"], op["eps"], out=o1)
    e.refold(0.3, 0.5, 0.7, -1.0)
    e.forward(op["x"], op["text"], op["eps"], out=o2)
    torch.cuda.synchronize()
    old = _engine(dt, tiny_sd).forward(op["x"], op["text"], op["eps"])
    new = _engine(dt, tiny_sd, (0.3, 0.5, 0.7, -1.0)).forward(op["x"], op["text"], op["eps"])
    torch.cuda.synchronize()
    assert torch.equal(o1.cpu(), old.cpu()) and torch.equal(o2.cpu(), new.cpu())
    assert not torch.equal(o1.cpu(), o2.cpu())


def test_only_what_changed(twin_sd):
    """Refolding to the same scalars launches nothing; changing r refolds the layers with LoRA, the skip convs and the
    TwinConv, and leaves the CLIP text tower (no LoRA, no scalar) alone, in one preparation launch."""
    import weights as W
    from test_gpu_clip import _model as clip_model
    dt = torch.bfloat16
    cross = W.TINY["cross_dim"]
    clip = clip_model(cross, 2, cross // 64, 2 * cross)
    sd = dict(twin_sd)
    sd.update({"text_encoder." + k: v for k, v in clip.state_dict().items()})
    e = _engine(dt, sd, (0.5, 0.5, 0.5, 0.5), text_heads=cross // 64)
    tokens = torch.randint(0, 49408, (1, 77), generator=torch.Generator().manual_seed(4))
    emb = e.encode_text(tokens, cross)
    op = _ops(dt)
    _fwd(e, op, 0.5)
    torch.cuda.synchronize()
    n = e.prep_launch_count()
    e.refold(0.5, 0.5, 0.5, 0.5)
    assert e.prep_launch_count() == n
    info = e._debug_refold_info()
    assert info["recipes"] == [] and info["jobs"] == 0 and info["bytes"] == 0
    e.refold(0.8, 0.8, 0.8, 0.8)
    info = e._debug_refold_info()
    assert e.prep_launch_count() == n + 1                       # no time-embedding GEMV: the time MLPs carry no LoRA
    touched = set(info["recipes"])
    assert touched and not any(k.startswith("text_encoder.") for k in touched)
    text_keys = [k for k in e.prepared_keys() if k.startswith("text_encoder.")]
    assert text_keys
    assert "unet.conv_in.conv_in_pretrained|twin" in touched
    assert any(".skip_conv_" in k for k in touched)
    assert info["jobs"] > 0 and info["bytes"] > 0
    assert torch.equal(e.encode_text(tokens, cross).cpu(), emb.cpu())
    got, _ = _fwd(e, op, 0.8)
    ref, _ = _fwd(_engine(dt, sd, (0.8, 0.8, 0.8, 0.8), text_heads=cross // 64), op, 0.8)
    torch.cuda.synchronize()
    assert torch.equal(got.cpu(), ref.cpu())


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
def test_checkpoint_in_place(dt, tiny_sd):
    """A second seeded checkpoint with the same keys and shapes, VAE norms included, registered over the live handle and
    refolded: the outputs equal a fresh handle's and no plan is built.  A shape change, a TwinConv switch, or a handle that was
    never finalized is refused before any launch, and the handle keeps its weights."""
    import weights as W
    sd2 = W.make_state_dict("pix2pix", W.TINY, seed=1, perturb_norm=True)
    op1, op2 = _ops(dt, 1), _ops(dt, 2, seed=5)
    e = _engine(dt, tiny_sd)
    _fwd(e, op1, 1.0)
    _fwd(e, op2, 1.0)
    torch.cuda.synchronize()
    builds = e.memory_stats()["plan_builds"]
    e.load_state_dict(sd2)
    e.refold(1.0, 1.0, 1.0, -1.0)
    fresh = _engine(dt, sd2)
    for op in (op1, op2):
        got, lat = _fwd(e, op, 1.0)
        ref, ref_lat = _fwd(fresh, op, 1.0)
        torch.cuda.synchronize()
        assert torch.equal(got.cpu(), ref.cpu()) and torch.equal(lat.cpu(), ref_lat.cpu())
    assert e.memory_stats()["plan_builds"] == builds
    _same_prepared(_prepared(e), _prepared(fresh))
    before = _fwd(e, op1, 1.0)[0].cpu()
    n = e.prep_launch_count()
    with pytest.raises(RuntimeError, match="twin_r >= 0"):
        e.refold(1.0, 1.0, 1.0, 0.5)
    lora = next(k for k in sd2 if ".lora_A." in k)
    e.load_state_dict({lora: torch.zeros(sd2[lora].shape[0] + 1, *sd2[lora].shape[1:])})
    with pytest.raises(RuntimeError, match="changed shape"):
        e.refold(0.5, 1.0, 1.0, -1.0)
    assert e.prep_launch_count() == n
    torch.cuda.synchronize()
    assert torch.equal(_fwd(e, op1, 1.0)[0].cpu(), before)
    never = _engine(dt, tiny_sd, fold=None)
    with pytest.raises(RuntimeError, match="never folded"):
        never.refold(1.0, 1.0, 1.0, -1.0)


def test_text_cache_dropped_after_refold(tiny_sd):
    """After a refold text_emb=None raises set_text's error; after set_text the output equals the inline prompt's."""
    import ctypes as C
    import i2it
    dt = torch.bfloat16
    op = _ops(dt)
    e = _engine(dt, tiny_sd)
    e.set_text(op["text"])
    kept, _ = _fwd(e, op, 1.0, text=None)
    with pytest.raises(RuntimeError, match="twin_r >= 0"):
        e.refold(0.4, 0.6, 0.8, 0.5)
    again, _ = _fwd(e, op, 1.0, text=None)                       # a refused refold keeps the prompt's cache
    torch.cuda.synchronize()
    assert torch.equal(again.cpu(), kept.cpu())
    e.refold(0.4, 0.6, 0.8, -1.0)
    with pytest.raises(ValueError, match="set_text"):          # the binding knows the cache is gone
        _fwd(e, op, 1.0, text=None)
    out = torch.empty_like(op["x"])
    ptr = lambda t: t.data_ptr()
    d = i2it.ForwardDesc(batch=1, H=64, W=64, x=ptr(op["x"]), text_batch=1, eps=ptr(op["eps"]), noise_map=ptr(op["noise"]),
                         r=1.0, out=ptr(out))
    rc = e.lib.i2it_forward(e._h, C.byref(d), None)
    assert rc != 0 and "call i2it_set_text first" in e.lib.i2it_last_error(e._h).decode()
    e.set_text(op["text"])
    cached, _ = _fwd(e, op, 1.0, text=None)
    inline, _ = _fwd(e, op, 1.0)
    ref, _ = _fwd(_engine(dt, tiny_sd, (0.4, 0.6, 0.8, -1.0)), op, 1.0)
    torch.cuda.synchronize()
    assert torch.equal(cached.cpu(), inline.cpu()) and torch.equal(inline.cpu(), ref.cpu())


# ---- wrappers ---------------------------------------------------------------------------------------------------------
def test_pix2pix_stochastic_r_refolds():
    """Pix2Pix_Turbo(twin=True), stochastic at r = 0.4, 0.7, 0.4: each output equals a fresh model's, on one engine that
    builds no plan after the first call."""
    from test_gpu_variations import _model
    g = torch.Generator().manual_seed(11)
    c_t = (torch.rand(1, 3, 64, 64, generator=g) < 0.1).half().cuda()
    eps = torch.randn(1, 4, 8, 8, generator=g).half().cuda()
    noise = torch.randn(1, 4, 8, 8, generator=g).half().cuda()
    run = lambda m, r: m(c_t, "a house by a lake", deterministic=False, r=r, noise_map=noise, eps=eps).cpu()
    m = _model(twin=True)
    outs = [run(m, 0.4)]
    eng = m._get_engine()
    builds = eng.memory_stats()["plan_builds"]
    outs += [run(m, 0.7), run(m, 0.4)]
    assert m._get_engine() is eng and eng.memory_stats()["plan_builds"] == builds
    for r, got in zip((0.4, 0.7, 0.4), outs):
        assert torch.equal(got, run(_model(twin=True), r)), r


def _cyclegan_ckpt(seed, rank_unet=8):
    """A checkpoint in train_cyclegan_turbo.py's format from a seeded state dict: the three UNet adapters and every VAE
    tensor of both directions (norms included)."""
    import weights as W
    sd = W.make_state_dict("cyclegan", W.TINY, seed=seed, lora_rank_unet=rank_unet, perturb_norm=True)
    ck = {"rank_unet": rank_unet, "rank_vae": 4, "sd_encoder": {}, "sd_decoder": {}, "sd_other": {}, "sd_vae_enc": {},
          "sd_vae_dec": {}}
    for k, v in sd.items():
        if k.startswith("unet.") and ".lora_" in k:
            for part, a in (("sd_encoder", "default_encoder"), ("sd_decoder", "default_decoder"), ("sd_other", "default_others")):
                if f".{a}." in k:
                    ck[part][k[len("unet."):].replace(f".{a}.", ".")] = v
        elif k.startswith(("vae.", "vae_b2a.")):
            ck["sd_vae_enc" if ".encoder." in k or k.split(".")[1] == "quant_conv" else "sd_vae_dec"][k] = v
    return ck


def _cyclegan():
    import weights as W
    from cyclegan_turbo import CycleGAN_Turbo
    m = CycleGAN_Turbo(cfg=W.TINY, perturb_norm=True, synthetic_caption="driving in the night", synthetic_direction="a2b")
    m.eval()
    return m.half()


def test_cyclegan_checkpoint_in_place():
    g = torch.Generator().manual_seed(12)
    x = (torch.rand(2, 3, 64, 64, generator=g) * 2 - 1).half().cuda()
    eps = torch.randn(2, 4, 8, 8, generator=g).half().cuda()
    run = lambda m: torch.cat([m(x, direction="a2b", eps=eps).flatten(), m(x, direction="b2a", eps=eps).flatten()]).cpu()

    def fresh(ck):
        f = _cyclegan()
        f.load_ckpt_from_state_dict(ck)
        return run(f)

    m = _cyclegan()
    run(m)
    eng = m._get_engine()
    builds = eng.memory_stats()["plan_builds"]
    for seed in (1, 2):
        ck = _cyclegan_ckpt(seed)
        m.load_ckpt_from_state_dict(ck)
        assert torch.equal(run(m), fresh(ck)), seed
        assert m._get_engine() is eng and eng.memory_stats()["plan_builds"] == builds
    # other keys (another UNet LoRA rank): a new engine, still the right outputs
    ck = _cyclegan_ckpt(3, rank_unet=4)
    m.load_ckpt_from_state_dict(ck)
    assert torch.equal(run(m), fresh(ck))
    assert m._get_engine() is not eng


def test_wrappers_see_in_place_edits():
    """The state dict or checkpoint a live model was loaded from, edited in place and loaded again: the model serves the
    edited weights, on the same engine, equal to a fresh model loaded with them."""
    g = torch.Generator().manual_seed(13)
    x = (torch.rand(1, 3, 64, 64, generator=g) * 2 - 1).half().cuda()
    eps = torch.randn(1, 4, 8, 8, generator=g).half().cuda()
    run = lambda m: m(x, direction="a2b", eps=eps).cpu()

    def edit(sd):
        for k in [k for k in sd if ".lora_B." in k][:4] + [k for k in sd if k.endswith("decoder.conv_norm_out.weight")]:
            sd[k].mul_(1.5).add_(0.01)

    m = _cyclegan()
    before = run(m)
    eng = m._get_engine()
    sd = m.unet.state_dict()                 # the model's own tensors
    edit(sd)
    m.unet.load_state_dict(sd)
    got = run(m)
    f = _cyclegan()
    fsd = f.unet.state_dict()
    edit(fsd)
    f.unet.load_state_dict(fsd)
    assert torch.equal(got, run(f)) and not torch.equal(got, before)
    assert m._get_engine() is eng

    ck = _cyclegan_ckpt(1)
    m.load_ckpt_from_state_dict(ck)
    loaded = run(m)
    for part in ("sd_other", "sd_vae_dec"):
        edit(ck[part])                       # the checkpoint dict edited in place, then loaded again
    m.load_ckpt_from_state_dict(ck)
    got = run(m)
    f = _cyclegan()
    f.load_ckpt_from_state_dict(ck)
    assert torch.equal(got, run(f)) and not torch.equal(got, loaded)
    assert m._get_engine() is eng
