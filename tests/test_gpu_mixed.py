"""-m gpu: CycleGAN batches that mix both directions in one forward (i2it_forward with directions / i2it_op_conv2d_sel).
Each image takes its own direction's prepared VAE weights in the same accumulation order, so every comparison with a
single-direction forward is BYTE FOR BYTE; the selecting op is also checked against float64."""
import ctypes as C

import pytest
import torch

import kref as K
from test_gpu_plans import _engine

pytestmark = pytest.mark.gpu

MIX = [0, 1, 1, 0, 0, 0, 1, 0]                     # a, b, b, a, a, a, b, a
OTHER_MIXES = [[1, 0, 0, 1, 1, 1, 0, 1], [1] * 4 + [0] * 4, [0, 1] * 4]


def _inputs(B, H, W, cross, dt, seed=0, tb=1):
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(B, 3, H, W, generator=g) * 2 - 1).to(dt).cuda()
    eps = torch.randn(B, 4, H // 8, W // 8, generator=g).to(dt).cuda()
    text = torch.randn(tb, 77, cross, generator=g).to(dt).cuda()
    return x, eps, text


def _single(e, x, text, eps, d):
    import i2it
    B, _, H, W = x.shape
    lat = torch.empty(B, 4, H // 8, W // 8, device="cuda", dtype=x.dtype)
    out = e.forward(x, text, eps, direction=i2it.B2A if d else i2it.A2B, out_latent=lat)
    return out.clone(), lat.clone()


def _check_rows(out, lat, refs, dirs):
    for i, d in enumerate(dirs):
        assert torch.equal(out[i], refs[d][0][i]), ("image", i, d)
        assert torch.equal(lat[i], refs[d][1][i]), ("latent", i, d)


def _mixed_vs_single(e, cfg, H, W, dt):
    B = len(MIX)
    x, eps, text = _inputs(B, H, W, cfg["cross_dim"], dt)
    refs = {d: _single(e, x, text, eps, d) for d in (0, 1)}
    out = torch.empty_like(x)
    lat = torch.empty(B, 4, H // 8, W // 8, device="cuda", dtype=dt)
    e.forward_mixed(x, text, eps, MIX, out=out, out_latent=lat)
    _check_rows(out, lat, refs, MIX)
    # one plan and one graph serve every mix: the same IO, other directions
    s0, g0 = e.memory_stats()["plan_builds"], e.graph_captures()
    for dirs in OTHER_MIXES + [[0] * B, [1] * B]:
        e.forward_mixed(x, text, eps, dirs, out=out, out_latent=lat)
        _check_rows(out, lat, refs, dirs)
    assert e.memory_stats()["plan_builds"] == s0 and e.graph_captures() == g0
    return x, eps, text, refs


@pytest.fixture(scope="module")
def tiny(tiny_sd_cyc):
    import weights as W
    return _engine("cyclegan", torch.float16, tiny_sd_cyc, W.TINY), W.TINY


def test_tiny_bytes_one_plan_one_graph(tiny):
    e, cfg = tiny
    _mixed_vs_single(e, cfg, 128, 128, torch.float16)


def test_sd_turbo_512_bytes_one_plan_one_graph():
    import weights as W
    sd = W.make_state_dict("cyclegan", W.SD_TURBO, seed=0, perturb_norm=True)
    e = _engine("cyclegan", torch.float16, sd, W.SD_TURBO)
    del sd
    _mixed_vs_single(e, W.SD_TURBO, 512, 512, torch.float16)
    e.close()


def test_launch_list_matches_single_direction(tiny):
    """Same launch count and tile geometry: a tapgemm launch differs only by its ' sel' tag, a GroupNorm apply by its kind."""
    e, cfg = tiny
    x, eps, text = _inputs(8, 128, 128, cfg["cross_dim"], torch.float16)
    e.forward(x, text, eps, direction=0)
    single = e.profile(1)
    e.forward_mixed(x, text, eps, MIX)
    mixed = e.profile(1)
    assert len(mixed) == len(single)
    nsel = 0
    for a, b in zip(single, mixed):
        if b["kind"] == "gn_apply_sel":
            assert a["kind"] == "gn_apply"
            nsel += 1
            continue
        assert a["kind"] == b["kind"]
        if b["shape"].endswith(" sel"):
            assert b["shape"][:-4] == a["shape"]
            nsel += 1
        else:
            assert b["shape"] == a["shape"]
    assert nsel > 40


def test_text_per_image_and_cached(tiny):
    e, cfg = tiny
    B = len(MIX)
    x, eps, text = _inputs(B, 128, 128, cfg["cross_dim"], torch.float16, seed=3, tb=B)
    refs = {d: _single(e, x, text, eps, d) for d in (0, 1)}
    lat = torch.empty(B, 4, 16, 16, device="cuda", dtype=torch.float16)
    out = e.forward_mixed(x, text, eps, MIX, out_latent=lat)
    _check_rows(out, lat, refs, MIX)
    e.set_text(text[:1].contiguous())
    refs = {d: _single(e, x, None, eps, d) for d in (0, 1)}
    out = e.forward_mixed(x, None, eps, MIX, out_latent=lat)
    _check_rows(out, lat, refs, MIX)


def test_ragged_uploads(tiny):
    """Uploads of five sizes, both directions, resize to the network size and back: output i equals the batch-1 forward_u8
    of upload i in its direction."""
    import i2it
    e, cfg = tiny
    sizes = [(90, 160), (100, 75), (128, 128), (150, 97), (37, 211)]
    dirs = [1, 0, 1, 1, 0]
    g = torch.Generator().manual_seed(7)
    imgs = [torch.randint(0, 256, hw + (3,), generator=g, dtype=torch.uint8).cuda() for hw in sizes]
    eps = torch.randn(len(sizes), 4, 16, 16, generator=g).half().cuda()
    text = torch.randn(1, 77, cfg["cross_dim"], generator=g).half().cuda()
    geoms = [{"resize": (128, 128), "crop": None, "out_size": hw} for hw in sizes]
    lat_buf = torch.empty(len(sizes), 4, 16, 16, device="cuda", dtype=torch.float16)
    got = [y.clone() for y in e.forward_u8_ragged_mixed(imgs, i2it.IN_NORMALIZE, text, eps, dirs, geometries=geoms,
                                                         out_latent=lat_buf)]
    lat = lat_buf.clone()
    for i, (x, gm, d) in enumerate(zip(imgs, geoms, dirs)):
        li = torch.empty(1, 4, 16, 16, device="cuda", dtype=torch.float16)
        ref = e.forward_u8(x[None], i2it.IN_NORMALIZE, text, eps[i:i + 1].contiguous(), direction=d, out_latent=li, **gm)
        assert torch.equal(got[i], ref[0]), (i, sizes[i], d)
        assert torch.equal(lat[i], li[0]), (i, d)
    s0, g0 = e.memory_stats()["plan_builds"], e.graph_captures()
    # other sizes, other directions, the same eps / latent buffers (the graph's IO): no plan, no capture
    e.forward_u8_ragged_mixed(imgs[::-1], i2it.IN_NORMALIZE, text, eps, dirs[::-1], geometries=geoms[::-1], out_latent=lat_buf)
    assert e.memory_stats()["plan_builds"] == s0 and e.graph_captures() == g0


def _refused(e, fn, msg):
    s0, g0 = e.memory_stats()["plan_builds"], e.graph_captures()
    torch.cuda.synchronize()
    rc = fn()
    assert rc != 0
    err = e.lib.i2it_last_error(e._h).decode()
    assert msg in err, err
    assert e.memory_stats()["plan_builds"] == s0 and e.graph_captures() == g0


def test_mixed_refusals(tiny, tiny_sd):
    import i2it
    import weights as W
    e, cfg = tiny
    st = i2it._stream()

    def call(eng, H, W_, dirs):
        d = i2it.ForwardDesc(batch=len(dirs), H=H, W=W_, text_batch=1, directions=(C.c_int * len(dirs))(*dirs))
        return lambda: eng.lib.i2it_forward(eng._h, C.byref(d), st)
    _refused(e, call(e, 720, 1280, [0, 1]), "multiple of 128")
    _refused(e, call(e, 32, 256, [0, 1]), "tile box")
    _refused(e, call(e, 128, 128, [0, 2]), "direction 2 of image 1")
    # without a direction array the request has one direction, A2B or B2A
    one = i2it.ForwardDesc(batch=2, H=128, W=128, direction=2, text_batch=1)
    _refused(e, lambda: e.lib.i2it_forward(e._h, C.byref(one), st), "direction 2 is neither I2IT_A2B (0) nor I2IT_B2A (1)")
    with pytest.raises(ValueError, match="multiple of 128"):
        x, eps, text = _inputs(2, 720, 1280, cfg["cross_dim"], torch.float16)
        e.forward_mixed(x, text, eps, [0, 1])
    p = _engine("pix2pix", torch.bfloat16, tiny_sd, W.TINY)
    _refused(p, call(p, 128, 128, [0, 1]), "pix2pix handle")
    p.close()


REFUSED_REQUESTS = {   # combination -> what the refusal says
    "directions with x_u8": "directions with the uint8 x_u8",
    "directions with shared_input": "directions with shared_input",
    "x_u8_list with shared_input": "shared_input (variations of one image) with a ragged x_u8_list",
    "geometry with x": "a resize geometry needs a uint8 input",
    "directions with noise_map": "directions with a noise_map",
}


@pytest.mark.parametrize("case", list(REFUSED_REQUESTS))
def test_refused_request_shapes(tiny, case):
    """A combination of i2it_forward_desc fields outside the accepted requests is refused before any launch, without a plan
    or a graph, although every operand it points at is valid."""
    import i2it
    e, cfg = tiny
    B, H, W = 2, 128, 128
    x, eps, text = _inputs(B, H, W, cfg["cross_dim"], torch.float16)
    out, noise = torch.empty_like(x), torch.randn_like(eps)
    imgs = torch.randint(0, 256, (B, H, W, 3), dtype=torch.uint8).cuda()
    outs_u8 = torch.empty_like(imgs)
    geom = (i2it.ResizeDesc * B)(*[i2it.ResizeDesc(H, W, H, W, 0, 0, H, W)] * B)
    dirs = (C.c_int * B)(0, 1)
    nchw = dict(x=x.data_ptr(), out=out.data_ptr())
    fields = {
        "directions with x_u8": dict(directions=dirs, x_u8=imgs.data_ptr(), in_mode=i2it.IN_NORMALIZE,
                                     out_u8=outs_u8.data_ptr()),
        "directions with shared_input": dict(nchw, directions=dirs, shared_input=1),
        "x_u8_list with shared_input": dict(x_u8_list=i2it._ptrs(list(imgs)), in_mode=i2it.IN_NORMALIZE, geometry=geom,
                                            max_side=4096, out_u8_list=i2it._ptrs(list(outs_u8)), shared_input=1),
        "geometry with x": dict(nchw, geometry=geom),
        "directions with noise_map": dict(nchw, directions=dirs, noise_map=noise.data_ptr(), r=0.5),
    }[case]
    d = i2it.ForwardDesc(batch=B, H=H, W=W, text_emb=text.data_ptr(), text_batch=1, eps=eps.data_ptr(), **fields)
    _refused(e, lambda: e.lib.i2it_forward(e._h, C.byref(d), i2it._stream()), REFUSED_REQUESTS[case])


# ------------------------------------------------------------------------------------------ the selecting op
def _sel_cases():
    return {   # N, H, W, Cin, Cout, keywords of op_conv2d_ex
        "3x3": (4, 16, 16, 64, 128, {}),
        "3x3 stride-2 asym": (4, 32, 32, 64, 128, dict(stride=2, asym_pad=True)),
        "1x1 tokens": (3, 16, 16, 64, 128, dict(tokens=True)),
        "3x3 dual-source": (4, 16, 16, 64, 128, dict(C2=72)),
        "up2x GroupNorm+SiLU, dual-source": (4, 16, 16, 64, 64, dict(up2x=True, gn=True, C2=72)),
        "conv_in im2col (1x1, K=32)": (4, 16, 16, 32, 128, {}),
    }


@pytest.mark.parametrize("case", list(_sel_cases()))
def test_op_conv2d_sel(case):
    """Both weight sets in one launch (directions [0, 1, 1, 0]): each image against float64 with its own weights, and
    byte-equal to the plain op run with those weights."""
    import i2it
    N, H, W, Cin, Cout, kw = _sel_cases()[case]
    kw = dict(kw)
    dt = torch.float16
    e = i2it.Engine(dt, i2it.CYCLEGAN)
    g = torch.Generator().manual_seed(11)
    k = 1 if (kw.get("tokens") or Cin == 32) else 3
    up, stride, asym = kw.get("up2x", False), kw.get("stride", 1), kw.get("asym_pad", False)

    def wt(*shape, fan):            # exactly representable in the handle dtype: the fold's rounding is exact
        return (torch.randn(*shape, generator=g) * fan ** -0.5).to(dt).float().cuda()
    x = torch.randn(N, H, W, Cin, generator=g).to(dt).cuda()
    ws = [wt(Cout, Cin, k, k, fan=Cin * k * k) for _ in range(2)]
    bs = [(torch.randn(Cout, generator=g) * 0.5).cuda() for _ in range(2)]
    C2 = kw.pop("C2", 0)
    Ho, Wo = (2 * H, 2 * W) if up else (H // stride, W // stride)
    x2 = torch.randn(N, Ho, Wo, C2, generator=g).to(dt).cuda() if C2 else None
    w2s = [wt(Cout, C2, 1, 1, fan=C2) for _ in range(2)] if C2 else [None, None]
    gn = None
    if kw.pop("gn", False):
        gn = ((1 + 0.1 * torch.randn(Cout, generator=g)).cuda(), (0.1 * torch.randn(Cout, generator=g)).cuda(), 1e-6, True)
    dirs = [0, 1, 1, 0][:N]
    res = e.op_conv2d_sel(x, ws[0], bs[0], ws[1], bs[1], dirs, x2=x2, w2=w2s[0], w2_alt=w2s[1], gn=gn, **kw)
    assert any(l["shape"].endswith(" sel") for l in e.op_launches())
    got, got_gn = (res[0].clone(), res[1].clone()) if gn is not None else (res.clone(), None)
    for d in (0, 1):
        plain = e.op_conv2d_ex(x, ws[d], bs[d], x2=x2, w2=w2s[d], gn=gn, **kw)
        ref_y, ref_gn = plain if gn is not None else (plain, None)
        for i in [i for i in range(N) if dirs[i] == d]:
            assert torch.equal(got[i], ref_y[i]), (case, i)
            if gn is not None:
                assert torch.equal(got_gn[i], ref_gn[i]), (case, i)
            xi = x[i:i + 1]
            if up:
                wsub = K.subpixel_weights(ws[d], dt)
                ref, mag, Kk = K.subpixel_conv64(xi, wsub, bs[d]), K.subpixel_conv64(xi.abs(), wsub.abs(), bs[d].abs()), 4 * Cin
            else:
                ref = K.conv64(xi, ws[d], bs[d], stride=stride, asym=asym)
                mag, Kk = K.conv64(xi.abs(), ws[d].abs(), bs[d].abs(), stride=stride, asym=asym), Cin * k * k
            if C2:
                ref, mag, Kk = ref + K.conv64(x2[i:i + 1], w2s[d]), mag + K.conv64(x2[i:i + 1].abs(), w2s[d].abs()), Kk + C2
            yi = got[i:i + 1].permute(0, 3, 1, 2).double()
            chk = K.check_gemm(f"{case} image {i}", yi, ref, mag, Kk, dt)
            assert chk, str(chk)
    e.close()


def test_op_conv2d_sel_refuses_a_tile_over_two_images():
    import i2it
    e = i2it.Engine(torch.float16, i2it.CYCLEGAN)
    x = torch.randn(2, 8, 8, 64).half().cuda()
    w = torch.randn(64, 64, 3, 3).cuda() * 0.05
    with pytest.raises(RuntimeError, match="two images"):
        e.op_conv2d_sel(x, w, None, w, None, [0, 1])
    with pytest.raises(ValueError, match="direction 2 of image 1"):
        e.op_conv2d_sel(x, w, None, w, None, [0, 2])
    e.close()
