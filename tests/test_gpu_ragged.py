"""-m gpu: ragged uint8 batches (i2it_forward with x_u8_list / i2it_op_resize_u8_ragged).  Images of their own sizes share one
forward plan and one graph; each goes through the same LANCZOS passes as a batch-1 resize forward, so every case here compares
BYTE FOR BYTE: the op with PIL, the forward with per-image forward_u8 calls (image i of a batch is computed alone)."""
import ctypes as C

import numpy as np
import pytest
import torch

import pil_resample as R
from test_gpu_plans import _engine
from test_gpu_resample import CASES as RESAMPLE_CASES

pytestmark = pytest.mark.gpu


def _img(H, W, seed):
    return torch.from_numpy(R.stripe_image(H, W, seed=seed)).cuda()


def _pil(img, hw):
    return torch.from_numpy(R.pil_resize(img.cpu().numpy(), hw))


# ------------------------------------------------------------------------------------------ the op
def test_op_equals_pil():
    """One call mixing every size pair of the fixed-pass tests (up, down, width only, height only, both unchanged), 1x1
    inputs and 12 MP -> 512x512 in both orientations: each image equals PIL, in exactly two launches."""
    import i2it
    e = i2it.Engine(torch.float16, i2it.CYCLEGAN)
    pairs = [(s, d) for s, d, _ in RESAMPLE_CASES] + [((1, 1), (1, 1)), ((1, 1), (512, 512)), ((4032, 3024), (512, 512)),
                                                      ((3024, 4032), (512, 512)), ((33, 21), (33, 21))]
    imgs = [_img(*s, seed=i) for i, (s, _) in enumerate(pairs)]
    got = e.op_resize_u8_ragged(imgs, [d for _, d in pairs])
    assert [k["kind"] for k in e.op_launches()] == ["resample_h_ragged", "resample_v_ragged"]
    for i, ((s, d), x, y) in enumerate(zip(pairs, imgs, got)):
        ref = _pil(x, d)
        assert y.shape == ref.shape and int((y.cpu() != ref).sum()) == 0, (i, s, d)


def test_op_rejections():
    import i2it
    e = i2it.Engine(torch.float16, i2it.CYCLEGAN)
    x = _img(40, 50, seed=0)
    with pytest.raises(RuntimeError, match="exceeds max_side"):
        e.op_resize_u8_ragged([x], [(64, 64)], max_side=60)
    with pytest.raises(RuntimeError, match="sizes must be positive"):
        e.op_resize_u8_ragged([x], [(0, 64)])
    out = torch.empty(8, 8, 3, dtype=torch.uint8, device="cuda")
    rc = e.lib.i2it_op_resize_u8_ragged(e._h, (C.c_void_p * 1)(0), (C.c_int * 2)(40, 50), i2it._ptrs([out]),
                                        (C.c_int * 2)(8, 8), 1, 4096, i2it._stream())
    assert rc != 0 and "null image pointer" in e.lib.i2it_last_error(e._h).decode()


# ------------------------------------------------------------------------------------------ the forward
SIZES = [(90, 160), (100, 75), (64, 64), (150, 97), (37, 211)]


def _short_side_crop(H, W, s=64):
    """resized_crop_512 at a network side of s: the short side to s, the long side int(s * long / short), centre crop."""
    rs = (int(s * H / W), s) if W <= H else (s, int(s * W / H))
    return {"resize": rs, "crop": (int(round((rs[0] - s) / 2.0)), int(round((rs[1] - s) / 2.0)), s, s), "out_size": (H, W)}


def _geoms(prep, sizes, net=(64, 64)):
    if prep == "resize":
        return [{"resize": net, "crop": None, "out_size": hw} for hw in sizes]
    return [_short_side_crop(*hw, s=net[0]) for hw in sizes]


FWD = {   # kind, dtype, input mode, text ("inline-1", "inline-n", "cached"), r (None: deterministic), direction, prep
    "cyclegan-fp16-a2b": ("cyclegan", torch.float16, "normalize", "inline-1", None, "a2b", "resize"),
    "cyclegan-fp16-b2a-crop": ("cyclegan", torch.float16, "normalize", "cached", None, "b2a", "crop"),
    "pix2pix-bf16-det": ("pix2pix", torch.bfloat16, "unit", "inline-n", None, "a2b", "crop"),
    "pix2pix-bf16-twin-sketch": ("twin", torch.bfloat16, "sketch", "cached", 0.4, "a2b", "resize"),
}


def _fwd_engine(kind, dt, tiny_sd, tiny_sd_cyc, **kw):
    import weights as W
    cfg = W.TINY
    if kind == "twin":
        sd = W.make_state_dict("pix2pix", cfg, seed=0, twin=True, perturb_norm=True)
    else:
        sd = tiny_sd if kind == "pix2pix" else tiny_sd_cyc
    return _engine("cyclegan" if kind == "cyclegan" else "pix2pix", dt, sd, cfg, **kw), cfg


@pytest.mark.parametrize("case", list(FWD))
def test_forward_equals_per_image(case, tiny_sd, tiny_sd_cyc):
    import i2it
    kind, dt, mode, text, r, d, prep = FWD[case]
    e, cfg = _fwd_engine(kind, dt, tiny_sd, tiny_sd_cyc)
    if r is not None:
        e.finalize(r, r, r, r)
    mode = {"normalize": i2it.IN_NORMALIZE, "unit": i2it.IN_UNIT, "sketch": i2it.IN_SKETCH}[mode]
    direction = i2it.B2A if d == "b2a" else i2it.A2B
    n = len(SIZES)
    g = torch.Generator().manual_seed(5)
    imgs = [_img(*hw, seed=10 + i) for i, hw in enumerate(SIZES)]
    tb = n if text == "inline-n" else 1
    temb = torch.randn(tb, 77, cfg["cross_dim"], generator=g).to(dt).cuda()
    eps = torch.randn(n, 4, 8, 8, generator=g).to(dt).cuda()
    noise = torch.randn(n, 4, 8, 8, generator=g).to(dt).cuda() if r is not None else None
    rr = 1.0 if r is None else r
    if text == "cached":
        e.set_text(temb)
    geoms = _geoms(prep, SIZES)
    lat = torch.empty(n, 4, 8, 8, device="cuda", dtype=dt)
    got = e.forward_u8_ragged(imgs, mode, None if text == "cached" else temb, eps, noise, rr, direction, geometries=geoms,
                              out_latent=lat)
    got = [y.clone() for y in got]
    lat = lat.clone()
    for i, (x, gm) in enumerate(zip(imgs, geoms)):
        ti = temb[i:i + 1] if tb == n else temb
        li = torch.empty(1, 4, 8, 8, device="cuda", dtype=dt)
        ref = e.forward_u8(x[None], mode, None if text == "cached" else ti, eps[i:i + 1].contiguous(),
                           None if noise is None else noise[i:i + 1].contiguous(), rr, direction, out_latent=li, **gm)
        assert got[i].shape == SIZES[i] + (3,)
        assert torch.equal(got[i], ref[0]), (i, SIZES[i])
        assert torch.equal(lat[i], li[0]), i
    assert not torch.equal(got[2], _img(64, 64, seed=12))                # the network did run


def test_uniform_ragged_batch_equals_resize_batch(tiny_sd_cyc):
    """A ragged batch whose images share one size equals the existing fixed-geometry batch forward."""
    import i2it
    import weights as W
    e = _engine("cyclegan", torch.float16, tiny_sd_cyc, W.TINY)
    g = torch.Generator().manual_seed(7)
    text = torch.randn(1, 77, W.TINY["cross_dim"], generator=g).half().cuda()
    eps = torch.randn(3, 4, 8, 8, generator=g).half().cuda()
    batch = torch.from_numpy(R.stripe_image(100, 75, seed=3, b=3)).cuda()
    gm = _short_side_crop(100, 75)
    ref = e.forward_u8(batch, i2it.IN_NORMALIZE, text, eps, **gm)
    got = e.forward_u8_ragged(list(batch), i2it.IN_NORMALIZE, text, eps, geometries=[gm] * 3)
    for i in range(3):
        assert torch.equal(got[i], ref[i]), i


@pytest.mark.parametrize("graph", [True, False])
def test_one_plan_for_any_mix(graph, tiny_sd_cyc):
    """Calls at one batch size and max_side with different size mixes and fresh tensors build one plan and capture one
    graph; the arena is poisoned between calls; every output equals its per-image forward."""
    import i2it
    import weights as W
    e = _engine("cyclegan", torch.float16, tiny_sd_cyc, W.TINY, use_cuda_graph=graph)
    g = torch.Generator().manual_seed(9)
    text = torch.randn(1, 77, W.TINY["cross_dim"], generator=g).half().cuda()
    eps = torch.randn(4, 4, 8, 8, generator=g).half().cuda()
    mixes = [[(90, 160), (100, 75), (64, 64), (150, 97)], [(720, 1280), (1, 1), (333, 517), (64, 100)],
             [(64, 64)] * 4, [(1080, 1920), (37, 211), (480, 640), (100, 75)]]
    runs = []
    for k, sizes in enumerate(mixes):
        imgs = [_img(*hw, seed=100 * k + i) for i, hw in enumerate(sizes)]
        geoms = _geoms("resize" if k % 2 == 0 else "crop", sizes)
        if k:
            e._debug_poison_workspace(0x5A + k)
        got = e.forward_u8_ragged(imgs, i2it.IN_NORMALIZE, text, eps, geometries=geoms)
        torch.cuda.synchronize()
        if k == 0:
            builds, captures = e.memory_stats()["plan_builds"], e.graph_captures()
        assert e.memory_stats()["plan_builds"] == builds and e.graph_captures() == captures, k
        runs.append((imgs, geoms, [y.clone() for y in got]))
        del got
    assert captures == (1 if graph else 0)
    for imgs, geoms, got in runs:
        for i, (x, gm) in enumerate(zip(imgs, geoms)):
            ref = e.forward_u8(x[None], i2it.IN_NORMALIZE, text, eps[i:i + 1].contiguous(), **gm)
            assert torch.equal(got[i], ref[0]), (i, tuple(x.shape))


def test_profile_and_launch_count(tiny_sd_cyc):
    import i2it
    import weights as W
    e = _engine("cyclegan", torch.float16, tiny_sd_cyc, W.TINY)
    g = torch.Generator().manual_seed(2)
    text = torch.randn(1, 77, W.TINY["cross_dim"], generator=g).half().cuda()
    eps = torch.randn(2, 4, 8, 8, generator=g).half().cuda()
    e.forward_u8(_img(64, 64, seed=0)[None].expand(2, -1, -1, -1).contiguous(), i2it.IN_NORMALIZE, text, eps)
    n_plain = e.launch_count(2, 64, 64)
    small = [_img(90, 160, seed=1), _img(100, 75, seed=2)]
    big = [_img(1080, 1920, seed=3), _img(720, 1280, seed=4)]
    byts = []
    for imgs in (small, big):
        e.forward_u8_ragged(imgs, i2it.IN_NORMALIZE, text, eps, geometries=_geoms("resize", [tuple(x.shape[:2]) for x in imgs]))
        assert e.launch_count(2, 64, 64) == n_plain + 4
        prof = e.profile(reps=1)
        rs = [p for p in prof if "ragged" in p["kind"]]
        assert [p["kind"] for p in rs] == ["resample_h_ragged", "resample_v_ragged"] * 2
        assert all(p["bytes"] > 0 and p["ms"] > 0 for p in rs)
        byts.append(sum(p["bytes"] for p in rs))
    assert byts[1] > 10 * byts[0]                     # the algorithmic bytes follow the last call's geometries


def test_ragged_rejections(tiny_sd_cyc):
    """Every rejection comes before any launch, with a message, and leaves the next valid call's output unchanged."""
    import i2it
    import weights as W
    e = _engine("cyclegan", torch.float16, tiny_sd_cyc, W.TINY)
    g = torch.Generator().manual_seed(4)
    text = torch.randn(1, 77, W.TINY["cross_dim"], generator=g).half().cuda()
    eps = torch.randn(2, 4, 8, 8, generator=g).half().cuda()
    imgs = [_img(90, 160, seed=1), _img(150, 97, seed=2)]
    geoms = _geoms("resize", [(90, 160), (150, 97)])
    good = [y.clone() for y in e.forward_u8_ragged(imgs, i2it.IN_NORMALIZE, text, eps, geometries=geoms)]
    bad = [
        (dict(geometries=[{"resize": (0, 64), "crop": (0, 0, 64, 64)}, geoms[1]]), "sizes must be positive"),
        (dict(geometries=[{"resize": (64, 64), "crop": (1, 0, 64, 64)}, geoms[1]]), "crop window"),
        (dict(geometries=geoms, max_side=120), "exceeds max_side"),
        (dict(geometries=geoms, max_side=0), "max_side must be positive"),
        (dict(geometries=[{"resize": (60, 60)}, {"resize": (60, 60)}], eps=torch.zeros(2, 4, 7, 7).half().cuda()),
         "multiples of 8"),
        (dict(geometries=geoms, in_mode=7), "in_mode"),
        (dict(geometries=geoms, text=None), "set_text"),
    ]
    for kw, msg in bad:
        args = dict(in_mode=i2it.IN_NORMALIZE, text=text, eps=eps)
        args.update(kw)
        with pytest.raises((RuntimeError, ValueError), match=msg):
            if args["text"] is None:    # past the binding's own check: the engine's
                e._text_batch = 1
            e.forward_u8_ragged(imgs, args.pop("in_mode"), args.pop("text"), args.pop("eps"), **args)
    with pytest.raises(ValueError, match="images but eps"):
        e.forward_u8_ragged(imgs[:1], i2it.IN_NORMALIZE, text, eps, geometries=geoms[:1])
    # a null image pointer, past the binding
    descs = i2it._ragged_descs(geoms, [(90, 160), (150, 97)])[2]
    outs = [torch.empty_like(y) for y in good]
    d = i2it.ForwardDesc(batch=2, H=64, W=64, direction=i2it.A2B, x_u8_list=(C.c_void_p * 2)(imgs[0].data_ptr(), 0),
                         in_mode=i2it.IN_NORMALIZE, geometry=descs, max_side=4096, text_emb=i2it._ptr(text), text_batch=1,
                         eps=i2it._ptr(eps), r=1.0, out_u8_list=i2it._ptrs(outs))
    rc = e.lib.i2it_forward(e._h, C.byref(d), i2it._stream())
    assert rc != 0 and "null image pointer" in e.lib.i2it_last_error(e._h).decode()
    again = e.forward_u8_ragged(imgs, i2it.IN_NORMALIZE, text, eps, geometries=geoms)
    for a, b in zip(good, again):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------ the wrappers
def test_cyclegan_wrapper_batch_at_sd_turbo_width():
    """CycleGAN-Turbo fp16 at SD-Turbo width: uploads of five sizes with resize_512x512 and resized_crop_512, each output
    back at its input size, equal to per-image forward_u8 calls; a second mix replays the same graph."""
    from _host import image_prep_geometry
    from cyclegan_turbo import CycleGAN_Turbo
    m = CycleGAN_Turbo(synthetic_caption="driving in the night", synthetic_direction="a2b")
    m.eval(); m.half()
    g = torch.Generator().manual_seed(6)
    sizes = [(720, 1280), (333, 517), (1080, 1920), (512, 512), (1000, 600)]
    imgs = [_img(*hw, seed=20 + i) for i, hw in enumerate(sizes)]
    eps = torch.randn(len(sizes), 4, 64, 64, generator=g).half().cuda()
    for prep in ("resize_512x512", "resized_crop_512"):
        got = [y.clone() for y in m.forward_u8_batch(imgs, eps=eps, image_prep=prep)]
        for i, (x, hw) in enumerate(zip(imgs, sizes)):
            rs, crop = image_prep_geometry(prep, *hw)
            ref = m.forward_u8(x[None], eps=eps[i:i + 1], resize=rs, crop=crop, out_size=hw)
            assert got[i].shape == hw + (3,) and torch.equal(got[i], ref[0]), (prep, hw)
    eng = m._get_engine()
    m.forward_u8_batch(imgs[::-1], eps=eps)
    captures = eng.graph_captures()
    m.forward_u8_batch([_img(*hw, seed=i) for i, hw in enumerate([(480, 640), (64, 64), (2000, 1500), (600, 800), (10, 10)])],
                       eps=eps)
    assert eng.graph_captures() == captures
    with pytest.raises(ValueError, match="random crops"):
        m.forward_u8_batch(imgs, image_prep="randomcrop_hflip")


def test_pix2pix_wrapper_batch_stochastic():
    import weights as W
    from pix2pix_turbo import Pix2Pix_Turbo
    m = Pix2Pix_Turbo(cfg=W.TINY, twin=True)
    m.set_eval(); m.to(torch.bfloat16)
    g = torch.Generator().manual_seed(8)
    sizes = [(90, 160), (100, 75), (64, 64)]
    imgs = [_img(*hw, seed=30 + i) for i, hw in enumerate(sizes)]
    eps = torch.randn(3, 4, 8, 12, generator=g).to(torch.bfloat16).cuda()
    noise = torch.randn(3, 4, 8, 12, generator=g).to(torch.bfloat16).cuda()
    got = [y.clone() for y in m.forward_u8_batch(imgs, "a cat", deterministic=False, r=0.4, noise_map=noise, resize=(64, 96),
                                                 sketch=True, eps=eps)]
    for i, (x, hw) in enumerate(zip(imgs, sizes)):
        ref = m.forward_u8(x[None], "a cat", deterministic=False, r=0.4, noise_map=noise[i:i + 1], eps=eps[i:i + 1],
                           sketch=True, resize=(64, 96), out_size=hw)
        assert got[i].shape == hw + (3,) and torch.equal(got[i], ref[0]), hw
