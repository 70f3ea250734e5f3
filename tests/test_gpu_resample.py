"""-m gpu: the LANCZOS resize passes (csrc/resample.cuh) equal PIL's Image.resize(..., Image.LANCZOS) byte for byte, alone
(i2it_op_resize_u8) and inside the uint8 forward (a geometry of i2it_forward), where they replace the CLIs' host resizes
(src/inference_unpaired.py:40-45,53; src/inference_paired.py:38-41)."""
import numpy as np
import pytest
import torch

import pil_resample as R

pytestmark = pytest.mark.gpu


def _pil(batch, hw):
    """PIL LANCZOS resize of every image of a uint8 [B, H, W, 3] tensor -> [B, H2, W2, 3] CPU tensor."""
    a = batch.cpu().numpy()
    return torch.from_numpy(np.stack([R.pil_resize(a[i], hw) for i in range(a.shape[0])]))


def _stripes(B, H, W, seed):
    return torch.from_numpy(R.stripe_image(H, W, seed=seed, b=B))


@pytest.fixture(scope="module")
def eng():
    import i2it
    return i2it.Engine(torch.float16, i2it.CYCLEGAN)


CASES = [   # (H, W) -> (H2, W2), launches
    ((720, 1280), (512, 512), 2), ((512, 512), (720, 1280), 2), ((1080, 1920), (512, 512), 2), ((512, 512), (1080, 1920), 2),
    ((3024, 4032), (512, 512), 2), ((512, 512), (3024, 4032), 2), ((517, 333), (512, 328), 2), ((300, 200), (256, 256), 2),
    ((64, 96), (286, 286), 2), ((1000, 37), (8, 512), 2), ((3024, 504), (512, 40), 2), ((1, 1), (5, 7), 2),
    ((97, 131), (97, 128), 1), ((40, 50), (61, 50), 1), ((9, 300), (1, 300), 1), ((40, 50), (40, 50), 0),
]


@pytest.mark.parametrize("src,dst,launches", CASES, ids=[f"{a[0]}x{a[1]}-{b[0]}x{b[1]}" for a, b, _ in CASES])
def test_op_resize_equals_pil(eng, src, dst, launches):
    x = _stripes(1, *src, seed=src[1] + dst[0])
    got = eng.op_resize_u8(x.cuda(), *dst)
    kinds = [k["kind"] for k in eng.op_launches()]
    assert len(kinds) == launches and set(kinds) <= {"resample_h", "resample_v"}, kinds
    if launches == 2:
        assert kinds == ["resample_h", "resample_v"]               # PIL's order: horizontal first
    ref = _pil(x, dst)
    assert got.shape == ref.shape and int((got.cpu() != ref).sum()) == 0


def test_op_resize_batch_is_per_image(eng):
    x = _stripes(3, 333, 517, seed=9)
    got = eng.op_resize_u8(x.cuda(), 256, 384).cpu()
    ref = _pil(x, (256, 384))
    for i in range(3):
        assert torch.equal(got[i], ref[i]), i


@pytest.mark.parametrize("src,dst", [((512, 512), (3024, 4032)), ((3024, 4032), (512, 512))])
def test_op_resize_past_2_31_bytes(eng, src, dst):
    """60 images of 12 MP: the big side passes 2^31 bytes.  Images at the start, across the 2^31 offset and at the end equal
    PIL (every image differs, so a wrapped offset reads or writes the wrong one)."""
    B = 60
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.randint(0, 256, (B,) + src + (3,), device="cuda", dtype=torch.uint8, generator=g)
    x[:, :, 3::11] = 255
    x[:, 7::13] = 0
    big = max(src[0] * src[1], dst[0] * dst[1]) * 3
    assert B * big > 2 ** 31
    got = eng.op_resize_u8(x, *dst)
    mid = (2 ** 31) // big
    for i in (0, mid, mid + 1, B - 1):
        ref = _pil(x[i:i + 1], dst)[0]
        assert torch.equal(got[i].cpu(), ref), i
    del x, got
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------ inside the forward
def _engine(kind, cfg, dt, sd):
    import i2it
    e = i2it.Engine(dt, i2it.CYCLEGAN if kind == "cyclegan" else i2it.PIX2PIX, cfg=cfg)
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


def _host_pipeline(e, img, mode, td, ed, resize, crop, out_size):
    """What the CLIs do: PIL resize (+ crop) on the host -> forward_u8 -> PIL resize of the output."""
    x = _pil(img, resize)
    if crop is not None:
        t, l, h, w = crop
        x = x[:, t:t + h, l:l + w].contiguous()
    y = e.forward_u8(x.cuda(), mode, td, ed).cpu()
    return _pil(y, out_size) if out_size is not None and tuple(out_size) != tuple(y.shape[1:3]) else y


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_forward_with_geometry_equals_host_pipeline(dt):
    import i2it
    import weights as W
    cfg = W.TINY
    cyc = _engine("cyclegan", cfg, dt, W.make_state_dict("cyclegan", cfg, seed=0, perturb_norm=True))
    g = torch.Generator().manual_seed(2)
    text = torch.randn(1, 77, cfg["cross_dim"], generator=g).to(dt).cuda()
    eps = torch.randn(2, 4, 8, 8, generator=g).to(dt).cuda()
    cases = [   # (input H, W), resize, crop, out_size
        ((90, 160), (64, 64), None, (90, 160)),                # resize_512x512-style, back to the input size
        ((100, 75), (85, 64), (10, 0, 64, 64), (100, 75)),     # resized_crop-style: short side to 64, centre crop
        ((64, 100), (64, 64), None, (64, 100)),                # width-only passes in and out
        ((64, 90), (64, 90), (0, 13, 64, 64), None),           # a crop of the input itself: no input pass
    ]
    # a forward without a geometry keeps its plan: the plain uint8 launch list is the float one plus the output conversion
    x = torch.rand(2, 3, 64, 64, generator=g).mul(2).sub(1).to(dt).cuda()
    cyc.forward(x, text, eps)
    n_float = cyc.launch_count(2, 64, 64)
    cyc.forward_u8(_stripes(2, 64, 64, seed=1).cuda(), i2it.IN_NORMALIZE, text, eps)
    n_plain = cyc.launch_count(2, 64, 64)
    assert n_plain == n_float + 1
    counts = {}
    for (H, W_), rs, cr, osz in cases:
        img = _stripes(2, H, W_, seed=H * W_)
        ref = _host_pipeline(cyc, img, i2it.IN_NORMALIZE, text, eps, rs, cr, osz)
        got = cyc.forward_u8(img.cuda(), i2it.IN_NORMALIZE, text, eps, resize=rs, crop=cr, out_size=osz)
        again = cyc.forward_u8(img.cuda(), i2it.IN_NORMALIZE, text, eps, resize=rs, crop=cr, out_size=osz)   # graph replay
        torch.cuda.synchronize()
        assert got.shape == ref.shape, (got.shape, ref.shape)
        assert int((got.cpu() != ref).sum()) == 0, (H, W_, rs, cr, osz)
        assert torch.equal(got, again)
        kinds = [p["kind"] for p in cyc.profile(reps=1)]
        passes = sum(k in ("resample_h", "resample_v") for k in kinds)
        expect = (W_ != rs[1]) + (H != rs[0]) + (osz is not None and ((osz[1] != 64) + (osz[0] != 64)))
        assert passes == expect, (kinds, expect)
        assert cyc.launch_count(2, 64, 64) == n_plain + passes
        counts[(H, W_)] = passes
    assert len(set(counts.values())) > 1                       # several geometries on one handle: one plan each
    # the first geometry again after the others: its own plan still gives the host pipeline's bytes
    img = _stripes(2, 90, 160, seed=90 * 160)
    got = cyc.forward_u8(img.cuda(), i2it.IN_NORMALIZE, text, eps, resize=(64, 64), out_size=(90, 160))
    assert torch.equal(got.cpu(), _host_pipeline(cyc, img, i2it.IN_NORMALIZE, text, eps, (64, 64), None, (90, 160)))
    cyc.forward_u8(_stripes(2, 64, 64, seed=1).cuda(), i2it.IN_NORMALIZE, text, eps)
    assert cyc.launch_count(2, 64, 64) == n_plain

    # pix2pix sketch branch: the CLI's resize to multiples of 8, output at the resized size
    from _host import paired_geometry
    p2p = _engine("pix2pix", cfg, dt, W.make_state_dict("pix2pix", cfg, seed=0, perturb_norm=True))
    img = _stripes(2, 70, 93, seed=5)
    rs = paired_geometry(70, 93)
    eps2 = torch.randn(2, 4, rs[0] // 8, rs[1] // 8, generator=g).to(dt).cuda()
    ref = _host_pipeline(p2p, img, i2it.IN_SKETCH, text, eps2, rs, None, None)
    got = p2p.forward_u8(img.cuda(), i2it.IN_SKETCH, text, eps2, resize=rs)
    assert got.shape == (2,) + rs + (3,) and torch.equal(got.cpu(), ref)


def test_bad_geometry_is_refused():
    import i2it
    import weights as W
    cfg = W.TINY
    e = _engine("cyclegan", cfg, torch.float16, W.make_state_dict("cyclegan", cfg, seed=0, perturb_norm=True))
    text = torch.zeros(1, 77, cfg["cross_dim"], dtype=torch.float16, device="cuda")
    img = _stripes(1, 90, 160, seed=0).cuda()
    eps = torch.zeros(1, 4, 8, 8, dtype=torch.float16, device="cuda")
    with pytest.raises(RuntimeError, match="crop window"):
        e.forward_u8(img, i2it.IN_NORMALIZE, text, eps, resize=(64, 100), crop=(1, 0, 64, 64))
    with pytest.raises(RuntimeError, match="sizes must be positive"):
        e.forward_u8(img, i2it.IN_NORMALIZE, text, eps, resize=(0, 100), crop=(0, 0, 64, 64))
    eps_odd = torch.zeros(1, 4, 8, 7, dtype=torch.float16, device="cuda")
    with pytest.raises(RuntimeError, match="multiples of 8"):
        e.forward_u8(img, i2it.IN_NORMALIZE, text, eps_odd, resize=(64, 60))
    with pytest.raises(RuntimeError, match="sizes must be positive"):
        e.op_resize_u8(img, 0, 5)


def test_wrapper_resize_at_sd_turbo_width():
    """CycleGAN fp16 at SD-Turbo width, batch 2: 1280x720 frames -> resize_512x512 -> forward -> back to 1280x720, on device,
    equal to the host pipeline (PIL resizes around the uint8 forward)."""
    from cyclegan_turbo import CycleGAN_Turbo
    from _host import image_prep_geometry
    m = CycleGAN_Turbo(synthetic_caption="driving in the night", synthetic_direction="a2b")
    m.eval(); m.half()
    img = _stripes(2, 720, 1280, seed=11)
    g = torch.Generator().manual_seed(3)
    eps = torch.randn(2, 4, 64, 64, generator=g).half().cuda()
    rs, crop = image_prep_geometry("resize_512x512", 720, 1280)
    got = m.forward_u8(img, eps=eps, resize=rs, crop=crop, out_size=(720, 1280))
    ref = _pil(m.forward_u8(_pil(img, rs), eps=eps), (720, 1280))
    assert got.shape == (2, 720, 1280, 3)
    assert int((got.cpu() != ref).sum()) == 0


@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("size", [(90, 160), (64, 100), (75, 64)], ids=["both-passes", "width-only", "height-only"])
def test_fixed_geometry_on_many_tensors(size, graph, tiny_sd_cyc):
    """A fixed plan's descriptors hold offsets from the caller's pointers, read at every launch: one geometry (resized to the
    64x64 network and back) alternates over more input / output pairs than the plan keeps graphs for, and every output equals
    the host pipeline (a pointer kept from an earlier call, or a stale graph, writes the wrong tensor)."""
    import i2it
    import weights as W
    from test_gpu_plans import _engine as _plans_engine
    e = _plans_engine("cyclegan", torch.float16, tiny_sd_cyc, W.TINY, use_cuda_graph=graph)
    g = torch.Generator().manual_seed(12)
    text = torch.randn(1, 77, W.TINY["cross_dim"], generator=g).half().cuda()
    eps = torch.randn(2, 4, 8, 8, generator=g).half().cuda()
    imgs = [_stripes(2, *size, seed=20 + i) for i in range(10)]
    refs = [_host_pipeline(e, x, i2it.IN_NORMALIZE, text, eps, (64, 64), None, size) for x in imgs]
    xs = [x.cuda() for x in imgs]
    outs = [torch.empty(2, *size, 3, dtype=torch.uint8, device="cuda") for _ in imgs]
    for rnd in range(2):
        for i, (x, o) in enumerate(zip(xs, outs)):
            o.zero_()
            e.forward_u8(x, i2it.IN_NORMALIZE, text, eps, out=o, resize=(64, 64), out_size=size)
            assert torch.equal(o.cpu(), refs[i]), (rnd, i)
        for i, o in enumerate(outs):
            assert torch.equal(o.cpu(), refs[i]), (rnd, i)
