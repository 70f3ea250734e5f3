"""-m gpu: every kernel variant the model builds, called alone through the diagnostic op ABI and held to the per-element
float64 criterion of tests/kref.py.  Each case asserts that the launch list contains the variant it targets (a case that
silently fell back to another path would test nothing) and prints that list, the worst err/bound and the mean-ulp statistic.
The engine reads its I2IT_NO_* switches when it is created, so each variant gets its own engine."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

import kref

pytestmark = pytest.mark.gpu

bf, hf = torch.bfloat16, torch.float16
DTYPES = [pytest.param(bf, id="bf16"), pytest.param(hf, id="fp16")]
_SWITCHES = ("I2IT_NO_TMAOUT", "I2IT_NO_GNEPI", "I2IT_NO_SPLITK")


def engine(dtype, off=()):
    import i2it
    saved = {k: os.environ.pop(k, None) for k in _SWITCHES}
    try:
        for k in off:
            os.environ[k] = "1"
        return i2it.Engine(dtype, use_cuda_graph=False)
    finally:
        for k, v in saved.items():
            os.environ.pop(k, None)
            if v is not None:
                os.environ[k] = v


def mk(*shape, dtype=torch.float32, scale=1.0, shift=0.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, device="cuda", generator=g) * scale + shift).to(dtype)


def weight(Cout, Cin, k, dtype, seed):
    """fp32 weights that are exactly representable in the engine dtype (the fold then rounds nothing)."""
    return mk(Cout, Cin, k, k, scale=1 / math.sqrt(Cin * k * k), seed=seed).to(dtype).float()


def launches(E, name):
    ops = E.op_launches()
    print(f"\n[{name}] launches: " + "; ".join(f"{o['kind']}({o['shape']})" if o["shape"] else o["kind"] for o in ops))
    return ops


def kinds(ops):
    return [o["kind"] for o in ops]


def report(*checks):
    for c in checks:
        print("   ", c)
    for c in checks:
        assert c, str(c)


def nchw(t):
    return t.double().permute(0, 3, 1, 2)


def channel_view(t, C, c0=0):
    """A channel slice [.., c0:c0+C] of a wider buffer: pixel stride > C, as the model's concat buffers hand them out."""
    return t[..., c0:c0 + C]


# ---------------------------------------------------------------------------------------------------------------------
# conv family
# ---------------------------------------------------------------------------------------------------------------------
def conv_case(E, dtype, x, w, b=None, *, stride=1, asym=False, res=None, act=0, x2=None, w2=None, up2x=False, tokens=False, gn=None,
              out=None, gn_out=None, name=""):
    """Runs op_conv2d_ex and checks the conv output element by element; returns (got, gn output, launches)."""
    import i2it
    r = E.op_conv2d_ex(x, w, b, stride=stride, asym_pad=asym, residual=res, act=act, x2=x2, w2=w2, up2x=up2x, tokens=tokens, gn=gn,
                       out=out, gn_out=gn_out)
    got, g = r if gn is not None else (r, None)
    torch.cuda.synchronize()
    ops = launches(E, name)
    Cout, Cin, k, _ = w.shape
    ref = kref.conv64(x, w, b, stride=stride, asym=asym, up2x=up2x)
    mag = kref.conv64(x.abs(), w.abs(), b.abs() if b is not None else None, stride=stride, asym=asym, up2x=up2x)
    K = Cin * k * k
    if x2 is not None:
        ref = ref + kref.conv64(x2, w2)
        mag = mag + kref.conv64(x2.abs(), w2.abs())
        K += x2.shape[3]
    factor = 1.0
    if act == i2it.ACT_GEGLU:
        h, gg = ref.chunk(2, dim=1)
        mh, mg = mag.chunk(2, dim=1)
        ref, mag, factor = h * kref.gelu64(gg), mh * kref.gelu64(gg).abs() + h.abs() * mg, 2.0
    elif act in (i2it.ACT_GELU, i2it.ACT_QUICKGELU):
        ref = kref.gelu64(ref) if act == i2it.ACT_GELU else kref.quick_gelu64(ref)
        factor = 2.0                                               # |GELU'| <= 1.13, |quick-GELU'| <= 1.1
    if res is not None:
        ref, mag = ref + nchw(res), mag + nchw(res).abs()
    if act == i2it.ACT_CLAMP1:
        ref = ref.clamp(-1, 1)
    report(kref.check_gemm(name, nchw(got), ref, mag, K, dtype, factor))
    return got, g, ops


def gn_params(C, seed=20):
    return mk(C, seed=seed) * 0.2 + 1, mk(C, seed=seed + 1) * 0.1


def check_gn(name, E, dtype, y, g, gamma, beta, eps, silu):
    ref, bound = kref.group_norm64(y, gamma, beta, eps, silu, dtype)
    c = kref.check_norm(name, g, ref, bound, dtype)
    report(c)


GN_WIDTHS = [128, 256, 512, 320, 640, 1280]      # gn_red 4 / 8 / 16, and 2 (1280: per_row = 640, the reduce kernel's limit)


@pytest.mark.parametrize("off", [(), ("I2IT_NO_GNEPI",), ("I2IT_NO_TMAOUT",)], ids=["epi", "nognepi", "notmaout"])
@pytest.mark.parametrize("C", GN_WIDTHS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_fused_groupnorm(dtype, C, off):
    """conv3x3 -> GroupNorm(+SiLU) with statistics from the GEMM epilogue; batch 2 of 20x20 maps (400 rows per image: not a
    multiple of 128).  The 320 and 512 cases have |mean| ~ 30 std, where E[x^2] - mean^2 cancels."""
    E = engine(dtype, off)
    N, H, W = 2, 20, 20
    Cin = min(C, 320)
    shift = 30.0 if C in (320, 512) else 0.0
    x = mk(N, H, W, Cin, dtype=dtype, seed=1)
    w = weight(C, Cin, 3, dtype, 2)
    b = mk(C, seed=3) * 0.1 + shift
    gamma, beta = gn_params(C)
    name = f"gn C={C} {dtype} off={off}"
    y, g, ops = conv_case(E, dtype, x, w, b, gn=(gamma, beta, 1e-6, True), name=name)
    fused = not off
    assert (" gn" in ops[0]["shape"]) == fused and ("gn_final_part" in kinds(ops)) == fused
    assert ("gn_stats" in kinds(ops)) == (not fused)
    check_gn(name, E, dtype, y, g, gamma, beta, 1e-6, True)
    # image i of the batch equals its own batch-1 op bit for bit
    y1, g1, _ = conv_case(E, dtype, x[1:].contiguous(), w, b, gn=(gamma, beta, 1e-6, True), name=name + " image 1 alone")
    assert torch.equal(y1, y[1:]) and torch.equal(g1, g[1:])
    if shift:
        # the same input through the statistics pass and through LayerNorm
        g2 = E.op_group_norm(y, gamma, beta, 1e-6, False)
        assert "gn_stats" in kinds(launches(E, name + " gn_stats"))
        ref, bound = kref.group_norm64(y, gamma, beta, 1e-6, False, dtype)
        ln = E.op_layer_norm(y.view(-1, C), gamma, beta)
        lref, lbound = kref.layer_norm64(y.view(-1, C), gamma, beta, 1e-5, dtype)
        report(kref.check_norm(name + " gn_stats", g2, ref, bound, dtype),
               kref.check_norm(name + " layernorm", ln, lref, lbound, dtype))


@pytest.mark.parametrize("dtype", DTYPES)
def test_fused_groupnorm_token_rows(dtype):
    """1x1 projection over token rows (proj_out of a transformer block) -> GroupNorm: per-image 128-row tiles."""
    E = engine(dtype)
    N, T, C = 2, 256, 640
    x = mk(N, 1, T, C, dtype=dtype, seed=1)
    w = weight(C, C, 1, dtype, 2)
    b = mk(C, seed=3) * 0.1
    res = mk(N, 1, T, C, dtype=dtype, seed=4)
    gamma, beta = gn_params(C)
    name = f"gn tokens {dtype}"
    y, g, ops = conv_case(E, dtype, x, w, b, res=res, tokens=True, gn=(gamma, beta, 1e-6, False), name=name)
    assert " gn" in ops[0]["shape"] and "gn_final_part" in kinds(ops)
    check_gn(name, E, dtype, y, g, gamma, beta, 1e-6, False)


SUBPIXEL = [(512, 64, 1, False), (512, 64, 2, True), (512, 128, 1, True), (256, 256, 1, True)]


@pytest.mark.parametrize("C,S,N,skip", SUBPIXEL, ids=[f"{c}@{s}x{s}b{n}{'skip' if k else ''}" for c, s, n, k in SUBPIXEL])
@pytest.mark.parametrize("dtype", DTYPES)
def test_subpixel_upconv(dtype, C, S, N, skip):
    """Decoder up-block conv: nearest-2x upsample + 3x3 conv as four parity launches with pre-summed taps, the skip conv at
    output resolution folded in, GroupNorm statistics shared across the phases."""
    E = engine(dtype)
    x = mk(N, S, S, C, dtype=dtype, seed=1)
    w = mk(C, C, 3, 3, scale=1 / math.sqrt(9 * C), seed=2)                     # fp32: the taps are pre-summed from these
    b = mk(C, seed=3) * 0.1
    x2 = mk(N, 2 * S, 2 * S, 128, dtype=dtype, seed=4) if skip else None
    w2 = weight(C, 128, 1, dtype, 5) if skip else None
    gamma, beta = gn_params(C)
    name = f"up2x {C}@{S} N={N} skip={skip} {dtype}"
    r = E.op_conv2d_ex(x, w, b, x2=x2, w2=w2, up2x=True, gn=(gamma, beta, 1e-6, True))
    got, g = r
    ops = launches(E, name)
    ups = [o for o in ops if o["kind"] == "tapgemm:conv_up2x"]
    assert len(ups) == 4 and all(" gn" in o["shape"] for o in ups) and "gn_final_part" in kinds(ops)
    wsub = kref.subpixel_weights(w, dtype)
    ref = kref.subpixel_conv64(x, wsub, b)
    mag = kref.subpixel_conv64(x.abs(), wsub.abs(), b.abs())
    K = 4 * C
    plain = kref.conv64(x, w, b, up2x=True)
    pmag = kref.conv64(x.abs(), w.abs(), b.abs(), up2x=True)
    if skip:
        ref, mag = ref + kref.conv64(x2, w2), mag + kref.conv64(x2.abs(), w2.abs())
        plain, pmag = plain + kref.conv64(x2, w2), pmag + kref.conv64(x2.abs(), w2.abs())
        K += 128
    tight = kref.check_gemm(name, nchw(got), ref, mag, K, dtype)
    # against interpolate(nearest) then conv2d: plus the rounding of the pre-summed weights
    comp = kref.Check(name + " vs upsample+conv", nchw(got), plain,
                      kref.gemm_bound(plain, pmag, K, dtype) + 2 * kref.unit_roundoff(dtype) * pmag, dtype)
    report(tight, comp)
    check_gn(name, E, dtype, got, g, gamma, beta, 1e-6, True)
    if N > 1:
        r1 = E.op_conv2d_ex(x[1:].contiguous(), w, b, x2=x2[1:].contiguous() if skip else None, w2=w2, up2x=True,
                            gn=(gamma, beta, 1e-6, True))
        assert torch.equal(r1[0], got[1:]) and torch.equal(r1[1], g[1:])


SPLITK = [(2, 8, 8, 1280), (2, 8, 8, 2560), (3, 2, 2, 1280), (3, 3, 4, 1280), (3, 5, 7, 1280)]


@pytest.mark.parametrize("off", [(), ("I2IT_NO_SPLITK",)], ids=["splitk", "nosplitk"])
@pytest.mark.parametrize("N,H,W,Cin", SPLITK, ids=[f"b{n}_{h}x{w}_{c}" for n, h, w, c in SPLITK])
@pytest.mark.parametrize("dtype", DTYPES)
def test_splitk_conv(dtype, N, H, W, Cin, off):
    """The deepest UNet convs (8x8, and the ragged 2x2 / 3x4 / 5x7 maps of 8-but-not-64 resolutions where one m-tile spans
    images) with bias and residual: five fixed K ranges reduced in a fixed order."""
    E = engine(dtype, off)
    x = mk(N, H, W, Cin, dtype=dtype, seed=1)
    w = weight(1280, Cin, 3, dtype, 2)
    b = mk(1280, seed=3) * 0.1
    res = mk(N, H, W, 1280, dtype=dtype, seed=4)
    name = f"splitk b{N} {H}x{W} {Cin}->1280 {dtype} off={off}"
    y, _, ops = conv_case(E, dtype, x, w, b, res=res, name=name)
    assert ("splitk_reduce" in kinds(ops)) == (not off)
    y1, _, _ = conv_case(E, dtype, x[1:2].contiguous(), w, b, res=res[1:2].contiguous(), name=name + " image 1 alone")
    assert torch.equal(y1, y[1:2])


SECOND = [(2, 16, 16, 640, 640, 320), (2, 32, 32, 320, 640, 320), (1, 32, 32, 512, 512, 512), (2, 24, 24, 256, 256, 128)]


@pytest.mark.parametrize("off", [(), ("I2IT_NO_TMAOUT",)], ids=["tmaout", "notmaout"])
@pytest.mark.parametrize("N,H,Cin,Cout,C2", [(n, h, ci, co, c2) for n, h, _, ci, co, c2 in SECOND],
                         ids=[f"b{n}_{h}_{ci}-{co}+{c2}" for n, h, _, ci, co, c2 in SECOND])
@pytest.mark.parametrize("dtype", DTYPES)
def test_second_source(dtype, N, H, Cin, Cout, C2, off):
    """Resnet conv2 + conv_shortcut (Cin != Cout) and decoder skip convs as one more K-slab; input, second source, residual
    and output are channel slices of wider buffers (pixel stride > C)."""
    E = engine(dtype, off)
    xb = mk(N, H, H, Cin + 64, dtype=dtype, seed=1)
    x2b = mk(N, H, H, C2 + 128, dtype=dtype, seed=2)
    x, x2 = channel_view(xb, Cin, 64), channel_view(x2b, C2, 128)
    w = weight(Cout, Cin, 3, dtype, 3)
    w2 = weight(Cout, C2, 1, dtype, 4)
    b = mk(Cout, seed=5) * 0.1
    outb = torch.full((N, H, H, Cout + 128), 7.0, device="cuda", dtype=dtype)
    out = channel_view(outb, Cout, 64)
    name = f"x2 b{N} {H}x{H} {Cin}->{Cout} +{C2} {dtype} off={off}"
    conv_case(E, dtype, x, w, b, x2=x2, w2=w2, out=out, name=name)
    assert torch.all(outb[..., :64] == 7) and torch.all(outb[..., 64 + Cout:] == 7)      # nothing outside the slice


@pytest.mark.parametrize("off", [(), ("I2IT_NO_TMAOUT",)], ids=["tmaout", "notmaout"])
@pytest.mark.parametrize("act", ["gelu", "quick_gelu"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_gelu_epilogues(dtype, act, off):
    """CLIP fc1: 77 * B rows, 1024 -> 4096 with the (quick-)GELU in the epilogue before the one rounding."""
    import i2it
    E = engine(dtype, off)
    B = 2
    x = mk(B, 1, 77, 1024, dtype=dtype, seed=1)
    w = weight(4096, 1024, 1, dtype, 2)
    b = mk(4096, seed=3) * 0.5
    a = i2it.ACT_GELU if act == "gelu" else i2it.ACT_QUICKGELU
    conv_case(E, dtype, x, w, b, act=a, name=f"{act} {dtype} off={off}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_geglu_and_clamp_epilogues(dtype):
    import i2it
    E = engine(dtype)
    conv_case(E, dtype, mk(1, 1, 300, 320, dtype=dtype, seed=1), weight(2560, 320, 1, dtype, 2), mk(2560, seed=3) * 0.1,
              act=i2it.ACT_GEGLU, name=f"geglu {dtype}")
    conv_case(E, dtype, mk(2, 16, 16, 64, dtype=dtype, seed=1), weight(64, 64, 3, dtype, 2), mk(64, seed=3),
              act=i2it.ACT_CLAMP1, name=f"clamp {dtype}")


# The bring-up shapes of tests/gpu_diag.py (ragged, wide, tiny-N, stride-2, many tiles per CTA) under the per-element bound
DIAG = [(1, 1, 128, 64, 64, 1, 1, False), (1, 1, 1000, 320, 320, 1, 1, True), (1, 1, 4096, 320, 2560, 1, 1, False),
        (1, 1, 512, 512, 8, 1, 1, False), (2, 16, 16, 64, 128, 3, 1, False), (1, 32, 32, 320, 320, 3, 1, True),
        (3, 8, 8, 128, 256, 3, 1, False), (2, 32, 32, 8, 128, 3, 1, False), (2, 16, 16, 128, 4, 3, 1, False),
        (2, 32, 32, 64, 64, 3, 2, False), (16, 40, 40, 64, 512, 3, 1, True), (1, 1, 128 * 301 + 17, 256, 512, 1, 1, False),
        (4, 256, 256, 128, 128, 3, -2, False)]          # stride -2: the VAE's asymmetric (0, 1, 0, 1) padding


@pytest.mark.parametrize("off", [(), ("I2IT_NO_TMAOUT",)], ids=["tmaout", "notmaout"])
@pytest.mark.parametrize("case", DIAG, ids=[f"b{n}_{h}x{w}_{ci}-{co}_k{k}s{s}{'r' if r else ''}" for n, h, w, ci, co, k, s, r in DIAG])
@pytest.mark.parametrize("dtype", DTYPES)
def test_conv_shapes(dtype, case, off):
    N, H, W, Cin, Cout, k, s, r = case
    asym, s = s < 0, abs(s)
    E = engine(dtype, off)
    Ho, Wo = -(-H // s), -(-W // s)
    conv_case(E, dtype, mk(N, H, W, Cin, dtype=dtype, seed=1), weight(Cout, Cin, k, dtype, 2), mk(Cout, seed=3), stride=s,
              asym=asym, res=mk(N, Ho, Wo, Cout, dtype=dtype, seed=4) if r else None, name=f"conv {case} {dtype} off={off}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_stride2_on_odd_maps_and_upsample_to(dtype):
    """Latents of 8-but-not-64 images: stride-2 conv of an odd map (padded to even, ceil(H/2) rows) and the decoder's
    interpolate(size=...) back to an explicit size."""
    E = engine(dtype)
    for N, H, W in ((2, 9, 11), (1, 5, 7), (1, 15, 15)):
        x = mk(N, H, W, 128, dtype=dtype, seed=1)
        y, _, ops = conv_case(E, dtype, x, weight(128, 128, 3, dtype, 2), mk(128, seed=3), stride=2,
                              name=f"s2 odd {N}x{H}x{W} {dtype}")
        assert y.shape == (N, (H + 1) // 2, (W + 1) // 2, 128) and "pad_even" in kinds(ops)
        u = E.op_upsample_to(y, H, W)
        ref = F.interpolate(y.permute(0, 3, 1, 2).float(), size=(H, W), mode="nearest").permute(0, 2, 3, 1).to(dtype)
        assert torch.equal(u, ref)


# ---------------------------------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------------------------------
def attn_case(E, dtype, B, Nq, Nk, heads, d, kvb, causal=False, name=""):
    C = heads * d
    q = mk(B, Nq, C, dtype=dtype, seed=1)
    k = mk(kvb, Nk, C, dtype=dtype, seed=2)
    v = mk(kvb, Nk, C, dtype=dtype, seed=3)
    ldv = (Nk + 7) // 8 * 8
    vt = torch.zeros(kvb, C, ldv, device="cuda", dtype=dtype)
    vt[:, :, :Nk] = v.transpose(1, 2)
    got = E.op_attention(q, k, vt, heads, causal=causal)
    ops = launches(E, name)
    ref, pav, e_s, psub = kref.attention64(q, k, v, heads, causal=causal, flash=d == 64)     # d = 64 runs flash_attn
    report(kref.check_attention(name, got, ref, pav, e_s, psub, Nk, dtype))
    return q, k, vt, got, ops


@pytest.mark.parametrize("B,N,heads", [(2, 77, 16), (2, 300, 4)], ids=["clip77", "n300"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_causal_flash_attention(dtype, B, N, heads):
    E = engine(dtype)
    q, k, vt, got, ops = attn_case(E, dtype, B, N, N, heads, 64, B, causal=True, name=f"causal N={N} {dtype}")
    assert kinds(ops)[0] == "flash_attn"
    one = E.op_attention(q[1:].contiguous(), k[1:].contiguous(), vt[1:].contiguous(), heads, causal=True)
    assert torch.equal(one, got[1:])


FLASH = [(2, 200, 63, 5, 1), (2, 200, 64, 5, 2), (2, 200, 65, 5, 2), (2, 256, 77, 10, 1), (1, 300, 4096, 2, 1),
         (2, 128, 4096, 2, 2)]


@pytest.mark.parametrize("B,Nq,Nk,heads,kvb", FLASH, ids=[f"b{b}_q{q}_k{k}_kv{v}" for b, q, k, _, v in FLASH])
@pytest.mark.parametrize("dtype", DTYPES)
def test_flash_attention(dtype, B, Nq, Nk, heads, kvb):
    E = engine(dtype)
    q, k, vt, got, ops = attn_case(E, dtype, B, Nq, Nk, heads, 64, kvb, name=f"flash q{Nq} k{Nk} kvb{kvb} {dtype}")
    assert kinds(ops)[0] == "flash_attn"
    if B > 1 and kvb == B:
        one = E.op_attention(q[1:].contiguous(), k[1:].contiguous(), vt[1:].contiguous(), heads)
        assert torch.equal(one, got[1:])


@pytest.mark.parametrize("ntok", [77, 4096])
@pytest.mark.parametrize("dtype", DTYPES)
def test_vt_projection(dtype, ntok):
    """V^T = Wv X^T + row bias (direct-store epilogue): the cross-attention operand layout."""
    E = engine(dtype)
    B, Cin, Cout = 2, 1024, 640
    x = mk(B, ntok, Cin, dtype=dtype, seed=1)
    w = weight(Cout, Cin, 1, dtype, 2).view(Cout, Cin)
    b = mk(Cout, seed=3)
    got = E.op_vt_proj(x, w, b)
    ops = launches(E, f"vt {ntok} {dtype}")
    assert kinds(ops)[0] == "tapgemm:vt"
    ref = w.double() @ x.double().transpose(1, 2) + b.double()[:, None]
    mag = w.double().abs() @ x.double().abs().transpose(1, 2) + b.double().abs()[:, None]
    report(kref.check_gemm(f"vt {ntok} {dtype}", got[:, :, :ntok], ref, mag, Cin, dtype))


# ---------------------------------------------------------------------------------------------------------------------
# LoRA fold
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("dtype", DTYPES)
def test_lora_fold_read_back(dtype, k):
    """W + s1 B1 A1 + s2 B2 A2 (ranks 4 and 8) folded in fp32 and rounded once, read back bit for bit by convolving one-hot
    inputs (a 16-bit weight times 1.0 plus zeros is exact in fp32); the GEGLU interleave through the GEGLU epilogue."""
    import i2it
    E = engine(dtype)
    Cout, Cin = 256, 64
    W = mk(Cout, Cin, k, k, scale=0.05, seed=1)
    ads = {"a_r4": (4, 0.75), "b_r8": (8, 0.3)}
    sd = {}
    for i, (name, (r, s)) in enumerate(ads.items()):
        sd[f"__op.conv.lora_A.{name}.weight"] = mk(r, Cin, k, k, scale=0.2, seed=10 + i)
        sd[f"__op.conv.lora_B.{name}.weight"] = mk(Cout, r, 1, 1, scale=0.2, seed=20 + i)
        E.set_adapter_scale(name, s)
    E.load_state_dict(sd)
    fold = W.double()
    for name, (r, s) in ads.items():
        A = sd[f"__op.conv.lora_A.{name}.weight"].double().reshape(r, -1)
        Bm = sd[f"__op.conv.lora_B.{name}.weight"].double().reshape(Cout, r)
        fold = fold + s * (Bm @ A).view(Cout, Cin, k, k)
    # one-hot: image i has channel i set at the centre pixel of a k x k map; output pixel (oy, ox) reads tap (k-1-oy, k-1-ox)
    eye = torch.zeros(Cin, k, k, Cin, device="cuda", dtype=dtype)
    eye[torch.arange(Cin), k // 2, k // 2, torch.arange(Cin)] = 1
    got = E.op_conv2d_ex(eye, W)
    launches(E, f"lora k={k} {dtype}")
    back = got.double().flip(1, 2).permute(3, 0, 1, 2)                        # [Cout, Cin, k, k]
    c = kref.check_weights(f"lora fold k={k} {dtype}", back, fold, dtype)
    print("    ", c, f"unequal={c.unequal:.4f}")
    assert c, str(c)
    if k == 1:
        got = E.op_conv2d_ex(eye.view(1, 1, Cin, Cin), W, act=i2it.ACT_GEGLU)
        # operands: the folded weights just read back (the fp32 fold may sit one ulp from round16(float64 fold))
        w16 = back.view(Cout, Cin)
        h, g = w16[: Cout // 2].t(), w16[Cout // 2:].t()                     # rows of the one-hot product: W^T
        ref = h * kref.gelu64(g)
        # a few fp32 operations on h * gelu(g), and the erf approximation (1.5e-7 absolute) scaled by |h| |g| / 2
        mag = h.abs() * (kref.gelu64(g).abs() + g.abs())
        report(kref.check_gemm(f"lora geglu {dtype}", got.view(Cin, Cout // 2), ref, mag, 4, dtype, 2.0))
