"""CPU tests of the kernel acceptance criterion (tests/kref.py): it accepts the correctly rounded float64 reference and rejects
the localised errors an averaged or max-relative bound lets through."""
import math

import pytest
import torch

import kref

DTYPES = [torch.bfloat16, torch.float16]


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _conv_case(dtype, seed=0, N=2, H=12, W=12, Cin=32, Cout=64):
    g = _gen(seed)
    x = torch.randn(N, H, W, Cin, generator=g).to(dtype)
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) / math.sqrt(9 * Cin)).to(dtype).float()
    b = torch.randn(Cout, generator=g) * 0.1
    ref = kref.conv64(x, w, b)
    mag = kref.conv64(x.abs(), w.abs(), b.abs())
    return x, w, b, ref, mag, 9 * Cin


def test_ulp16_is_the_dtype_spacing():
    y = torch.tensor([1.0, 1.5, 2.0, -3.0, 0.0, 1e-30], dtype=torch.float64)
    assert kref.ulp16(y, torch.bfloat16)[:4].tolist() == [2 ** -7, 2 ** -7, 2 ** -6, 2 ** -6]
    assert kref.ulp16(y, torch.float16)[:4].tolist() == [2 ** -10, 2 ** -10, 2 ** -9, 2 ** -9]
    assert kref.ulp16(y, torch.float16)[4:].tolist() == [2 ** -24, 2 ** -24]          # fp16 subnormal spacing
    # nextafter in the dtype is exactly one ulp away
    for dt in DTYPES:
        v = torch.randn(1000, generator=_gen(1), dtype=torch.float64).to(dt)
        nxt = torch.nextafter(v.float(), torch.full_like(v.float(), math.inf)).to(dt)
        nxt = torch.where(nxt == v, (v.float() + kref.ulp16(v.double(), dt).float()).to(dt), nxt)
        assert torch.equal((nxt.double() - v.double()).abs(), kref.ulp16(v.double(), dt))


@pytest.mark.parametrize("dtype", DTYPES)
def test_gemm_accepts_correct_rounding_rejects_dropped_tap_and_ulp_bias(dtype):
    x, w, b, ref, mag, K = _conv_case(dtype)
    good = kref.check_gemm("ok", kref.round16(ref, dtype), ref, mag, K, dtype)
    assert good, str(good)
    assert 0.2 < good.mean_ulp < 0.3, good.mean_ulp
    w_drop = w.clone()
    w_drop[:, :, 0, 2] = 0                                      # one of nine taps missing
    bad = kref.check_gemm("drop", kref.round16(kref.conv64(x, w_drop, b), dtype), ref, mag, K, dtype)
    assert not bad and bad.n_bad > 0, str(bad)
    got = kref.round16(ref, dtype)
    sel = torch.rand(got.shape, generator=_gen(5)) < 0.01       # +1 ulp on 1 % of the elements
    got = torch.where(sel, got + kref.ulp16(got, dtype), got)
    bad = kref.check_gemm("ulp", got, ref, mag, K, dtype)
    assert not bad and bad.n_bad > 0, str(bad)


@pytest.mark.parametrize("dtype", DTYPES)
def test_gemm_rejects_one_stale_128_row_tile(dtype):
    g = _gen(2)
    M, Kd, Nn = 640, 256, 192
    x = torch.randn(M, Kd, generator=g).to(dtype)
    w = (torch.randn(Nn, Kd, generator=g) / 16).to(dtype)
    ref = x.double() @ w.double().t()
    mag = x.double().abs() @ w.double().abs().t()
    got = kref.round16(ref, dtype)
    assert kref.check_gemm("ok", got, ref, mag, Kd, dtype)
    stale = got.clone()
    x2 = torch.randn(M, Kd, generator=_gen(3)).to(dtype)       # what an earlier launch left in the buffer
    stale[256:384] = kref.round16(x2.double() @ w.double().t(), dtype)[256:384]
    bad = kref.check_gemm("stale", stale, ref, mag, Kd, dtype)
    assert not bad and bad.n_bad > 0.9 * 128 * Nn, str(bad)


@pytest.mark.parametrize("dtype", DTYPES)
def test_group_norm_rejects_one_group_with_stats_off_by_half_a_percent(dtype):
    g = _gen(4)
    N, H, W, C = 2, 8, 8, 128
    x = (torch.randn(N, H, W, C, generator=g) * 1.7 + 0.3).to(dtype)
    gamma, beta = torch.randn(C, generator=g) * 0.2 + 1, torch.randn(C, generator=g) * 0.1
    for silu in (False, True):
        ref, bound = kref.group_norm64(x, gamma, beta, 1e-6, silu, dtype)
        ok = kref.check_norm("ok", kref.round16(ref, dtype), ref, bound, dtype)
        assert ok, str(ok)
        # group 5 of image 1 normalised with rstd * 1.005
        xd = x.double().reshape(N, H * W, 32, C // 32)
        mean = xd.mean(dim=(1, 3), keepdim=True)
        rstd = 1 / torch.sqrt(((xd - mean) ** 2).mean(dim=(1, 3), keepdim=True) + 1e-6)
        rstd[1, :, 5] *= 1.005
        y = ((xd - mean) * rstd).reshape(N, H, W, C) * gamma.double() + beta.double()
        y = y * torch.sigmoid(y) if silu else y
        bad = kref.check_norm("stats", kref.round16(y, dtype), ref, bound, dtype)
        assert not bad and bad.n_bad > 0, str(bad)
        assert all(i[0] == 1 and (i[3] // 4) == 5 for i in bad.where)


@pytest.mark.parametrize("dtype", DTYPES)
def test_attention_rejects_a_causal_mask_one_key_off(dtype):
    g = _gen(6)
    B, N, heads, d = 1, 77, 2, 64
    q, k, v = (torch.randn(B, N, heads * d, generator=g).to(dtype) for _ in range(3))
    ref, pav, e_s, psub = kref.attention64(q, k, v, heads, causal=True)
    ok = kref.check_attention("ok", kref.round16(ref, dtype), ref, pav, e_s, psub, N, dtype)
    assert ok, str(ok)
    # the mask admits key i+1 for query i
    qf = q.double().view(B, N, heads, d).transpose(1, 2)
    kf = k.double().view(B, N, heads, d).transpose(1, 2)
    vf = v.double().view(B, N, heads, d).transpose(1, 2)
    s = (qf @ kf.transpose(-1, -2) / math.sqrt(d)).masked_fill(torch.ones(N, N, dtype=torch.bool).triu(2), float("-inf"))
    leak = (torch.softmax(s, -1) @ vf).transpose(1, 2).reshape(B, N, heads * d)
    bad = kref.check_attention("leak", kref.round16(leak, dtype), ref, pav, e_s, psub, N, dtype)
    assert not bad and bad.n_bad > 0, str(bad)


@pytest.mark.parametrize("dtype", DTYPES)
def test_subpixel_taps_equal_upsample_then_conv(dtype):
    """Pre-summed taps in float64 are exactly interpolate(nearest) then conv2d; rounded once they stay within 2u mag."""
    g = _gen(7)
    x = torch.randn(1, 5, 6, 16, generator=g).to(dtype)
    w = torch.randn(24, 16, 3, 3, generator=g) / 12
    b = torch.randn(24, generator=g)
    exact = kref.conv64(x, w, b, up2x=True)
    wsub64 = kref.subpixel_weights(w.double(), torch.float64)
    assert torch.allclose(kref.subpixel_conv64(x, wsub64, b), exact, rtol=0, atol=1e-12)
    mag = kref.conv64(x.abs(), w.abs(), b.abs(), up2x=True)
    got = kref.round16(kref.subpixel_conv64(x, kref.subpixel_weights(w, dtype), b), dtype)
    c = kref.Check("comp", got, exact, kref.ulp16(exact, dtype) + 2 * kref.unit_roundoff(dtype) * mag, dtype)
    assert c, str(c)


def test_weight_check_counts_unequal_elements():
    dtype = torch.bfloat16
    w = torch.randn(64, 64, generator=_gen(8), dtype=torch.float64)
    assert kref.check_weights("ok", kref.round16(w, dtype), w, dtype)
    off = kref.round16(w, dtype)
    off[:2] += kref.ulp16(off[:2], dtype)                      # 3 % one ulp away: inside the bound, too many unequal
    c = kref.check_weights("unequal", off, w, dtype)
    assert not c and c.n_bad == 0
