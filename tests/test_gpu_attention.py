"""-m gpu: the d = 64 attention (every UNet self- and cross-attention layer, every CLIP text layer) through op_attention,
held to kref.check_attention against float64 at the tails, diagonals, strides and key counts the model gives it.

Operands come as the model lays them out (tests/attn_operands.py): Q and K as column slices of one [B, N, 2C] projection,
V^T with NaN padding columns past Nk.  Every case asserts the path it targets from the launch list (a case that silently
fell back to another path would test nothing), prints that list, the worst err/bound and the mean-ulp statistic, and checks
the bit-for-bit properties that apply to it:
  1. image i equals its own batch-1 call            4. slice operands equal contiguous copies
  2. a shared K/V (kv_batch 1) equals K/V repeated   5. NaN in the V^T padding gives the zero-padded result
  3. head h equals a 1-head call on its 64 columns   6. causal: other K/V at keys > i leave rows <= i unchanged
The unfused path (I2IT_NO_FLASH: fp32 logits GEMM, softmax by row length, PV GEMM) runs the same non-causal cases with
properties 1-5.  At the large key counts the per-element bound is loose (tests/kref.py header), so those checks also cap
the mean-ulp statistic.
The engine reads I2IT_NO_FLASH when it is created, so each path gets its own engine."""
import os
import time

import pytest
import torch

import kref
from attn_operands import D, operands, padded_vt

pytestmark = pytest.mark.gpu

bf, hf = torch.bfloat16, torch.float16
DTYPES = [pytest.param(bf, id="bf16"), pytest.param(hf, id="fp16")]
_ENGINES = {}


def engine(dtype, no_flash=False):
    """One engine per (dtype, path) for the whole module."""
    key = (dtype, no_flash)
    if key not in _ENGINES:
        import i2it
        saved = os.environ.pop("I2IT_NO_FLASH", None)
        try:
            if no_flash:
                os.environ["I2IT_NO_FLASH"] = "1"
            _ENGINES[key] = i2it.Engine(dtype, use_cuda_graph=False)
        finally:
            os.environ.pop("I2IT_NO_FLASH", None)
            if saved is not None:
                os.environ["I2IT_NO_FLASH"] = saved
    return _ENGINES[key]


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


FLASH, UNFUSED = "flash_attn", "tapgemm:attn_qk"             # the launch that identifies each path


def check(name, got, q, k, v, heads, dtype, path, causal=False, rows=None, mean_ulp_max=None):
    """float64 reference for every query row, or for `rows` ((start, stop) ranges) only (non-causal)."""
    assert not (causal and rows)
    Nk = k.shape[1]
    checks = []
    for a, b in rows or [(0, q.shape[1])]:
        ref, pav, e_s, psub = kref.attention64(q[:, a:b], k, v, heads, causal=causal, flash=path == FLASH)
        checks.append(kref.check_attention(f"{name} rows {a}:{b}", got[:, a:b], ref, pav, e_s, psub, Nk, dtype, mean_ulp_max))
    report(*checks)


def flash_call(E, name, q, k, vt, heads, causal=False):
    got = E.op_attention(q, k, vt, heads, causal=causal)
    assert kinds(launches(E, name))[0] == FLASH
    return got


def same(E, path, got, q, k, vt, heads, causal=False):
    """op_attention on these operands gives `got` bit for bit (and still runs on `path`)."""
    other = E.op_attention(q, k, vt, heads, causal=causal)
    assert path in kinds(E.op_launches())
    return torch.equal(other, got)


def head_cols(t, h):
    return t[..., h * D:(h + 1) * D]


def properties(E, path, got, q, k, v, vt, heads, causal=False):
    """Bit-for-bit properties 1-5 of one case on `path`."""
    B, kvb = q.shape[0], k.shape[0]
    if B > 1:                                                    # 1. the last image alone
        i = B - 1
        ki = slice(i, i + 1) if kvb == B else slice(0, 1)
        assert same(E, path, got[i:], q[i:], k[ki], vt[ki], heads, causal), "image B-1 differs from its batch-1 call"
    if B > 1 and kvb == 1:                                       # 2. shared K/V vs K/V repeated per image
        assert same(E, path, got, q, k.expand(B, -1, -1).contiguous(), vt.expand(B, -1, -1).contiguous(), heads, causal), \
            "kv_batch = 1 differs from kv_batch = B"
    if heads > 1:                                                # 3. heads 0 and h-1 as 1-head calls
        for h in (0, heads - 1):
            vth = padded_vt(head_cols(v, h))
            assert same(E, path, head_cols(got, h).contiguous(), head_cols(q, h), head_cols(k, h), vth, 1, causal), \
                f"head {h} differs from its 1-head call"
    if not q.is_contiguous() or not k.is_contiguous():           # 4. slices vs contiguous copies
        assert same(E, path, got, q.contiguous(), k.contiguous(), vt, heads, causal), "slice operands differ from copies"
    assert same(E, path, got, q, k, padded_vt(v, nan=False), heads, causal), "NaN V^T padding changed the result"   # 5.


# ---------------------------------------------------------------------------------------------------------------------
# non-causal matrix: (B, kv_batch, Nq, Nk, heads, regime, layout)
# ---------------------------------------------------------------------------------------------------------------------
CASES = [
    (1, 1, 1, 1, 1, "flat", "dense"),            # one token attending to one token
    (2, 2, 1, 1, 2, "spiky", "slice"),           # an 8x8 image: self-attention over its 1x1 latent
    (2, 2, 4, 4, 5, "flat", "slice"),            # 2x2 latent map, level-0 heads
    (2, 2, 9, 9, 5, "peaked", "slice"),          # 3x3
    (16, 1, 4, 77, 5, "flat", "dense"),          # cross-attention, one prompt shared by 16 images
    (4, 4, 9, 77, 10, "spiky", "dense"),         # per-image prompts
    (2, 2, 63, 63, 5, "spiky", "slice"),
    (2, 2, 64, 64, 5, "peaked", "slice"),
    (2, 2, 65, 65, 10, "spiky", "slice"),
    (2, 1, 127, 1, 4, "flat", "dense"),          # a single key
    (3, 3, 128, 4, 2, "uniform", "slice"),
    (2, 2, 129, 9, 1, "flat", "slice"),
    (2, 2, 136, 136, 5, "spiky", "slice"),       # q0 < Nq <= q1 inside one thread
    (16, 1, 136, 77, 5, "peaked", "dense"),
    (8, 1, 300, 77, 20, "flat", "dense"),        # 480 CTAs: several waves
    (16, 16, 300, 129, 10, "spiky", "dense"),
    (16, 16, 64, 64, 20, "flat", "slice"),
    (16, 16, 1024, 1024, 5, "flat", "slice"),    # 32x32 latent, 640 CTAs
    (2, 2, 300, 1024, 5, "peaked", "slice"),
    (2, 1, 77, 1024, 10, "spiky", "dense"),
    (1, 1, 65, 1025, 10, "spiky", "slice"),
    (2, 2, 64, 1025, 5, "peaked", "dense"),
    (2, 1, 300, 4096, 5, "uniform", "dense"),
    (1, 1, 63, 4096, 10, "spiky", "dense"),
    (1, 1, 129, 4097, 10, "spiky", "dense"),
    (2, 2, 300, 4097, 5, "peaked", "slice"),
    (2, 2, 4, 4097, 20, "peaked", "dense"),
    (1, 1, 300, 14400, 5, "spiky", "slice"),
    (2, 2, 136, 14400, 10, "flat", "dense"),
    (1, 1, 9, 14400, 1, "uniform", "dense"),
    (2, 2, 65, 65, 5, "sunken", "slice"),        # every real logit near -32: an unmasked tail would win every row
    (1, 1, 129, 4097, 10, "sunken", "dense"),
    (2, 1, 300, 14401, 5, "sunken", "slice"),
]
IDS = [f"b{b}_kv{kv}_q{nq}_k{nk}_h{h}_{r}_{lay}" for b, kv, nq, nk, h, r, lay in CASES]


@pytest.mark.parametrize("case", CASES, ids=IDS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_flash_attention_d64(dtype, case):
    B, kvb, Nq, Nk, heads, regime, layout = case
    E = engine(dtype)
    q, k, v, vt = operands(B, kvb, Nq, Nk, heads, regime, dtype, layout=layout, seed=Nq + Nk)
    name = f"flash {IDS[CASES.index(case)]} {dtype}"
    got = flash_call(E, name, q, k, vt, heads)
    check(name, got, q, k, v, heads, dtype, FLASH)
    properties(E, FLASH, got, q, k, v, vt, heads)


def softmax_variant(Nk):
    return "32" if Nk <= 1024 else "128" if Nk <= 4096 else "long"


@pytest.mark.parametrize("case", CASES, ids=IDS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_unfused_attention_d64(dtype, case):
    """I2IT_NO_FLASH: fp32 logits GEMM, softmax_kernel<32> up to 1024 keys, <128> up to 4096, softmax_long above, PV GEMM."""
    B, kvb, Nq, Nk, heads, regime, layout = case
    lds = (Nk + 7) // 8 * 8
    assert B * heads * Nq * lds * 6 < (8 << 30)                  # S (fp32) and P (16 bit) of every case fit
    E = engine(dtype, no_flash=True)
    q, k, v, vt = operands(B, kvb, Nq, Nk, heads, regime, dtype, layout=layout, seed=Nq + Nk)
    name = f"unfused {IDS[CASES.index(case)]} {dtype}"
    got = E.op_attention(q, k, vt, heads)
    ops = launches(E, name)
    assert FLASH not in kinds(ops) and {UNFUSED, "tapgemm:attn_pv"} <= set(kinds(ops))
    assert [o["shape"] for o in ops if o["kind"] == "softmax"] == [softmax_variant(Nk)]
    check(name, got, q, k, v, heads, dtype, UNFUSED)
    properties(E, UNFUSED, got, q, k, v, vt, heads)


@pytest.mark.parametrize("dtype", DTYPES)
def test_unfused_refuses_causal(dtype):
    """Causal attention runs on the flash path only; the refusal leaves the handle usable."""
    E = engine(dtype, no_flash=True)
    q, k, v, vt = operands(2, 2, 77, 77, 2, "flat", dtype, layout="slice", seed=5)
    with pytest.raises(RuntimeError, match="causal attention runs on the flash path"):
        E.op_attention(q, k, vt, 2, causal=True)
    got = E.op_attention(q, k, vt, 2)
    assert UNFUSED in kinds(launches(E, f"unfused after refusal {dtype}"))
    check(f"unfused after refusal {dtype}", got, q, k, v, 2, dtype, UNFUSED)


# ---------------------------------------------------------------------------------------------------------------------
# causal (CLIP text tower): the diagonal at every warp offset inside a 128-row Q tile
# ---------------------------------------------------------------------------------------------------------------------
CAUSAL_N = [1, 2, 63, 64, 65, 77, 127, 128, 129, 191, 192, 193, 300]
CAUSAL_BH = [(1, 1, "flat"), (16, 16, "peaked"), (1, 16, "flat"), (16, 1, "peaked")]


@pytest.mark.parametrize("N", CAUSAL_N)
@pytest.mark.parametrize("dtype", DTYPES)
def test_causal_flash_attention_d64(dtype, N):
    E = engine(dtype)
    for B, heads, regime in CAUSAL_BH:
        q, k, v, vt = operands(B, B, N, N, heads, regime, dtype, layout="slice", seed=N + B)
        name = f"causal N={N} B={B} h={heads} {regime} {dtype}"
        got = flash_call(E, name, q, k, vt, heads, causal=True)
        check(name, got, q, k, v, heads, dtype, FLASH, causal=True)
        properties(E, FLASH, got, q, k, v, vt, heads, causal=True)
        # 6. other finite K and V at keys > i leave rows <= i unchanged
        for i in sorted({0, N // 2, max(N - 2, 0)}):
            k2, v2 = k.clone(), v.clone()
            g = torch.Generator(device="cuda").manual_seed(i)
            k2[:, i + 1:] = torch.randn(k2[:, i + 1:].shape, device="cuda", generator=g).to(dtype) * 4
            v2[:, i + 1:] = torch.randn(v2[:, i + 1:].shape, device="cuda", generator=g).to(dtype)
            other = E.op_attention(q, k2, padded_vt(v2), heads, causal=True)
            assert torch.equal(other[:, :i + 1], got[:, :i + 1]), f"{name}: keys > {i} changed rows <= {i}"


# ---------------------------------------------------------------------------------------------------------------------
# the key counts of large images: UNet levels of a 4032x3024 image, and one batch whose Q/K buffer passes 2^31 elements
# ---------------------------------------------------------------------------------------------------------------------
N12 = (3024 // 8) * (4032 // 8)                  # 190512 latent tokens at UNet level 0
LARGE = [(1, N12, 5), (2, N12 // 2, 10), (1, N12 // 4, 20), (18, N12, 5)]


def sample_rows(N):
    """The first Q tile, rows across a tile boundary a third of the way in, the middle, the last 100 rows."""
    t = 128 * (N // 384)
    return [(0, 128), (t - 40, t + 40), (N // 2 - 32, N // 2 + 32), (N - 100, N)]


@pytest.mark.parametrize("B,N,heads", LARGE, ids=[f"b{b}_n{n}_h{h}" for b, n, h in LARGE])
@pytest.mark.parametrize("dtype", DTYPES)
def test_flash_attention_large(dtype, B, N, heads):
    """Self-attention over every latent token of a 12 MP image's UNet levels.  At B = 18 the fused Q/K buffer holds
    18 * 190512 * 640 = 2.19e9 > 2^31 elements; the last image is checked against float64 and against its batch-1 call.
    The sampled rows are also held to kref.ATTN_MEAN_ULP_MAX: at these key counts the per-element bound alone would pass
    a dropped KV tile (tests/test_flash_emulation.py shows that the cap does not)."""
    t0 = time.time()
    E = engine(dtype)
    C = heads * D
    g = torch.Generator(device="cuda").manual_seed(N + heads)
    qk = torch.randn(B, N, 2 * C, device="cuda", generator=g, dtype=dtype)
    v = torch.randn(B, N, C, device="cuda", generator=g, dtype=dtype)
    vt = padded_vt(v)
    q, k = qk[..., :C], qk[..., C:]
    name = f"large B={B} N={N} h={heads} {dtype}"
    got = flash_call(E, name, q, k, vt, heads)
    torch.cuda.synchronize()
    i = B - 1
    check(name + f" image {i}", got[i:], q[i:], k[i:], v[i:], heads, dtype, FLASH, rows=sample_rows(N),
          mean_ulp_max=kref.ATTN_MEAN_ULP_MAX)
    if B > 1:
        assert same(E, FLASH, got[i:], q[i:], k[i:], vt[i:], heads), "the last image differs from its batch-1 call"
    print(f"[{name}] wall {time.time() - t0:.1f} s")
    del qk, v, vt, got
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------
# the smallest images: teacher-forced layer audits of forwards whose latents are 1x1 and 3x5
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W", [(2, 8, 8), (1, 24, 40)], ids=["8x8_b2", "24x40"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_tiny_images_layer_audit(dtype, B, H, W):
    """Attention over 1 to 15 tokens, stride-2 convs of 1-pixel maps and GroupNorm over one pixel, every layer held to
    its float64 bound on the engine's own inputs (tests/test_gpu_layers.run_case)."""
    import weights as Wt
    from test_gpu_layers import run_case
    sd = Wt.make_state_dict("pix2pix", Wt.TINY, seed=0, perturb_norm=True)
    run_case(f"tiny {H}x{W} b{B} {dtype}", "pix2pix", Wt.TINY, sd, dtype, B, H, W)
