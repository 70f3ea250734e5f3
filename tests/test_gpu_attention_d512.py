"""-m gpu: the VAE mid-block attention (one head of 512, Nq = Nk = (H/8)(W/8) tokens) through op_attention, held to
kref.check_attention against float64 at the tails, batches, layouts and key counts the VAE gives it.

Above 8192 keys the engine runs flash_attn512_kernel (csrc/flash.cuh); at and below it, the unfused path: fp32 logits GEMM,
softmax by row length, PV GEMM.  Operands come as the model lays them out (tests/attn_operands.py): Q and K as column
slices of one [B, N, 1024] projection, V^T with NaN padding columns past Nk, or V^T straight from op_vt_proj.  Every case
asserts the path it targets from the launch list, prints that list, the worst err/bound and the mean-ulp statistic, and
checks the bit-for-bit properties that apply to it:
  1. image B-1 equals its batch-1 call               4. NaN in the V^T padding gives the zero-padded result
  2. a shared K/V (kv_batch 1) equals K/V repeated    5. fused path: a call on a 64-aligned block of query rows gives
  3. slice operands equal contiguous copies              those rows of the full call
Every query row is checked up to 16384 keys; above that, sampled rows (the first Q tile, a window across a tile boundary,
the middle, the last 100 rows with the ragged last Q tile).  From 32400 keys up the per-element bound is loose (tests/kref.py
header), so those checks also cap the mean-ulp statistic (on the unfused path in bf16 only: tests/kref.py header).
The engine reads I2IT_NO_FLASH when it is created, so each path gets its own engine."""
import os
import time

import pytest
import torch

import kref
from attn_operands import operands, padded_vt

pytestmark = pytest.mark.gpu

bf, hf = torch.bfloat16, torch.float16
DTYPES = [pytest.param(bf, id="bf16"), pytest.param(hf, id="fp16")]
D5 = 512
FUSED, UNFUSED = "flash_attn512", "tapgemm:attn_qk"          # the launch that identifies each path
THRESHOLD = 8192                                             # Engine::attention: fused above this many keys
FULL_ROWS_NK = 16384                                         # every query row checked up to this key count
CAP_NK = 32400                                               # mean-ulp cap from this key count up
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


def softmax_variant(Nk):
    return "32" if Nk <= 1024 else "128" if Nk <= 4096 else "long"


def assert_path(E, name, path, Nk):
    ops = launches(E, name)
    if path == FUSED:
        assert FUSED in kinds(ops) and UNFUSED not in kinds(ops) and "softmax" not in kinds(ops), kinds(ops)
    else:
        assert FUSED not in kinds(ops) and {UNFUSED, "tapgemm:attn_pv"} <= set(kinds(ops)), kinds(ops)
        assert [o["shape"] for o in ops if o["kind"] == "softmax"] == [softmax_variant(Nk)]


def sample_rows(N):
    """The first Q tile, rows across a 64-row tile boundary a third of the way in, the middle, the last 100 rows."""
    t = 64 * (N // 192)
    return [(0, 64), (t - 40, t + 40), (N // 2 - 32, N // 2 + 32), (N - 100, N)]


def check_rows(B, Nq, Nk):
    """Every row in chunks of about 2^25 logits per float64 temporary, or the sampled rows of a long query sequence."""
    if Nk > FULL_ROWS_NK and Nq > 400:
        return sample_rows(Nq)
    step = max(1, (1 << 25) // (B * Nk))
    return [(a, min(Nq, a + step)) for a in range(0, Nq, step)]


def check(name, got, q, k, v, dtype, path, rows=None):
    """float64 reference of the query rows `rows` ((start, stop) ranges; default check_rows) on `path`'s subnormal set."""
    Nk = k.shape[1]
    # the unfused path's fp16 probabilities are relative to the row sum: past ~16384 keys most fall below fp16's normal
    # range, where their rounding is absolute (kref.py header), so the mean-ulp cap holds on the fused path and in bf16
    cap = kref.ATTN_MEAN_ULP_MAX if Nk >= CAP_NK and (path == FUSED or dtype == bf) else None
    checks = []
    for a, b in rows or check_rows(q.shape[0], q.shape[1], Nk):
        ref, pav, e_s, psub = kref.attention64(q[:, a:b], k, v, 1, flash=path == FUSED)
        checks.append(kref.check_attention(f"{name} rows {a}:{b}", got[:, a:b], ref, pav, e_s, psub, Nk, dtype, cap))
        del ref, pav, e_s, psub
    for c in checks:
        print("   ", c)
    print(f"    [{name}] worst err/bound {max(c.worst for c in checks):.3f}, "
          f"mean-ulp {max(c.mean_ulp for c in checks):.3f}" + (f"/{cap:.2f}" if cap else ""))
    for c in checks:
        assert c, str(c)


def same(E, path, got, q, k, vt):
    """op_attention on these operands gives `got` bit for bit (and still runs on `path`)."""
    other = E.op_attention(q, k, vt, 1)
    assert path in kinds(E.op_launches())
    return torch.equal(other, got)


def query_blocks(Nq):
    """64-aligned blocks of query rows: the last Q tile (ragged where Nq % 64 != 0) and two tiles from the middle."""
    blocks = [(64 * ((Nq - 1) // 64), Nq)] if Nq > 64 else []
    if Nq >= 256:
        a = 64 * (Nq // 128)
        blocks.append((a, a + 128))
    return blocks


def properties(E, path, got, q, k, v, vt):
    """Bit-for-bit properties 1-5 of one case on `path`."""
    B, kvb, Nq = q.shape[0], k.shape[0], q.shape[1]
    if B > 1:                                                    # 1. the last image alone
        i = B - 1
        ki = slice(i, i + 1) if kvb == B else slice(0, 1)
        assert same(E, path, got[i:], q[i:], k[ki], vt[ki]), "image B-1 differs from its batch-1 call"
    if B > 1 and kvb == 1:                                       # 2. shared K/V vs K/V repeated per image
        assert same(E, path, got, q, k.expand(B, -1, -1).contiguous(), vt.expand(B, -1, -1).contiguous()), \
            "kv_batch = 1 differs from kv_batch = B"
    if not q.is_contiguous() or not k.is_contiguous():           # 3. slices vs contiguous copies
        assert same(E, path, got, q.contiguous(), k.contiguous(), vt), "slice operands differ from copies"
    assert same(E, path, got, q, k, padded_vt(v, nan=False)), "NaN V^T padding changed the result"   # 4.
    if path == FUSED:                                            # 5. a block of query rows as a call of its own
        for a, b in query_blocks(Nq):
            qb = q[:, a:b] if B == 1 else q[:, a:b].contiguous()
            assert same(E, path, got[:, a:b], qb, k, vt), f"query rows {a}:{b} differ from the full call"


def model_operands(E, B, N, dtype, seed):
    """The operands vae_attn (csrc/model.cu) hands the kernel: Q and K as column slices of one [B, N, 1024] projection,
    V^T = Wv X^T + b from op_vt_proj ([B, 512, round_up(N, 8)], its padding columns whatever that launch leaves there)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    qk = torch.randn(B, N, 2 * D5, device="cuda", generator=g).to(dtype)
    x = torch.randn(B, N, D5, device="cuda", generator=g).to(dtype)
    w = torch.randn(D5, D5, device="cuda", generator=g) / D5 ** 0.5
    b = torch.randn(D5, device="cuda", generator=g) * 0.1
    vt = E.op_vt_proj(x, w, b)
    assert vt.shape == (B, D5, (N + 7) // 8 * 8)
    return qk[..., :D5], qk[..., D5:], vt[:, :, :N].transpose(1, 2), vt


def case_operands(E, case, dtype):
    B, kvb, Nq, Nk, regime, layout = case
    if layout == "model":
        assert B == kvb and Nq == Nk and regime == "flat"
        return model_operands(E, B, Nk, dtype, seed=Nk)
    return operands(B, kvb, Nq, Nk, 1, regime, dtype, layout=layout, seed=Nq + Nk, d=D5)


# ---------------------------------------------------------------------------------------------------------------------
# fused matrix (Nk > 8192): the key counts of real images and every tail position, (B, kv_batch, Nq, Nk, regime, layout)
# ---------------------------------------------------------------------------------------------------------------------
FUSED_CASES = [
    (1, 1, 300, 8193, "flat", "dense"),
    (2, 2, 300, 8193, "flat", "dense"),
    (1, 1, 8193, 8193, "spiky", "slice"),        # tail 1: the first key count past the threshold
    (3, 3, 72, 8193, "sunken", "slice"),         # q0 < Nq <= q1 inside one thread
    (16, 1, 8, 8193, "sunken", "slice"),
    (2, 2, 8255, 8255, "sunken", "slice"),       # tail 63
    (16, 1, 300, 8255, "spiky", "slice"),        # 160 CTAs: two waves
    (1, 1, 63, 8255, "peaked", "dense"),
    (2, 2, 8256, 8256, "peaked", "slice"),       # the first whole-tile count past the threshold
    (1, 1, 1, 8256, "uniform", "dense"),
    (3, 3, 9216, 9216, "flat", "slice"),         # 768^2
    (16, 16, 64, 9216, "peaked", "slice"),
    (2, 2, 12065, 12065, "flat", "model"),       # 1016x760, tail 33
    (1, 1, 12065, 12065, "spiky", "slice"),
    (3, 1, 65, 12065, "sunken", "slice"),
    (1, 1, 12100, 12100, "sunken", "slice"),     # 880^2, tail 4
    (16, 16, 72, 12100, "spiky", "slice"),
    (1, 1, 300, 14400, "flat", "dense"),
    (2, 1, 129, 14400, "flat", "dense"),
    (1, 1, 300, 14400, "peaked", "dense"),
    (1, 1, 14400, 14400, "flat", "model"),       # 1280x720
    (2, 2, 300, 16384, "flat", "dense"),
    (1, 1, 300, 16384, "flat", "dense"),
    (1, 1, 16384, 16384, "peaked", "slice"),     # 1024^2
    (2, 2, 129, 16384, "uniform", "slice"),
    (1, 1, 32400, 32400, "sunken", "slice"),     # 1920x1080, tail 16
    (2, 2, 72, 32400, "spiky", "slice"),
    (1, 1, 300, 65536, "flat", "dense"),
    (1, 1, 65536, 65536, "peaked", "slice"),     # 2048^2
    (1, 1, 129600, 129600, "flat", "slice"),     # 3840x2160
    (1, 1, 190512, 190512, "flat", "dense"),     # 4032x3024, tail 48
    (1, 1, 190512, 190512, "spiky", "slice"),
    (1, 1, 300, 190512, "sunken", "slice"),
]
FUSED_IDS = [f"b{b}_kv{kv}_q{nq}_k{nk}_{r}_{lay}" for b, kv, nq, nk, r, lay in FUSED_CASES]


def run_case(E, case, case_id, dtype, path):
    t0 = time.time()
    name = f"{'fused' if path == FUSED else 'unfused'} {case_id} {dtype}"
    q, k, v, vt = case_operands(E, case, dtype)
    got = E.op_attention(q, k, vt, 1)
    torch.cuda.synchronize()
    assert_path(E, name, path, k.shape[1])
    check(name, got, q, k, v, dtype, path)
    properties(E, path, got, q, k, v, vt)
    print(f"    [{name}] wall {time.time() - t0:.2f} s")
    del q, k, v, vt, got
    torch.cuda.empty_cache()


@pytest.mark.parametrize("case", FUSED_CASES, ids=FUSED_IDS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_fused_attention_d512(dtype, case):
    run_case(engine(dtype), case, FUSED_IDS[FUSED_CASES.index(case)], dtype, FUSED)


# the fused cases whose unfused S (fp32) and P (16 bit) buffers fit in 8 GB, run with I2IT_NO_FLASH
NO_FLASH_CASES = [c for c in FUSED_CASES if c[0] * c[2] * ((c[3] + 7) // 8 * 8) * 6 <= (8 << 30)]


@pytest.mark.parametrize("case", NO_FLASH_CASES, ids=[FUSED_IDS[FUSED_CASES.index(c)] for c in NO_FLASH_CASES])
@pytest.mark.parametrize("dtype", DTYPES)
def test_no_flash_attention_d512(dtype, case):
    """I2IT_NO_FLASH keeps the d = 512 attention unfused above the threshold too (`long` softmax)."""
    run_case(engine(dtype, no_flash=True), case, FUSED_IDS[FUSED_CASES.index(case)], dtype, UNFUSED)


# ---------------------------------------------------------------------------------------------------------------------
# unfused path (Nk <= 8192): 8x8, 24x40, 256^2, 512^2, 512x768, 560x840, 720^2 and the threshold
# ---------------------------------------------------------------------------------------------------------------------
UNFUSED_CASES = [
    (2, 2, 1, 1, "flat", "slice"),               # an 8x8 image: one latent token
    (16, 1, 1, 1, "flat", "slice"),
    (2, 2, 15, 15, "spiky", "slice"),            # 24x40
    (3, 1, 15, 15, "sunken", "slice"),
    (1, 1, 300, 1024, "flat", "dense"),          # softmax_kernel<32>
    (2, 2, 1024, 1024, "peaked", "slice"),       # 256^2
    (1, 1, 300, 1025, "flat", "dense"),          # softmax_kernel<128>
    (1, 1, 300, 4096, "flat", "dense"),
    (2, 2, 4096, 4096, "flat", "model"),         # 512^2
    (16, 16, 72, 4096, "spiky", "slice"),
    (1, 1, 300, 4097, "flat", "dense"),          # softmax_long_kernel
    (1, 1, 6144, 6144, "uniform", "slice"),      # 512x768
    (1, 1, 300, 7350, "flat", "dense"),
    (1, 1, 7350, 7350, "sunken", "slice"),       # 560x840
    (2, 1, 129, 7350, "spiky", "dense"),
    (1, 1, 8100, 8100, "spiky", "slice"),        # 720^2
    (3, 3, 65, 8100, "sunken", "slice"),
    (1, 1, 300, 8192, "flat", "dense"),          # the threshold
    (1, 1, 8192, 8192, "peaked", "slice"),
]
UNFUSED_IDS = [f"b{b}_kv{kv}_q{nq}_k{nk}_{r}_{lay}" for b, kv, nq, nk, r, lay in UNFUSED_CASES]


@pytest.mark.parametrize("case", UNFUSED_CASES, ids=UNFUSED_IDS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_unfused_attention_d512(dtype, case):
    """The path of every forward up to 720^2: fp32 logits GEMM, softmax_kernel<32> up to 1024 keys, <128> up to 4096,
    softmax_long above, PV GEMM."""
    run_case(engine(dtype), case, UNFUSED_IDS[UNFUSED_CASES.index(case)], dtype, UNFUSED)


@pytest.mark.parametrize("dtype", DTYPES)
def test_d512_path_threshold(dtype):
    """8192 keys run unfused with the `long` softmax, 8193 keys run fused; each passes its bound."""
    E = engine(dtype)
    for Nk, path in ((THRESHOLD, UNFUSED), (THRESHOLD + 1, FUSED)):
        q, k, v, vt = operands(1, 1, 300, Nk, 1, "flat", dtype, seed=Nk, d=D5)
        got = E.op_attention(q, k, vt, 1)
        name = f"threshold k{Nk} {dtype}"
        assert_path(E, name, path, Nk)
        check(name, got, q, k, v, dtype, path)


# ---------------------------------------------------------------------------------------------------------------------
# past 2^31 elements: 256 images of 16400 tokens
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_fused_attention_d512_past_2g_elements(dtype):
    """B = 256 at N = 16400 (tail 16): the Q/K slice buffer holds 256 * 16400 * 1024 = 4.3e9 elements, V^T and the output
    2.15e9 each (17 GB in all).  Images 0, 127 and 255 are checked on sampled rows against float64 with the mean-ulp cap,
    and image 255 against its batch-1 call."""
    t0 = time.time()
    E = engine(dtype)
    B, N = 256, 16400
    g = torch.Generator(device="cuda").manual_seed(N)
    qk = torch.randn(B, N, 2 * D5, device="cuda", generator=g, dtype=dtype)
    vt = torch.randn(B, D5, (N + 7) // 8 * 8 + 8, device="cuda", generator=g, dtype=dtype)
    vt[:, :, N:] = float("nan")
    q, k = qk[..., :D5], qk[..., D5:]
    name = f"B={B} N={N} {dtype}"
    got = E.op_attention(q, k, vt, 1)
    torch.cuda.synchronize()
    assert_path(E, name, FUSED, N)
    checks = []
    for i in (0, 127, 255):
        v = vt[i:i + 1, :, :N].transpose(1, 2)
        for a, b in sample_rows(N):
            ref, pav, e_s, psub = kref.attention64(q[i:i + 1, a:b], k[i:i + 1], v, 1, flash=True)
            checks.append(kref.check_attention(f"{name} image {i} rows {a}:{b}", got[i:i + 1, a:b], ref, pav, e_s, psub, N,
                                               dtype, kref.ATTN_MEAN_ULP_MAX))
    for c in checks:
        print("   ", c)
    print(f"    [{name}] worst err/bound {max(c.worst for c in checks):.3f}, mean-ulp {max(c.mean_ulp for c in checks):.3f}")
    for c in checks:
        assert c, str(c)
    assert same(E, FUSED, got[255:], q[255:], k[255:], vt[255:]), "image 255 differs from its batch-1 call"
    print(f"    [{name}] wall {time.time() - t0:.1f} s")
    del qk, vt, got, q, k
    torch.cuda.empty_cache()
