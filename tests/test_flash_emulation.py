"""CPU proof that the attention matrices of tests/test_gpu_attention.py (d = 64) and tests/test_gpu_attention_d512.py
(d = 512) would catch a wrong kernel.

`flash_emulate` repeats flash_attn_kernel's arithmetic (csrc/flash.cuh) in torch: 64-key tiles, fp32 logits, a running
maximum in raw logit units with exp2 at scale * log2(e), P rounded to the activation dtype with l summed over the ROUNDED P,
the rescale of O and l by exp2((m_old - m_new) * scale * log2(e)), the causal and ragged-tail masks, one final rounding.
At d = 512 with one head the same arithmetic is flash_attn512_kernel's, element by element: each of its two CTAs per Q tile
recomputes the whole S of its rows and runs that online softmax, and only splits the output columns.
It passes kref.check_attention on CPU-sized versions of the GPU cases; each mutation below (one plausible kernel bug) must
fail at least one of them, so a kernel with that bug could not pass the GPU suite either."""
import functools
import math

import pytest
import torch

import kref
from attn_operands import operands

BN = 64
LOG2E = 1.4426950408889634
MUTATIONS = ["no_rescale", "tail_unmasked", "last_tile_dropped", "causal_one_late", "next_head_k", "scale_1_over_d"]
# flash_attn512_kernel's own failure modes: S without one of K's eight 64-wide d-chunks (the last), the four V^T column
# blocks of a half read one block along ((c + 1) mod 4), and the d = 64 kernel's 1/sqrt(64) scale
MUTATIONS_D512 = ["no_rescale", "tail_unmasked", "last_tile_dropped", "k_chunk_dropped", "v_block_rotated", "scale_d64"]


def flash_emulate(q, k, v, heads, dtype, causal=False, mutation=None):
    """q [B, Nq, C], k / v [kvB, Nk, C] in `dtype` -> out [B, Nq, C] in `dtype`, computed as flash_attn_kernel does."""
    B, Nq, C = q.shape
    kvb, Nk, _ = k.shape
    d = C // heads
    hk = [(h + 1) % heads if mutation == "next_head_k" else h for h in range(heads)]
    qf = q.float().view(B, Nq, heads, d).transpose(1, 2)                                       # [B, h, Nq, d]
    kf = k.float().view(kvb, Nk, heads, d)[:, :, hk].transpose(1, 2).expand(B, -1, -1, -1)
    vf = v.float().view(kvb, Nk, heads, d).transpose(1, 2).expand(B, -1, -1, -1)
    nkv = (Nk + BN - 1) // BN
    # the TMA boxes zero-fill keys past Nk
    kf = torch.cat([kf, kf.new_zeros(B, heads, nkv * BN - Nk, d)], dim=2)
    vf = torch.cat([vf, vf.new_zeros(B, heads, nkv * BN - Nk, d)], dim=2)
    if mutation == "k_chunk_dropped":
        kf[..., d - 64:] = 0
    if mutation == "v_block_rotated":                                                          # halves of 256 columns
        vf = vf[..., torch.arange(d).view(-1, 4, 64).roll(-1, dims=1).reshape(-1)]
    scale = {"scale_1_over_d": 1.0 / d, "scale_d64": 1.0 / 8}.get(mutation, 1.0 / math.sqrt(d))
    sc = torch.tensor(scale * LOG2E, dtype=torch.float32)
    rows = torch.arange(Nq).view(Nq, 1)
    o = torch.zeros(B, heads, Nq, d)
    m = torch.full((B, heads, Nq, 1), -math.inf)
    l = torch.zeros(B, heads, Nq, 1)
    for j in range(nkv - 1 if mutation == "last_tile_dropped" else nkv):
        keys = torch.arange(j * BN, (j + 1) * BN).view(1, BN)
        s = qf @ kf[:, :, j * BN:(j + 1) * BN].transpose(-1, -2)                               # fp32 logits
        hidden = torch.zeros(Nq, BN, dtype=torch.bool)
        if mutation != "tail_unmasked":
            hidden |= keys >= Nk
        if causal:
            hidden |= keys > rows + (1 if mutation == "causal_one_late" else 0)
        s = s.masked_fill(hidden, -math.inf)
        mn = torch.maximum(m, s.amax(-1, keepdim=True))
        none = mn == -math.inf                                                                # no visible key yet
        f = torch.where(none, torch.ones_like(mn), torch.exp2((m - mn) * sc))
        if mutation == "no_rescale":
            f = torch.ones_like(f)
        ng = torch.where(none, torch.zeros_like(mn), -mn * sc)
        m = mn
        p = torch.exp2(s * sc + ng).to(dtype).float()                                          # P rounded to 16 bits
        l = l * f + p.sum(-1, keepdim=True)
        o = o * f + p @ vf[:, :, j * BN:(j + 1) * BN]
    return (o / l).transpose(1, 2).reshape(B, Nq, C).to(dtype)


# CPU-sized versions of the GPU matrix: (B, kvB, Nq, Nk, heads, regime, causal)
CASES = [
    (1, 1, 1, 1, 1, "flat", False),
    (2, 2, 9, 9, 2, "peaked", False),
    (2, 1, 4, 77, 2, "flat", False),
    (2, 2, 65, 65, 2, "spiky", False),
    (1, 1, 136, 129, 2, "spiky", False),
    (2, 2, 64, 200, 2, "peaked", False),
    (1, 1, 63, 65, 3, "flat", False),
    (1, 1, 40, 128, 2, "spiky", False),
    (2, 1, 20, 100, 2, "uniform", False),
    (1, 1, 72, 129, 2, "sunken", False),
    (2, 1, 8, 1000, 1, "sunken", False),
    (1, 1, 300, 300, 2, "flat", True),
    (2, 2, 129, 129, 2, "peaked", True),
    (1, 1, 65, 65, 1, "flat", True),
]
IDS = [f"b{b}_kv{kv}_q{nq}_k{nk}_h{h}_{r}{'_causal' if c else ''}" for b, kv, nq, nk, h, r, c in CASES]
DTYPES = [pytest.param(torch.bfloat16, id="bf16"), pytest.param(torch.float16, id="fp16")]


def run(case, dtype, mutation=None):
    B, kvb, Nq, Nk, heads, regime, causal = case
    q, k, v, _ = operands(B, kvb, Nq, Nk, heads, regime, dtype, device="cpu", seed=3)
    got = flash_emulate(q, k, v, heads, dtype, causal, mutation)
    ref, pav, e_s, psub = kref.attention64(q, k, v, heads, causal=causal)
    return kref.check_attention(f"{IDS[CASES.index(case)]} {mutation}", got, ref, pav, e_s, psub, Nk, dtype)


@pytest.mark.parametrize("case", CASES, ids=IDS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_emulation_passes_the_bound(dtype, case):
    c = run(case, dtype)
    print("   ", c)
    assert c, str(c)


@pytest.mark.parametrize("mutation", MUTATIONS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_every_mutation_fails_a_case(dtype, mutation):
    applies = [c for c in CASES if c[6] or mutation != "causal_one_late"]
    results = [run(c, dtype, mutation) for c in applies]
    caught = [str(r) for r in results if not r]
    print(f"\n[{mutation} {dtype}] caught by {len(caught)}/{len(results)} cases")
    for s in caught:
        print("   ", s)
    assert caught, f"{mutation}: every case passed"


def test_spike_placement():
    """The spiky regime's planted keys: first tile, last full tile, last key (a ragged tail where Nk % 64 != 0)."""
    from attn_operands import spike_keys
    assert spike_keys(129) == [5, 101, 128] and spike_keys(64) == [5, 37, 63] and spike_keys(4) == [3, 2, 3]
    q, k, _, _ = operands(1, 1, 6, 129, 2, "spiky", torch.float32, device="cpu")
    s = (q.view(6, 2, 64).transpose(0, 1) @ k.view(129, 2, 64).permute(1, 2, 0)) / 8         # [h, Nq, Nk]
    top2 = s.topk(2, dim=-1)
    assert top2.indices[..., 0].tolist() == [[5, 101, 128] * 2] * 2
    assert (top2.values[..., 0] - top2.values[..., 1]).min() > 10


# d = 512, one head: flash_attn512_kernel at the GPU matrix's key counts past the 8192-key threshold (every tail position the
# model meets there: 1, 63, whole tiles, 33, 4, 16), with the short query blocks, (B, kvB, Nq, Nk, regime)
CASES_D512 = [
    (1, 1, 8, 8193, "spiky"),
    (1, 1, 72, 8193, "sunken"),
    (2, 2, 63, 8255, "sunken"),
    (1, 1, 65, 8255, "spiky"),
    (2, 1, 64, 8256, "peaked"),
    (1, 1, 1, 8256, "uniform"),
    (1, 1, 72, 9216, "flat"),
    (1, 1, 33, 12065, "spiky"),
    (1, 1, 8, 12065, "sunken"),
    (1, 1, 72, 12100, "sunken"),
    (1, 1, 72, 14400, "peaked"),
    (1, 1, 64, 16384, "flat"),
    (1, 1, 72, 16400, "sunken"),
    (1, 1, 72, 16400, "spiky"),
]
IDS_D512 = [f"b{b}_kv{kv}_q{nq}_k{nk}_{r}" for b, kv, nq, nk, r in CASES_D512]


@functools.lru_cache(maxsize=None)
def _d512_operands(case, dtype):
    B, kvb, Nq, Nk, regime = case
    q, k, v, _ = operands(B, kvb, Nq, Nk, 1, regime, dtype, device="cpu", seed=Nq + Nk, d=512)
    return q, k, v, kref.attention64(q, k, v, 1, flash=True)


def run_d512(case, dtype, mutation=None):
    q, k, v, (ref, pav, e_s, psub) = _d512_operands(case, dtype)
    Nk = k.shape[1]
    got = flash_emulate(q, k, v, 1, dtype, mutation=mutation)
    return kref.check_attention(f"d512 {IDS_D512[CASES_D512.index(case)]} {mutation}", got, ref, pav, e_s, psub, Nk, dtype)


@pytest.mark.parametrize("case", CASES_D512, ids=IDS_D512)
@pytest.mark.parametrize("dtype", DTYPES)
def test_emulation_passes_the_bound_d512(dtype, case):
    c = run_d512(case, dtype)
    print("   ", c)
    assert c, str(c)


@pytest.mark.parametrize("mutation", MUTATIONS_D512)
@pytest.mark.parametrize("dtype", DTYPES)
def test_every_mutation_fails_a_case_d512(dtype, mutation):
    results = [run_d512(c, dtype, mutation) for c in CASES_D512]
    caught = [str(r) for r in results if not r]
    print(f"\n[d512 {mutation} {dtype}] caught by {len(caught)}/{len(results)} cases")
    for s in caught:
        print("   ", s)
    assert caught, f"{mutation}: every case passed"


def test_spike_and_sink_logits_d512():
    """At d = 512 the planted key sits about 30 logits above the rest, and the sunken regime puts every real logit near
    -11.3, below the logit 0 of a zero-filled key."""
    q, k, _, _ = operands(1, 1, 6, 8255, 1, "spiky", torch.float32, device="cpu", d=512)
    s = (q[0] @ k[0].T) / math.sqrt(512)
    top2 = s.topk(2, dim=-1)
    assert top2.indices[:, 0].tolist() == [5, 8165, 8254] * 2
    assert (top2.values[:, 0] - top2.values[:, 1]).min() > 15 and (top2.values[:, 0] - 29.7).abs().max() < 10
    q, k, _, _ = operands(1, 1, 6, 8255, 1, "sunken", torch.bfloat16, device="cpu", d=512)
    s = (q[0].double() @ k[0].double().T) / math.sqrt(512)
    assert (s.mean() + 11.3).abs() < 0.1 and s.max() < -4


# 190512 keys (UNet level 0, and the VAE attention, of a 4032x3024 image), 32 query rows: the per-element bound's Nk * 2^-24
# term is about the size of the output here, so the large GPU cases also cap the mean-ulp statistic; the cap must pass the
# emulated kernel and fail these mutations and an all-zero output.  The unmasked tail is checked under the sunken regime:
# with flat logits its 16 zero keys of 190512 move the output by 8e-5 of itself, under a sixth of an fp16 ulp, while sunken
# logits give the zero keys most of the weight.  Not listed: the causal mask (the large cases are not causal), and at d = 512
# the chunk and block mutations, which the smaller cases above catch.
LARGE_MUTATIONS = {64: ["no_rescale", "last_tile_dropped", "next_head_k", "scale_1_over_d"],
                   512: ["no_rescale", "last_tile_dropped", "scale_d64"]}
LARGE_HEADS = {64: 2, 512: 1}
_LARGE = {}


def _large(d, regime, dtype):
    """(q, k, v, float64 reference) of the 190512-key case at head dim d, built once per module."""
    key = (d, regime, dtype)
    if key not in _LARGE:
        q, k, v, _ = operands(1, 1, 32, 190512, LARGE_HEADS[d], regime, dtype, device="cpu", seed=4, d=d)
        _LARGE[key] = (q, k, v, kref.attention64(q, k, v, LARGE_HEADS[d], flash=True))
    return _LARGE[key]


def _large_check(d, dtype, mutation=None, zero=False, regime="flat"):
    q, k, v, (ref, pav, e_s, psub) = _large(d, regime, dtype)
    got = torch.zeros_like(q) if zero else flash_emulate(q, k, v, LARGE_HEADS[d], dtype, mutation=mutation)
    what = mutation or ("zero" if zero else "emulated")
    return kref.check_attention(f"d{d} k190512 {regime} {what} {dtype}", got, ref, pav, e_s, psub, k.shape[1], dtype,
                                kref.ATTN_MEAN_ULP_MAX)


def _separates(d, dtype):
    good = [_large_check(d, dtype), _large_check(d, dtype, regime="sunken")]
    bad = [_large_check(d, dtype, m) for m in LARGE_MUTATIONS[d]] + [_large_check(d, dtype, zero=True),
                                                                     _large_check(d, dtype, "tail_unmasked", regime="sunken")]
    for c in good + bad:
        print("   ", c)
    assert all(good), [str(c) for c in good if not c]
    assert not any(bad), [str(c) for c in bad if c]


@pytest.mark.parametrize("dtype", DTYPES)
def test_large_key_count_cap_separates_mutations(dtype):
    _separates(64, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_large_key_count_cap_separates_mutations_d512(dtype):
    _separates(512, dtype)
