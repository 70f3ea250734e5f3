"""CPU proof that the d = 64 attention matrix of tests/test_gpu_attention.py would catch a wrong kernel.

`flash_emulate` repeats flash_attn_kernel's arithmetic (csrc/flash.cuh) in torch: 64-key tiles, fp32 logits, a running
maximum in raw logit units with exp2 at scale * log2(e), P rounded to the activation dtype with l summed over the ROUNDED P,
the rescale of O and l by exp2((m_old - m_new) * scale * log2(e)), the causal and ragged-tail masks, one final rounding.
It passes kref.check_attention on CPU-sized versions of the GPU cases; each mutation below (one plausible kernel bug) must
fail at least one of them, so a kernel with that bug could not pass the GPU suite either."""
import math

import pytest
import torch

import kref
from attn_operands import operands

BN = 64
LOG2E = 1.4426950408889634
MUTATIONS = ["no_rescale", "tail_unmasked", "last_tile_dropped", "causal_one_late", "next_head_k", "scale_1_over_d"]


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
    scale = 1.0 / d if mutation == "scale_1_over_d" else 1.0 / math.sqrt(d)
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


# 190512 keys (UNet level 0 of a 4032x3024 image), 32 query rows, 2 heads: the per-element bound's Nk * 2^-24 term is about
# the size of the output here, so the large GPU cases also cap the mean-ulp statistic; the cap must pass the emulated
# kernel and fail these mutations and an all-zero output.  Not listed: the causal mask (the large cases are not causal), and
# the unmasked tail, whose 16 zero keys of 190512 move the output by 8e-5 of itself, under a sixth of an fp16 ulp (the
# small cases above catch it).
LARGE_MUTATIONS = ["no_rescale", "last_tile_dropped", "next_head_k", "scale_1_over_d"]


@pytest.fixture(scope="module")
def large_case():
    Nk = 190512
    out = {}
    for dtype in (torch.bfloat16, torch.float16):
        q, k, v, _ = operands(1, 1, 32, Nk, 2, "flat", dtype, device="cpu", seed=4)
        out[dtype] = (q, k, v, kref.attention64(q, k, v, 2, flash=True))
    return out


def _large_check(large_case, dtype, mutation=None, zero=False):
    q, k, v, (ref, pav, e_s, psub) = large_case[dtype]
    got = torch.zeros_like(q) if zero else flash_emulate(q, k, v, 2, dtype, mutation=mutation)
    return kref.check_attention(f"k190512 {mutation or ('zero' if zero else 'emulated')} {dtype}", got, ref, pav, e_s, psub,
                                k.shape[1], dtype, kref.ATTN_MEAN_ULP_MAX)


@pytest.mark.parametrize("dtype", DTYPES)
def test_large_key_count_cap_separates_mutations(large_case, dtype):
    good = _large_check(large_case, dtype)
    bad = [_large_check(large_case, dtype, m) for m in LARGE_MUTATIONS] + [_large_check(large_case, dtype, zero=True)]
    for c in [good] + bad:
        print("   ", c)
    assert good, str(good)
    assert not any(bad), [str(c) for c in bad if c]
