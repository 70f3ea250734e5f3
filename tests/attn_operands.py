"""Operands of the d = 64 attention tests, laid out as the model hands them to the kernel, in four logit regimes.

  layout "slice"   Q and K are column slices [..., :C] and [..., C:] of one [B, N, 2C] projection (the self-attention and the
                   CLIP tower's fused to_q / to_k output).  Where Nq != Nk or K is shared, Q and K come from two such buffers
                   and the half nobody should read is NaN.
  layout "dense"   contiguous Q [B, Nq, C] and K [kvB, Nk, C] (cross-attention: to_q output, text K)
  V^T              [kvB, C, ldv] with ldv = round_up(Nk, 8) + 8; the padding columns [Nk, ldv) are NaN

  regime "flat"     q, k, v ~ N(0, 1): logits of std ~1
  regime "peaked"   q scaled x4: logits of std ~4, the running maximum moves from tile to tile
  regime "spiky"    rows r = 0, 1, 2 (mod 3) each get one planted key about 30 logits above the rest: in the first 64-key tile,
                    in the last full tile, and at key Nk - 1 (the ragged tail where Nk % 64 != 0), so the maximum moves late
  regime "uniform"  every key identical: P = 1 / Nk exactly
"""
import torch

D = 64
SPIKE_Q, SPIKE_K = 8.0, 30.0             # planted logit (8 + z) * 30 / sqrt(64) = 30 + 3.75 z; both exact in bf16 and fp16


def spike_keys(Nk):
    """Planted key of rows r = 0, 1, 2 (mod 3): first tile, last full tile, last key."""
    first = min(5, Nk - 1)
    last_full = (Nk // 64 - 1) * 64 + 37 if Nk >= 64 else Nk // 2
    return [first, last_full, Nk - 1]


def padded_vt(v, nan=True):
    """V [kvB, Nk, C] -> V^T [kvB, C, round_up(Nk, 8) + 8], padding columns NaN (or zero)."""
    kvb, Nk, C = v.shape
    ldv = (Nk + 7) // 8 * 8 + 8
    vt = torch.full((kvb, C, ldv), float("nan") if nan else 0.0, device=v.device, dtype=v.dtype)
    vt[:, :, :Nk] = v.transpose(1, 2)
    return vt


def operands(B, kvb, Nq, Nk, heads, regime, dtype, device="cuda", layout="dense", seed=0):
    """-> q [B, Nq, C], k [kvB, Nk, C], v [kvB, Nk, C] (dense), vt (NaN-padded V^T).  q and k are views for layout "slice"."""
    C = heads * D
    g = torch.Generator(device=device).manual_seed(seed)
    q = torch.randn(B, Nq, C, device=device, generator=g)
    k = torch.randn(kvb, Nk, C, device=device, generator=g)
    v = torch.randn(kvb, Nk, C, device=device, generator=g)
    if regime == "peaked":
        q *= 4
    elif regime == "uniform":
        k = k[:, :1].expand(kvb, Nk, C).clone()
    elif regime == "spiky":
        for grp, key in enumerate(spike_keys(Nk)):
            cols = torch.arange(heads, device=device) * D + grp          # coordinate grp of every head
            k[:, key, cols] = SPIKE_K
            q[:, grp::3, cols] += SPIKE_Q
    else:
        assert regime == "flat", regime
    q, k, v = q.to(dtype), k.to(dtype), v.to(dtype)
    if layout == "slice":
        if Nq == Nk and kvb == B:
            qk = torch.cat([q, k], dim=2)
            q, k = qk[..., :C], qk[..., C:]
        else:
            nan = torch.full_like(q, float("nan"))
            q = torch.cat([q, nan], dim=2)[..., :C]
            k = torch.cat([torch.full_like(k, float("nan")), k], dim=2)[..., C:]
    else:
        assert layout == "dense", layout
    return q, k, v, padded_vt(v)
