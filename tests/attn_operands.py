"""Operands of the attention tests, laid out as the model hands them to the kernel, in five logit regimes.

Head dim d = 64 (every UNet self- and cross-attention layer, the CLIP text tower) or d = 512 (the VAE mid-block: one head).

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
  regime "sunken"   flat, with coordinate 3 of every head (one the spikes do not use) set to q = +16, k = -16: every real logit
                    moves by -256 / sqrt(d) (-32 at d = 64, -11.3 at d = 512), well below 0.  A zero-filled key past Nk has
                    logit exactly 0, so an unmasked tail outweighs every real key and pulls the output toward zero at any Nk.
"""
import torch

D = 64
# planted logit (q_spike + z) * k_spike / sqrt(d), about 30; every value is exact in bf16 and fp16
SPIKE = {64: (8.0, 30.0),                # (8 + z) * 30 / 8 = 30 + 3.75 z
         512: (16.0, 42.0)}              # (16 + z) * 42 / sqrt(512) = 29.7 + 1.86 z
SINK_COL, SINK = 3, 16.0                 # the sunken regime's coordinate and |q| = |k| on it


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


def operands(B, kvb, Nq, Nk, heads, regime, dtype, device="cuda", layout="dense", seed=0, d=D):
    """-> q [B, Nq, C], k [kvB, Nk, C], v [kvB, Nk, C] (dense), vt (NaN-padded V^T).  q and k are views for layout "slice".
    C = heads * d.  The generator draws q, k, v in that order whatever the regime, so each d = 64 call gives the tensors it
    always gave."""
    C = heads * d
    g = torch.Generator(device=device).manual_seed(seed)
    q = torch.randn(B, Nq, C, device=device, generator=g)
    k = torch.randn(kvb, Nk, C, device=device, generator=g)
    v = torch.randn(kvb, Nk, C, device=device, generator=g)
    if regime == "peaked":
        q *= 4
    elif regime == "uniform":
        k = k[:, :1].expand(kvb, Nk, C).clone()
    elif regime == "spiky":
        sq, sk = SPIKE[d]
        for grp, key in enumerate(spike_keys(Nk)):
            cols = torch.arange(heads, device=device) * d + grp          # coordinate grp of every head
            k[:, key, cols] = sk
            q[:, grp::3, cols] += sq
    elif regime == "sunken":
        cols = torch.arange(heads, device=device) * d + SINK_COL
        q[:, :, cols] = SINK
        k[:, :, cols] = -SINK
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
