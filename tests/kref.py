"""Float64 references of the engine's single ops and the per-element acceptance criterion the kernel tests apply.

The references take the same 16-bit-rounded operands the kernel sees and compute in float64; the bounds are what the
engine's arithmetic (DESIGN section 4: fp32 accumulation, one rounding per layer output) can legitimately add on top of
that, element by element, so a localised error (one tile, one group, one key) is not averaged away:

  GEMM family   |got - ref| <= ulp16(ref) + f * K * 2^-24 * mag        mag: the op on |x|, |w|, |bias|, |res|; K: reduction
                mean|got - ref| / mean ulp16(ref) <= 0.30              (a single correct rounding lands near 0.25)
  attention     |got - ref| <= ulp16(ref) + (2u + e_s + Nk * 2^-24) * (P @ |V|) + eta * sub     P: the exact softmax
                mean|got - ref| / mean ulp16(ref) <= 0.75 where the caller asks for it (large key counts)
  norms         |got - ref| <= ulp16(ref) + c * 2^-20 * ((1 + k^2) |xh g| + (1 + k) |g| + |b|)    k = |mean| / std

ulp16(y) is the spacing of the engine dtype at |y|; u its unit roundoff (2^-8 bf16, 2^-11 fp16).
Attention's eta * sub: both attention paths round probabilities of at most 1 to 16 bits (normalised to the running
maximum in the flash kernels, to the row sum in the unfused softmax), and below the dtype's normal range that rounding is
absolute, not relative: up to eta = 2^-25 per element in fp16 (half its subnormal spacing 2^-24), 2^-126 in bf16
(ex2.approx.ftz flushes fp32 denormals).  Only keys whose rounded probability can be subnormal pay it: in a flash kernel
exp(s_j - m_running) >= exp(s_j - max s), in the unfused softmax p_j itself, so the set S is exp(s_j - max s) < 2^-13 for a
flash path and p_j < 2^-13 otherwise (fp16's smallest normal 2^-14, doubled for the fp32 logit and exp2 errors; the p_j
set contains the other, so it is the default where the path is not known).  Each such key moves the numerator by
eta |V_j|, and, in the flash kernels, the row sum l by eta, which moves the output by eta |out| / l <= eta |out|:
sub = sum_{j in S} |V_j| + |S| |out|.  Where the row's weight sits on a key whose V column is small and the other keys carry
|V| ~ 1, P @ |V| does not cover these errors.
The attention bound's Nk * 2^-24 term (the fp32 P V chain's worst case) is 1.1 % of P @ |V| at 190512 keys, about the size of
the output itself, so there the per-element bound alone would pass a dropped KV tile or an all-zero output.  Those checks
also cap the mean-ulp statistic at 0.75: a correct 16-bit rounding lands near 0.25 and the flash kernel's fp32 chains over
190512 keys measure 0.40 (bf16) to 0.49 (fp16) on an H100, while one dropped KV tile already gives several ulps on average;
the d = 512 flash kernel measures the same (0.41 and 0.50 at 190512 keys).  The cap does not hold on the unfused path in
fp16 past about 16384 keys, and is not applied there: its probabilities are relative to the row sum, p_j ~ 1 / Nk falls below
fp16's smallest normal 2^-14, and each then carries an absolute rounding error up to 2^-25, several percent of itself.  The
per-element bound covers that through eta * sub, but the mean error grows with Nk: 0.60 ulp at 32400 keys, 1.03 at 65536,
2.88 at 190512 (H100, d = 512, I2IT_NO_FLASH).  The model runs that path only up to 8192 keys, where p_j stays normal.
Everything here runs on CPU or GPU tensors alike.
"""
import math

import torch
import torch.nn.functional as F

_MANT = {torch.bfloat16: 7, torch.float16: 10, torch.float32: 23, torch.float64: 52}      # float64: rounding switched off
_EMIN = {torch.bfloat16: -126, torch.float16: -14, torch.float32: -126, torch.float64: -1022}
EPS24 = 2.0 ** -24                       # fp32 unit roundoff
MEAN_ULP_MAX = 0.30
ATTN_MEAN_ULP_MAX = 0.75                 # attention at large key counts (header)
# Norm statistics: sums of x and x^2 run in fp32 chains before the double finalisation, so var = E[x^2] - mean^2 carries
# a relative error of about L * 2^-24 * (1 + k^2) for a chain of L terms, and the fp32 apply x * (rstd g) + (b - mean rstd g)
# adds a few 2^-24 of (|xh| + 2k) |g| + |b|.  c * 2^-20 = 16 * 2^-20 = 2^-16 is 256 * 2^-24: the worst case of chains up to
# ~170 terms (epilogue slots sum 32 rows; gn_stats chains are longer but add errors of random sign, ~sqrt(L)) times 1.5 for
# the square root, with the SiLU approximations (ex2.approx, __fdividef: a few 2^-24 relative) inside the same margin.
NORM_C = 16.0


def unit_roundoff(dtype):
    return 2.0 ** -(_MANT[dtype] + 1)


def ulp16(y, dtype):
    """Spacing of `dtype` at |y| (float64 tensor), subnormal spacing below the normal range."""
    a = y.detach().double().abs()
    _, e = torch.frexp(a)
    e = torch.where(a > 0, e - 1, torch.full_like(e, _EMIN[dtype])).clamp(min=_EMIN[dtype])
    return torch.ldexp(torch.ones_like(a), (e - _MANT[dtype]).to(torch.int32))


def round16(y, dtype):
    return y.to(dtype).double()


class Check:
    """Result of one comparison: worst err/bound, mean-ulp statistic, where it failed."""

    def __init__(self, name, got, ref, bound, dtype, mean_ulp_max=None):
        got, ref, bound = got.detach().double(), ref.detach().double(), bound.detach().double()
        assert got.shape == ref.shape == bound.shape, (got.shape, ref.shape, bound.shape)
        err = (got - ref).abs()
        ratio = err / bound
        self.name = name
        self.finite = bool(torch.isfinite(got).all())
        self.worst = float(ratio.max()) if ratio.numel() else 0.0
        self.mean_ulp = float(err.mean() / ulp16(ref, dtype).mean()) if err.numel() else 0.0
        self.mean_ulp_max = mean_ulp_max
        self.n_bad = int((ratio > 1).sum())
        self.numel = err.numel()
        self.where = (ratio > 1).nonzero()[:4].tolist()
        self.ok = self.finite and self.n_bad == 0 and (mean_ulp_max is None or self.mean_ulp <= mean_ulp_max)

    def __bool__(self):
        return self.ok

    def __str__(self):
        lim = f"/{self.mean_ulp_max:.2f}" if self.mean_ulp_max is not None else ""
        return (f"{'PASS' if self.ok else 'FAIL'} [{self.name}] worst err/bound={self.worst:.3f} mean_ulp={self.mean_ulp:.3f}{lim} "
                f"bad={self.n_bad}/{self.numel}" + (f" at {self.where}" if self.n_bad else ""))


# ---------------------------------------------------------------------------------------------------------------------
# GEMM family
# ---------------------------------------------------------------------------------------------------------------------
def conv64(x_nhwc, w, bias=None, stride=1, asym=False, up2x=False):
    """float64 conv of NHWC activations with a PyTorch-layout weight -> NCHW float64.  Also used on |x|, |w| for mag."""
    x = x_nhwc.double().permute(0, 3, 1, 2)
    if up2x:
        x = F.interpolate(x, scale_factor=2.0, mode="nearest")
    k = w.shape[-1]
    w = w.double()
    b = bias.double() if bias is not None else None
    if asym:
        return F.conv2d(F.pad(x, (0, 1, 0, 1)), w, b, stride=stride)
    return F.conv2d(x, w, b, stride=stride, padding=k // 2)


def subpixel_weights(w, dtype):
    """The 16 pre-summed 2x2 taps the sub-pixel up-conv multiplies, [phase(py,px)][ty][tx] -> [4, Cout, Cin, 2, 2]: per
    parity, the 3x3 taps that land on the same low-res pixel summed in fp32 from the fp32 weights and rounded once."""
    w = w if w.dtype == torch.float64 else w.float()
    # rows of the 3x3 kernel that fold onto low-res offset (ty) for output parity p: p=0 -> {0}, {1,2}; p=1 -> {0,1}, {2}
    fold = {0: ([0], [1, 2]), 1: ([0, 1], [2])}
    out = torch.empty(4, w.shape[0], w.shape[1], 2, 2, dtype=w.dtype, device=w.device)
    for py in (0, 1):
        for px in (0, 1):
            for ty in (0, 1):
                for tx in (0, 1):
                    s = torch.zeros_like(w[:, :, 0, 0])
                    for ky in fold[py][ty]:
                        for kx in fold[px][tx]:
                            s = s + w[:, :, ky, kx]
                    out[py * 2 + px, :, :, ty, tx] = s
    return out.to(dtype).double()


def subpixel_conv64(x_nhwc, wsub, bias=None):
    """float64 sub-pixel up-conv with pre-summed taps `wsub` [4, Cout, Cin, 2, 2] -> NCHW at 2x resolution."""
    x = x_nhwc.double().permute(0, 3, 1, 2)
    N, _, H, W = x.shape
    out = torch.empty(N, wsub.shape[1], 2 * H, 2 * W, dtype=torch.float64, device=x.device)
    xp = F.pad(x, (1, 1, 1, 1))
    for py in (0, 1):
        for px in (0, 1):
            # output (2y+py, 2x+px) reads low-res rows y-1+py .. y+py, cols x-1+px .. x+px
            win = xp[:, :, py:py + H + 1, px:px + W + 1]
            out[:, :, py::2, px::2] = F.conv2d(win, wsub[py * 2 + px].double(), bias.double() if bias is not None else None)
    return out


def gemm_bound(ref, mag, K, dtype, factor=1.0):
    """ulp16(ref) + factor * K * 2^-24 * mag.  factor covers an epilogue's derivative (GELU' <= 1.13 -> 2)."""
    return ulp16(ref, dtype) + factor * K * EPS24 * mag


def check_gemm(name, got, ref, mag, K, dtype, factor=1.0, out_fp32=False):
    """Per-element bound plus the mean-ulp aggregate (per-element only, with fp32's ulp, for fp32 outputs)."""
    if out_fp32:
        return Check(name, got, ref, gemm_bound(ref, mag, K, torch.float32, factor), torch.float32)
    return Check(name, got, ref, gemm_bound(ref, mag, K, dtype, factor), dtype, MEAN_ULP_MAX)


def gelu64(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def quick_gelu64(x):
    return x * torch.sigmoid(1.702 * x)


# ---------------------------------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------------------------------
P_FLOOR = {torch.bfloat16: 2.0 ** -126, torch.float16: 2.0 ** -25}     # absolute rounding error of a probability <= 1
SUBNORMAL_P = 2.0 ** -13                 # fp16's smallest normal 2^-14, doubled for the fp32 logit and exp2 errors


def attention64(q, k, v, heads, causal=False, flash=False):
    """Exact float64 softmax attention.  q [B,Nq,C], k/v [kvB,Nk,C] (kvB 1 or B)
    -> (out [B,Nq,C], P @ |V|, logit error, sub: what subnormal probabilities can move per unit of eta (header)).
    flash=True: the result comes from a flash kernel, whose probabilities are relative to the row maximum."""
    B, Nq, C = q.shape
    kvb, Nk, _ = k.shape
    d = C // heads
    qf = q.double().view(B, Nq, heads, d).transpose(1, 2)
    kf = k.double().view(kvb, Nk, heads, d).transpose(1, 2).expand(B, -1, -1, -1)
    vf = v.double().view(kvb, Nk, heads, d).transpose(1, 2).expand(B, -1, -1, -1)
    s = qf @ kf.transpose(-1, -2) / math.sqrt(d)
    smag = qf.abs() @ kf.abs().transpose(-1, -2) / math.sqrt(d)
    if causal:
        mask = torch.ones(Nq, Nk, dtype=torch.bool, device=q.device).triu(1)
        s = s.masked_fill(mask, float("-inf"))
        smag = smag.masked_fill(mask, 0.0)
    p = torch.softmax(s, dim=-1)
    of = p @ vf
    o = of.transpose(1, 2).reshape(B, Nq, C)
    pav = (p @ vf.abs()).transpose(1, 2).reshape(B, Nq, C)
    small = (torch.exp(s - s.amax(-1, keepdim=True)) if flash else p) < SUBNORMAL_P
    if causal:
        small &= ~mask
    small = small.double()
    sub = (small @ vf.abs() + small.sum(-1, keepdim=True) * of.abs()).transpose(1, 2).reshape(B, Nq, C)
    # fp32 logits carry d * 2^-24 * |q||k| of accumulation error; P moves by at most twice the row's largest
    e_s = (2 * d * EPS24 * smag.amax(-1, keepdim=True)).expand(-1, -1, -1, d).transpose(1, 2).reshape(B, Nq, C)
    return o, pav, e_s, sub


def check_attention(name, got, ref, pav, e_s, sub, Nk, dtype, mean_ulp_max=None):
    """P rounded to 16 bits relative to the running maximum (u, twice: numerator and denominator), logit error, fp32 PV,
    and the absolute rounding of probabilities below the dtype's normal range; optionally the mean-ulp cap."""
    bound = ulp16(ref, dtype) + (2 * unit_roundoff(dtype) + e_s + Nk * EPS24) * pav + P_FLOOR[dtype] * sub
    return Check(name, got, ref, bound, dtype, mean_ulp_max)


# ---------------------------------------------------------------------------------------------------------------------
# GroupNorm / LayerNorm
# ---------------------------------------------------------------------------------------------------------------------
def _norm_bound(ref, xh, kappa, gamma, beta, dtype, silu, two_pass):
    k2 = torch.zeros_like(kappa) if two_pass else kappa * kappa
    mag = (1 + k2) * (xh * gamma).abs() + (1 + kappa) * gamma.abs() + beta.abs()
    return ulp16(ref, dtype) + NORM_C * 2.0 ** -20 * mag * (1.1 if silu else 1.0)


def group_norm64(x_nhwc, gamma, beta, eps, silu, dtype, groups=32):
    """GroupNorm(+SiLU) of the engine's own 16-bit input, in float64 -> (ref NHWC, bound NHWC)."""
    x = x_nhwc.double()
    N, H, W, C = x.shape
    xg = x.reshape(N, H * W, groups, C // groups)
    mean = xg.mean(dim=(1, 3), keepdim=True)
    var = ((xg - mean) ** 2).mean(dim=(1, 3), keepdim=True)
    xh = ((xg - mean) / torch.sqrt(var + eps)).reshape(N, H, W, C)
    kappa = (mean.abs() / torch.sqrt(var + eps)).expand_as(xg).reshape(N, H, W, C)
    g, b = gamma.double().view(1, 1, 1, C), beta.double().view(1, 1, 1, C)
    y = xh * g + b
    ref = y * torch.sigmoid(y) if silu else y
    bound = _norm_bound(ref, xh, kappa, g.expand_as(xh), b.expand_as(xh), dtype, silu, two_pass=False)
    return ref, bound


def layer_norm64(x, gamma, beta, eps, dtype):
    """LayerNorm over the last dim of the engine's 16-bit input, float64 (the kernel is two-pass: no E[x^2] - mean^2)."""
    xd = x.double()
    mean = xd.mean(-1, keepdim=True)
    var = ((xd - mean) ** 2).mean(-1, keepdim=True)
    xh = (xd - mean) / torch.sqrt(var + eps)
    kappa = (mean.abs() / torch.sqrt(var + eps)).expand_as(xh)
    g, b = gamma.double().expand_as(xh), beta.double().expand_as(xh)
    ref = xh * g + b
    return ref, _norm_bound(ref, xh, kappa, g, b, dtype, False, two_pass=True)


def check_norm(name, got, ref, bound, dtype):
    return Check(name, got, ref, bound, dtype)


# ---------------------------------------------------------------------------------------------------------------------
# prepared weights
# ---------------------------------------------------------------------------------------------------------------------
def check_weights(name, got, ref64, dtype, max_unequal=0.01, fold_err=None):
    """Weights read back from the engine against round16(float64 fold): every element within one weight ulp, and at most
    `max_unequal` of them not bit-equal (an fp32 fold rounds differently from float64 only next to a rounding tie).
    `fold_err` (per element) adds the fp32 fold's own error, n * 2^-24 * (|W| + sum |s| |B| |A|): where W and the LoRA
    term cancel, a result near zero is many 16-bit ulps of itself away from the float64 fold."""
    ref16 = round16(ref64, dtype)
    bound = ulp16(ref16, dtype) if fold_err is None else ulp16(ref16, dtype) + fold_err
    c = Check(name, got, ref16, bound, dtype)
    c.unequal = float((got.double() != ref16).double().mean())
    c.ok = c.ok and c.unequal <= max_unequal
    return c
