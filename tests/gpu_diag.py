"""GPU bring-up diagnostics: each case checks one libi2it kernel path against plain torch fp32 on the same
(16-bit-rounded) inputs and prints an error summary instead of asserting.  Run one case per process so a
trapped kernel cannot poison the others:   python tests/gpu_diag.py <case>|list|all
"""
import os
import sys
import math

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "img2img-turbo_b200"))
import i2it  # noqa: E402

torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False


def report(name, got, ref, tol):
    got, ref = got.float(), ref.float()
    err = (got - ref).abs()
    scale = ref.abs().max().item() + 1e-12
    bad = err > tol * scale
    msg = (f"[{name}] max_abs_err={err.max().item():.4e} ref_max={scale:.4e} rel={err.max().item()/scale:.3e} "
           f"mean_err={err.mean().item():.3e} bad={bad.sum().item()}/{bad.numel()}")
    ok = bad.sum().item() == 0 and math.isfinite(err.max().item())
    print(("PASS " if ok else "FAIL ") + msg, flush=True)
    if not ok:
        idx = bad.nonzero()[:8].tolist()
        for i in idx:
            print("   at", i, "got", got[tuple(i)].item(), "ref", ref[tuple(i)].item())
        # structure of the error: per leading / trailing dim
        if got.dim() >= 2:
            flat = bad.reshape(-1, bad.shape[-1])
            print("   bad cols (first 32):", flat.any(0).nonzero().flatten()[:32].tolist())
            print("   bad rows (first 32):", flat.any(1).nonzero().flatten()[:32].tolist())
    return ok


def mk(dtype, *shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(dtype)


def case_linear(dtype, M, K, N, bias=True, res=False, tag=""):
    E = i2it.Engine(dtype, use_cuda_graph=False)
    x = mk(dtype, 1, 1, M, K, seed=1)
    w = mk(torch.float32, N, K, 1, 1, scale=1 / math.sqrt(K), seed=2).to(dtype).float()
    b = mk(torch.float32, N, seed=3) if bias else None
    r = mk(dtype, 1, 1, M, N, seed=4) if res else None
    y = E.op_conv2d(x, w, b, residual=r)
    ref = F.linear(x.float().view(M, K), w.view(N, K), b)
    if res:
        ref = ref + r.float().view(M, N)
    return report(f"linear{tag} {dtype} M={M} K={K} N={N} bias={bias} res={res}", y.view(M, N), ref,
                  6e-3 if dtype == torch.bfloat16 else 1.5e-3)


def case_conv(dtype, N, H, W, Cin, Cout, k=3, stride=1, asym=False, res=False, act=i2it.ACT_NONE, out_fp32=False):
    E = i2it.Engine(dtype, use_cuda_graph=False)
    x = mk(dtype, N, H, W, Cin, seed=1)
    w = mk(torch.float32, Cout, Cin, k, k, scale=1 / math.sqrt(Cin * k * k), seed=2).to(dtype).float()
    b = mk(torch.float32, Cout, seed=3)
    oc = Cout // 2 if act == i2it.ACT_GEGLU else Cout
    r = mk(dtype, N, H // stride, W // stride, oc, seed=4) if res else None
    y = E.op_conv2d(x, w, b, stride=stride, asym_pad=asym, residual=r, act=act, out_fp32=out_fp32)
    xin = x.float().permute(0, 3, 1, 2)
    if stride == 2 and asym:
        ref = F.conv2d(F.pad(xin, (0, 1, 0, 1)), w, b, stride=2)
    else:
        ref = F.conv2d(xin, w, b, stride=stride, padding=k // 2)
    if act == i2it.ACT_GEGLU:
        hh, gg = ref.chunk(2, dim=1)
        ref = hh * F.gelu(gg)
    if res:
        ref = ref + r.float().permute(0, 3, 1, 2)
    if act == i2it.ACT_CLAMP1:
        ref = ref.clamp(-1, 1)
    return report(f"conv {dtype} N={N} {H}x{W} {Cin}->{Cout} k={k} s={stride} asym={asym} res={res} act={act} f32={out_fp32}",
                  y.float().permute(0, 3, 1, 2), ref, 6e-3 if dtype == torch.bfloat16 else 1.5e-3)


def case_gn(dtype, N, H, W, C, silu, eps=1e-6):
    E = i2it.Engine(dtype, use_cuda_graph=False)
    x = (mk(dtype, N, H, W, C, seed=1).float() * 1.7 + 0.3).to(dtype)
    g = mk(torch.float32, C, seed=2) * 0.2 + 1
    b = mk(torch.float32, C, seed=3) * 0.1
    y = E.op_group_norm(x, g, b, eps, silu)
    ref = F.group_norm(x.float().permute(0, 3, 1, 2), 32, g, b, eps)
    if silu:
        ref = F.silu(ref)
    return report(f"groupnorm {dtype} N={N} {H}x{W} C={C} silu={silu}", y.float().permute(0, 3, 1, 2), ref,
                  6e-3 if dtype == torch.bfloat16 else 1.5e-3)


def case_ln(dtype, rows, C):
    E = i2it.Engine(dtype, use_cuda_graph=False)
    x = (mk(dtype, rows, C, seed=1).float() * 2 - 0.5).to(dtype)
    g = mk(torch.float32, C, seed=2) * 0.2 + 1
    b = mk(torch.float32, C, seed=3) * 0.1
    y = E.op_layer_norm(x, g, b)
    ref = F.layer_norm(x.float(), (C,), g, b, 1e-5)
    return report(f"layernorm {dtype} rows={rows} C={C}", y, ref, 6e-3 if dtype == torch.bfloat16 else 1.5e-3)


def case_attn(dtype, B, Nq, Nk, heads, d, kvb=None):
    kvb = kvb or B
    E = i2it.Engine(dtype, use_cuda_graph=False)
    C = heads * d
    q = mk(dtype, B, Nq, C, seed=1)
    k = mk(dtype, kvb, Nk, C, seed=2)
    v = mk(dtype, kvb, Nk, C, seed=3)
    ldv = (Nk + 7) // 8 * 8
    vt = torch.zeros(kvb, C, ldv, device="cuda", dtype=dtype)
    vt[:, :, :Nk] = v.transpose(1, 2)
    y = E.op_attention(q, k, vt, heads)
    qf = q.float().view(B, Nq, heads, d).transpose(1, 2)
    kf = k.float().view(kvb, Nk, heads, d).transpose(1, 2).expand(B, -1, -1, -1)
    vf = v.float().view(kvb, Nk, heads, d).transpose(1, 2).expand(B, -1, -1, -1)
    p = torch.softmax(qf @ kf.transpose(-1, -2) / math.sqrt(d), dim=-1)
    ref = (p.to(dtype).float() @ vf).transpose(1, 2).reshape(B, Nq, C)
    return report(f"attention {dtype} B={B} Nq={Nq} Nk={Nk} heads={heads} d={d} kvb={kvb}", y, ref,
                  1e-2 if dtype == torch.bfloat16 else 3e-3)


def case_up(dtype):
    E = i2it.Engine(dtype, use_cuda_graph=False)
    x = mk(dtype, 2, 8, 8, 64, seed=1)
    y = E.op_upsample2x(x)
    ref = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest")
    return report("upsample2x", y.float().permute(0, 3, 1, 2), ref, 0.0 + 1e-9)


bf, hf = torch.bfloat16, torch.float16
CASES = {
    "lin_small": lambda: case_linear(bf, 128, 64, 64, bias=False),
    "lin_k2": lambda: case_linear(bf, 128, 128, 64, bias=False),
    "lin_n256": lambda: case_linear(bf, 256, 256, 256),
    "lin_ragged": lambda: case_linear(bf, 1000, 320, 320, res=True),
    "lin_wide": lambda: case_linear(hf, 4096, 320, 2560),
    "lin_tiny_n": lambda: case_linear(bf, 512, 512, 8),
    "lin_f16": lambda: case_linear(hf, 300, 1280, 640, res=True),
    "conv_basic": lambda: case_conv(bf, 2, 16, 16, 64, 128),
    "conv_320": lambda: case_conv(bf, 1, 32, 32, 320, 320, res=True),
    "conv_8x8": lambda: case_conv(hf, 3, 8, 8, 128, 256),
    "conv_cin8": lambda: case_conv(bf, 2, 32, 32, 8, 128),
    "conv_cout4": lambda: case_conv(bf, 2, 16, 16, 128, 4),
    "conv_big": lambda: case_conv(bf, 1, 128, 128, 128, 128),
    "conv_s2_sym": lambda: case_conv(bf, 2, 32, 32, 64, 64, stride=2),
    "conv_s2_asym": lambda: case_conv(hf, 2, 32, 32, 128, 128, stride=2, asym=True),
    "conv_1x1": lambda: case_conv(bf, 2, 16, 16, 128, 256, k=1, res=True),
    "conv_geglu": lambda: case_conv(bf, 1, 1, 512, 320, 2560, k=1, act=i2it.ACT_GEGLU),
    "conv_clamp": lambda: case_conv(bf, 1, 16, 16, 64, 64, act=i2it.ACT_CLAMP1),
    "gn_128": lambda: case_gn(bf, 2, 64, 64, 128, True),
    "gn_320": lambda: case_gn(hf, 2, 16, 16, 320, False, 1e-5),
    "gn_1920": lambda: case_gn(bf, 1, 8, 8, 1920, True),
    "ln_320": lambda: case_ln(bf, 1000, 320),
    "ln_1280": lambda: case_ln(hf, 77, 1280),
    "attn_64": lambda: case_attn(bf, 2, 256, 256, 5, 64),
    "attn_cross": lambda: case_attn(hf, 2, 256, 77, 5, 64, kvb=1),
    "attn_4096": lambda: case_attn(bf, 1, 4096, 4096, 2, 64),
    "attn_vae": lambda: case_attn(bf, 1, 1024, 1024, 1, 512),
    # many waves of tiles per persistent CTA (ring / staging-tile reuse across tiles), residual and ragged variants
    "pair_conv": lambda: case_conv(bf, 4, 128, 128, 128, 128, res=True),
    "pair_conv256": lambda: case_conv(hf, 2, 128, 128, 256, 256),
    "halo_ragged": lambda: case_conv(bf, 16, 40, 40, 64, 512, res=True),
    "halo_k320": lambda: case_conv(hf, 8, 64, 64, 320, 320),
    "pair_lin": lambda: case_linear(bf, 65536, 320, 320, res=True),
    "pair_lin_odd": lambda: case_linear(hf, 128 * 301 + 17, 256, 512),
    "pair_geglu": lambda: case_conv(bf, 1, 1, 32768, 320, 2560, k=1, act=i2it.ACT_GEGLU),
    "pair_s2": lambda: case_conv(bf, 4, 256, 256, 128, 128, stride=2, asym=True),
    "attn_small": lambda: case_attn(hf, 3, 64, 64, 20, 64),
    "attn_ragged": lambda: case_attn(bf, 2, 200, 150, 2, 64),
    "attn_1024": lambda: case_attn(hf, 2, 1024, 1024, 10, 64),
    "upsample": lambda: case_up(bf),
}

if __name__ == "__main__":
    which = sys.argv[1] if len(sys.argv) > 1 else "list"
    if which == "list":
        print(" ".join(CASES))
        sys.exit(0)
    names = list(CASES) if which == "all" else sys.argv[1:]
    ok = True
    for n in names:
        try:
            ok = CASES[n]() and ok
        except Exception as e:  # keep going: print what the library said
            ok = False
            print(f"ERROR [{n}] {type(e).__name__}: {e}", flush=True)
    sys.exit(0 if ok else 1)
