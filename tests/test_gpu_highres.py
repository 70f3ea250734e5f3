"""-m gpu: images past 512^2.  The decoder's full-resolution tensors of a 12-megapixel image (256 x 4032 x 3024 = 3.1e9
elements) pass 2^31 elements.  The VAE mid-block attention (one head of 512, fused above 8192 keys) has its own file,
tests/test_gpu_attention_d512.py.

  2^31        the decoder's largest convs and GroupNorm at 4032x3024x256, checked on row bands (first rows, the rows around
              the 2^31-element offset, last rows) against float64 references computed for those bands only
  end to end  1280x720 against the CPU fp32 oracle stage by stage; 4032x3024 through the public wrapper (finite, in range)
"""
import math
import sys

import pytest
import torch

import kref

pytestmark = pytest.mark.gpu

bf, hf = torch.bfloat16, torch.float16
DTYPES = [pytest.param(bf, id="bf16"), pytest.param(hf, id="fp16")]
H12, W12 = 3024, 4032            # a 12 MP phone photo (landscape 4032 x 3024)


def engine(dtype):
    import i2it
    return i2it.Engine(dtype, use_cuda_graph=False)


def mk(*shape, dtype=torch.float32, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(dtype)


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


# ---------------------------------------------------------------------------------------------------------------------
# tensors past 2^31 elements
# ---------------------------------------------------------------------------------------------------------------------
def bands(H, W, C):
    """Output row ranges: the first rows, the rows around element offset 2^31, the last rows."""
    r = (1 << 31) // (W * C)
    return [(0, 3), (r - 2, r + 3), (H - 3, H)]


def gn_stats64(y, groups=32, chunk=256):
    """Per-group float64 mean and variance of a [1, H, W, C] tensor, in row chunks."""
    C = y.shape[3]
    s = torch.zeros(groups, dtype=torch.float64, device=y.device)
    s2 = torch.zeros_like(s)
    for a in range(0, y.shape[1], chunk):
        t = y[0, a:a + chunk].double().reshape(-1, groups, C // groups)
        s += t.sum(dim=(0, 2))
        s2 += (t * t).sum(dim=(0, 2))
    n = y.shape[1] * y.shape[2] * (C // groups)
    mean = s / n
    return mean, s2 / n - mean * mean


def check_gn_band(name, got, y, a, b, mean, var, gamma, beta, eps, silu, dtype, groups=32):
    C = y.shape[3]
    yb = y[:, a:b].double()
    m, rstd = mean.view(1, 1, 1, groups, 1), torch.rsqrt(var.view(1, 1, 1, groups, 1) + eps)
    xh = ((yb.reshape(*yb.shape[:3], groups, C // groups) - m) * rstd).reshape(yb.shape)
    kappa = (m.abs() * rstd).expand(*yb.shape[:3], groups, C // groups).reshape(yb.shape)
    g, bb = gamma.double().view(1, 1, 1, C).expand_as(xh), beta.double().view(1, 1, 1, C).expand_as(xh)
    yy = xh * g + bb
    ref = yy * torch.sigmoid(yy) if silu else yy
    bound = kref._norm_bound(ref, xh, kappa, g, bb, dtype, silu, two_pass=False)
    return kref.check_norm(name, got[:, a:b], ref, bound, dtype)


def nchw(t):
    return t.double().permute(0, 3, 1, 2)


def gn_params(C, seed=20):
    return mk(C, seed=seed) * 0.2 + 1, mk(C, seed=seed + 1) * 0.1


def test_subpixel_upconv_past_2g_elements():
    """up_blocks.2's upsampler conv at 12 MP: 2016x1512x256 -> 4032x3024x256 (3.1e9 elements) with the GroupNorm(+SiLU) of
    up_blocks.3.resnets.0.norm1 fused into its epilogue."""
    dtype, C = bf, 256
    E = engine(dtype)
    x = mk(1, H12 // 2, W12 // 2, C, dtype=dtype, seed=1)
    w = mk(C, C, 3, 3, scale=1 / math.sqrt(9 * C), seed=2)
    b = mk(C, seed=3) * 0.1
    gamma, beta = gn_params(C)
    got, g = E.op_conv2d_ex(x, w, b, up2x=True, gn=(gamma, beta, 1e-6, True))
    torch.cuda.synchronize()
    ops = launches(E, "up2x 12MP")
    assert sum(k == "tapgemm:conv_up2x" for k in kinds(ops)) == 4 and "gn_final_part" in kinds(ops)
    wsub = kref.subpixel_weights(w, dtype)
    mean, var = gn_stats64(got)
    checks = []
    for r0, r1 in bands(H12, W12, C):
        a, bb = max(0, r0 // 2 - 1), min(H12 // 2, (r1 - 1) // 2 + 2)
        xs = x[:, a:bb]
        ref = kref.subpixel_conv64(xs, wsub, b)[:, :, r0 - 2 * a:r1 - 2 * a]
        mag = kref.subpixel_conv64(xs.abs(), wsub.abs(), b.abs())[:, :, r0 - 2 * a:r1 - 2 * a]
        # the zero padding of a band that does not start at row 0 / end at the last row is not the image's: those rows
        # of the band reference are cropped away above, and every kept row reads only rows inside the band
        checks.append(kref.check_gemm(f"up2x rows {r0}:{r1}", nchw(got[:, r0:r1]), ref, mag, 4 * C, dtype))
        checks.append(check_gn_band(f"up2x gn rows {r0}:{r1}", g, got, r0, r1, mean, var, gamma, beta, 1e-6, True, dtype))
    report(*checks)


def conv3_band(x, w, b, r0, r1):
    """3x3 conv (padding 1) of output rows [r0, r1) from input rows r0-1 .. r1 (zero rows only at the image border)."""
    H = x.shape[1]
    a, bb = max(0, r0 - 1), min(H, r1 + 1)
    y = kref.conv64(x[:, a:bb], w, b)
    return y[:, :, r0 - a:r1 - a]


def test_conv_second_source_past_2g_elements():
    """up_blocks.3.resnets.0.conv2 + conv_shortcut shape at 12 MP: 3x3 256 -> 128 over a 3.1e9-element input, plus a 1x1
    second source of 256 channels."""
    dtype, Cin, Cout = bf, 256, 128
    E = engine(dtype)
    x = mk(1, H12, W12, Cin, dtype=dtype, seed=1)
    x2 = mk(1, H12, W12, Cin, dtype=dtype, seed=2)
    w = mk(Cout, Cin, 3, 3, scale=1 / math.sqrt(9 * Cin), seed=3).to(dtype).float()
    w2 = mk(Cout, Cin, 1, 1, scale=1 / math.sqrt(Cin), seed=4).to(dtype).float()
    b = mk(Cout, seed=5) * 0.1
    got = E.op_conv2d_ex(x, w, b, x2=x2, w2=w2)
    torch.cuda.synchronize()
    launches(E, "conv3x3 + 1x1 12MP")
    checks = []
    for r0, r1 in bands(H12, W12, Cin):
        ref = conv3_band(x, w, b, r0, r1) + kref.conv64(x2[:, r0:r1], w2)
        mag = conv3_band(x.abs(), w.abs(), b.abs(), r0, r1) + kref.conv64(x2[:, r0:r1].abs(), w2.abs())
        checks.append(kref.check_gemm(f"conv rows {r0}:{r1}", nchw(got[:, r0:r1]), ref, mag, 9 * Cin + Cin, dtype))
    report(*checks)


def test_group_norm_past_2g_elements():
    dtype, C = bf, 256
    E = engine(dtype)
    y = mk(1, H12, W12, C, dtype=dtype, scale=2.0, seed=1)
    y[..., 64:128] += 3.0                        # groups with |mean| > std
    gamma, beta = gn_params(C)
    got = E.op_group_norm(y, gamma, beta, 1e-6, True)
    torch.cuda.synchronize()
    assert "gn_stats" in kinds(launches(E, "groupnorm 12MP"))
    mean, var = gn_stats64(y)
    report(*[check_gn_band(f"gn rows {r0}:{r1}", got, y, r0, r1, mean, var, gamma, beta, 1e-6, True, dtype)
             for r0, r1 in bands(H12, W12, C)])


# ---------------------------------------------------------------------------------------------------------------------
# end to end
# ---------------------------------------------------------------------------------------------------------------------
BOUNDS_FP16 = {"skip0": 1e-3, "skip3": 5e-3, "latent": 3e-3, "model_pred": 7e-3, "x_denoised": 7e-3, "pre_clamp": 1e-2}
BOUNDS_BF16 = {"skip0": 8e-3, "skip3": 4e-2, "latent": 2e-2, "model_pred": 5e-2, "x_denoised": 5e-2, "pre_clamp": 7e-2}


def stage_report(tag, name, got, ref, rel_bound):
    got, ref = got.float().cpu(), ref.float().cpu()
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    assert torch.isfinite(got).all(), f"{tag}/{name}: non-finite values"
    err = (got - ref).abs()
    rel = err.mean().item() / (ref.abs().mean().item() + 1e-12)
    print(f"[{tag}] {name:12s} mean|err|={err.mean().item():.3e} ({rel:.2%} of mean|ref|) max={err.max().item():.3e}")
    assert rel < rel_bound, (tag, name, rel)


def test_e2e_1280x720_stage_table():
    """pix2pix at 1280x720 (14400 VAE tokens: the fused attention in encoder and decoder), bf16 and fp16, batch 1, stage by
    stage against the fp32 CPU oracle with the 512^2 bounds."""
    import i2it
    import oracle as O
    import weights as W
    H, Wd = 720, 1280
    sd = W.make_state_dict("pix2pix", W.SD_TURBO, seed=0)
    g = torch.Generator().manual_seed(1)
    x = (torch.rand(1, 1, H, Wd, generator=g) < 0.08).float().expand(-1, 3, -1, -1).contiguous()
    text = torch.randn(1, 77, 1024, generator=g)
    eps = torch.randn(1, 4, H // 8, Wd // 8, generator=g)
    for dt, bounds in ((bf, BOUNDS_BF16), (hf, BOUNDS_FP16)):
        q = lambda t: t.to(dt).float()
        st = {}
        with torch.no_grad():
            ref = O.pix2pix_forward(sd, q(x), q(text), q(eps), W.SD_TURBO, stages=st)
        e = i2it.Engine(dt, i2it.PIX2PIX, cfg=W.SD_TURBO, keep_stages=True)
        e.load_state_dict(sd)
        e.set_adapter_scale("default", 1.0)
        e.set_adapter_scale("vae_skip", 2.0)
        e.finalize(1.0, 1.0, 1.0, -1.0)
        lat = torch.empty(1, 4, H // 8, Wd // 8, device="cuda", dtype=dt)
        out = e.forward(x.to(dt).cuda(), text.to(dt).cuda(), eps.to(dt).cuda(), out_latent=lat)
        torch.cuda.synchronize()
        plan = [o["kind"] for o in e.profile(1)]
        assert plan.count("flash_attn512") == 2 and "softmax" not in plan, sorted(set(plan))
        rd = lambda n, c=None: (e.read_stage(n, max_elems=1 << 28)[:, :c] if c else e.read_stage(n, max_elems=1 << 28)).cpu()
        mine = {"skip0": rd("skip0"), "skip3": rd("skip3"), "latent": rd("latent", 4), "model_pred": rd("model_pred", 4),
                "pre_clamp": rd("pre_clamp", 3)}
        refs = {"skip0": st["skips"][0], "skip3": st["skips"][3], "latent": st["latent"], "model_pred": st["model_pred"],
                "pre_clamp": st["pre_clamp"]}
        tag = "1280x720_" + ("bf16" if dt == bf else "fp16")
        for name, rr in refs.items():
            stage_report(tag, name, mine[name], rr, bounds[name])
        stage_report(tag, "x_denoised", lat, st["x_denoised"], bounds["x_denoised"])
        stage_report(tag, "image", out, ref, 7e-2 if dt == bf else 1e-2)
        e.close()


def test_e2e_12mp_public_wrapper():
    """A 4032x3024 photo through Pix2Pix_Turbo as inference_paired.py calls it (random-init weights, bf16, batch 1).  The
    oracle cannot run here (its explicit softmax alone would need 290 GB); the op tests above carry the numerics."""
    from pix2pix_turbo import Pix2Pix_Turbo
    dt = bf
    m = Pix2Pix_Turbo()
    m.set_eval()
    m.to(dt)
    g = torch.Generator().manual_seed(1)
    small = (torch.rand(1, 1, 720, 1280, generator=g) < 0.08).float().expand(-1, 3, -1, -1).to(dt).cuda()
    with torch.no_grad():
        m(small, "a photo")
    eng = m._get_engine()
    ws_small = eng.workspace_bytes(1, 720, 1280)
    torch.cuda.empty_cache()                     # blocks the caching allocator kept from earlier tests count as free here
    # every buffer of a plan grows linearly in pixels once the attention is fused
    need = int(ws_small * (H12 * W12) / (720 * 1280) * 1.15) + 4 * 3 * H12 * W12 * 2
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"device has {free / 2**30:.1f} GiB free, a 4032x3024 plan needs about {need / 2**30:.1f} GiB")
    x = (torch.rand(1, 1, H12, W12, generator=g) < 0.08).float().expand(-1, 3, -1, -1).to(dt).cuda()
    free0, _ = torch.cuda.mem_get_info()
    with torch.no_grad():
        out = m(x, "a photo")
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    assert out.shape == x.shape and torch.isfinite(out.float()).all() and out.abs().max() <= 1.0
    ws = eng.workspace_bytes(1, H12, W12)
    plan = [o["kind"] for o in eng.profile(1)]
    print(f"\n[12MP] workspace_bytes={ws / 2**30:.2f} GiB (estimate {need / 2**30:.2f}), cudaMemGetInfo drop "
          f"{(free0 - free1) / 2**30:.2f} GiB, launches={len(plan)}")
    assert plan.count("flash_attn512") == 2 and "softmax" not in plan
