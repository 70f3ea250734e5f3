"""-m gpu: the BASELINE configs at SD-Turbo width (VERDICT r1 item 1).

  config #3/#5  cyclegan-turbo fp16, batch 16, a2b and b2a (three adapters, two VAEs, three-rounding DDPM step)
  config #4     pix2pix-turbo stochastic, bf16, gamma = 0.4, noise map, distinct TwinConv weight sets
  config #2     pix2pix-turbo deterministic bf16 (the stage table; the e2e bound lives in test_gpu_e2e.py)

Each test runs the ENGINE at the config's batch size, then checks selected images of the batch stage by stage against the fp32
CPU oracle run at batch 1 on the same weights / inputs / eps (image i of a batch == its batch-1 forward bit for bit is tested in
test_gpu_e2e.py, so two images pin the batch).  Per stage it asserts finiteness and an error bound relative to the stage's scale,
and PRINTS the north-star band — the fraction of elements with |got - ref| <= 1e-4 + 1e-3*|ref| (rtol 1e-3 / atol 1e-4) — so that
the tolerance gap of a 16-bit pipeline is a number, not an argument (also written to $I2IT_PARITY_DIR/parity_bands.json when that directory exists)."""
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BANDS = {}


def band(got, ref, rtol=1e-3, atol=1e-4):
    got, ref = got.float().cpu(), ref.float().cpu()
    return ((got - ref).abs() <= atol + rtol * ref.abs()).float().mean().item()


def stage_report(tag, name, got, ref, rel_bound):
    got, ref = got.float().cpu(), ref.float().cpu()
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    assert torch.isfinite(got).all(), f"{tag}/{name}: non-finite values"
    err = (got - ref).abs()
    scale = ref.abs().mean().item() + 1e-12
    row = {"mean_abs_err": err.mean().item(), "max_abs_err": err.max().item(), "ref_mean_abs": scale,
           "rel_mean_err": err.mean().item() / scale, "north_star_band_frac": band(got, ref),
           "band_rtol1e-2_atol1e-3": band(got, ref, 1e-2, 1e-3)}
    BANDS.setdefault(tag, {})[name] = row
    print(f"[{tag}] {name:12s} mean|err|={row['mean_abs_err']:.3e} ({row['rel_mean_err']:.2%} of mean|ref|) max={row['max_abs_err']:.3e} "
          f"in north-star band (rtol 1e-3, atol 1e-4): {row['north_star_band_frac']:.1%}; in 10x band: {row['band_rtol1e-2_atol1e-3']:.1%}")
    assert row["rel_mean_err"] < rel_bound, (tag, name, row)
    return row


def _flush_bands():
    d = os.environ.get("I2IT_PARITY_DIR")
    if d and os.path.isdir(d):
        json.dump(BANDS, open(os.path.join(d, "parity_bands.json"), "w"), indent=1)


def _engine(kind, dt, sd, **kw):
    import i2it
    import weights as W
    e = i2it.Engine(dt, i2it.CYCLEGAN if kind == "cyclegan" else i2it.PIX2PIX, cfg=W.SD_TURBO, keep_stages=True, **kw)
    e.load_state_dict(sd)
    if kind == "pix2pix":
        e.set_adapter_scale("default", 1.0)
        e.set_adapter_scale("vae_skip", 2.0)
    else:
        for a in ("default_encoder", "default_decoder", "default_others"):
            e.set_adapter_scale(a, 1.0)
        e.set_adapter_scale("vae_skip", 2.0)
    return e


def _stages(e, pick):
    """engine stages of image `pick` as fp32 CPU tensors (channel padding stripped)."""
    g = lambda n, c=None: (e.read_stage(n, image=pick)[:, :c] if c else e.read_stage(n, image=pick)).cpu()
    return {"skip0": g("skip0"), "skip3": g("skip3"), "latent": g("latent", 4), "model_pred": g("model_pred", 4),
            "pre_clamp": g("pre_clamp", 3)}


# bounds: relative mean error per stage vs the fp32 oracle (16-bit storage of every activation; the DDPM step multiplies the
# UNet error by 14.6 and /0.18215 by another 5.5 before the decoder — SURVEY fact 6)
BOUNDS_FP16 = {"skip0": 1e-3, "skip3": 5e-3, "latent": 3e-3, "model_pred": 7e-3, "x_denoised": 7e-3, "pre_clamp": 1e-2}
BOUNDS_BF16 = {"skip0": 8e-3, "skip3": 4e-2, "latent": 2e-2, "model_pred": 5e-2, "x_denoised": 5e-2, "pre_clamp": 7e-2}


@pytest.fixture(scope="module")
def cyclegan_fp16():
    import weights as W
    sd = W.make_state_dict("cyclegan", W.SD_TURBO, seed=0)
    e = _engine("cyclegan", torch.float16, sd)
    e.finalize(1.0, 1.0, 1.0, -1.0)
    return sd, e


@pytest.mark.parametrize("direction", ["a2b", "b2a"])
def test_config3_cyclegan_fp16_batch16(cyclegan_fp16, direction):
    """BASELINE config #3 (and #5's per-GPU shape): cyclegan fp16, batch 16, 512x512, one caption embedding broadcast."""
    import i2it
    import oracle as O
    import weights as W
    sd, e = cyclegan_fp16
    dt, B, S = torch.float16, 16, 512
    g = torch.Generator().manual_seed(1)
    x = torch.rand(B, 3, S, S, generator=g) * 2 - 1
    text = torch.randn(1, 77, 1024, generator=torch.Generator().manual_seed(2))
    eps = torch.randn(B, 4, S // 8, S // 8, generator=torch.Generator().manual_seed(3))
    lat = torch.empty(B, 4, S // 8, S // 8, device="cuda", dtype=dt)
    out = e.forward(x.to(dt).cuda(), text.to(dt).cuda(), eps.to(dt).cuda(), direction=i2it.B2A if direction == "b2a" else i2it.A2B,
                    out_latent=lat)
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all() and torch.isfinite(lat.float()).all(), "fp16 overflow somewhere on the path"
    assert out.abs().max() <= 1.0
    q = lambda t: t.to(dt).float()
    tag = f"cfg3_cyclegan_fp16_b16_{direction}"
    for pick in (0, 11):
        st = {}
        with torch.no_grad():
            ref = O.cyclegan_forward(sd, q(x[pick:pick + 1]), q(text), q(eps[pick:pick + 1]), direction, W.SD_TURBO, stages=st)
        mine = _stages(e, pick)
        refs = {"skip0": st["skips"][0], "skip3": st["skips"][3], "latent": st["latent"], "model_pred": st["model_pred"],
                "pre_clamp": st["pre_clamp"]}
        for name, r in refs.items():
            stage_report(f"{tag}_img{pick}", name, mine[name], r, BOUNDS_FP16[name])
        stage_report(f"{tag}_img{pick}", "x_denoised", lat[pick:pick + 1], st["x_denoised"], BOUNDS_FP16["x_denoised"])
        row = stage_report(f"{tag}_img{pick}", "image", out[pick:pick + 1], ref, 1e-2)
        assert row["mean_abs_err"] < 3e-3, row
    _flush_bands()


def test_config4_pix2pix_stochastic_bf16(capsys):
    """BASELINE config #4's per-GPU shape: pix2pix stochastic, bf16, batch 8, gamma = 0.4, noise map seed 42, TwinConv with two
    distinct random weight sets; LoRA scale, skip gamma and the TwinConv blend all re-folded at r = 0.4."""
    import oracle as O
    import weights as W
    dt, B, S, r = torch.bfloat16, 8, 512, 0.4
    sd = W.make_state_dict("pix2pix", W.SD_TURBO, seed=0, twin=True)
    assert not torch.equal(sd["unet.conv_in.conv_in_pretrained.weight"], sd["unet.conv_in.conv_in_curr.weight"])
    e = _engine("pix2pix", dt, sd)
    e.finalize(r, r, r, r)
    g = torch.Generator().manual_seed(1)
    x = (torch.rand(B, 1, S, S, generator=g) < 0.5).float().expand(-1, 3, -1, -1).contiguous()
    text = torch.randn(1, 77, 1024, generator=torch.Generator().manual_seed(2))
    eps = torch.randn(B, 4, S // 8, S // 8, generator=torch.Generator().manual_seed(3))
    noise = torch.randn(B, 4, S // 8, S // 8, generator=torch.Generator().manual_seed(42))
    lat = torch.empty(B, 4, S // 8, S // 8, device="cuda", dtype=dt)
    out = e.forward(x.to(dt).cuda(), text.to(dt).cuda(), eps.to(dt).cuda(), noise.to(dt).cuda(), r, out_latent=lat)
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all() and out.abs().max() <= 1.0
    q = lambda t: t.to(dt).float()
    pick = 5
    st = {}
    with torch.no_grad():
        ref = O.pix2pix_forward(sd, q(x[pick:pick + 1]), q(text), q(eps[pick:pick + 1]), W.SD_TURBO, deterministic=False, r=r,
                                noise_map=q(noise[pick:pick + 1]), stages=st)
    mine = _stages(e, pick)
    tag = "cfg4_pix2pix_stochastic_bf16_b8"
    # "latent" of the engine is the UNet input (enc*r + noise*(1-r)) in stochastic mode
    refs = {"skip0": st["skips"][0], "skip3": st["skips"][3], "latent": st["unet_in"], "model_pred": st["model_pred"],
            "pre_clamp": st["pre_clamp"]}
    for name, rr in refs.items():
        stage_report(tag, name, mine[name], rr, BOUNDS_BF16[name])
    stage_report(tag, "x_denoised", lat[pick:pick + 1], st["x_denoised"], BOUNDS_BF16["x_denoised"])
    row = stage_report(tag, "image", out[pick:pick + 1], ref, 5e-2)
    assert row["mean_abs_err"] < 1.2e-2, row
    # gamma matters: the deterministic fold of the same weights gives a different image
    e.finalize(1.0, 1.0, 1.0, 1.0)
    out_r1 = e.forward(x.to(dt).cuda(), text.to(dt).cuda(), eps.to(dt).cuda(), noise.to(dt).cuda(), 1.0)
    assert (out_r1.float() - out.float()).abs().mean() > 1e-3
    _flush_bands()


def test_config2_stage_table_bf16_and_fp16():
    """Config #1/#2 inputs at B=1: the same stage table for bf16 and fp16 (fp16 at SD-Turbo width was never run in round 1)."""
    import oracle as O
    import weights as W
    sd = W.make_state_dict("pix2pix", W.SD_TURBO, seed=0)
    g = torch.Generator().manual_seed(1)
    x = (torch.rand(1, 1, 512, 512, generator=g) < 0.08).float().expand(-1, 3, -1, -1).contiguous()
    text = torch.randn(1, 77, 1024, generator=g)
    eps = torch.randn(1, 4, 64, 64, generator=g)
    for dt, bounds in ((torch.bfloat16, BOUNDS_BF16), (torch.float16, BOUNDS_FP16)):
        q = lambda t: t.to(dt).float()
        st = {}
        with torch.no_grad():
            ref = O.pix2pix_forward(sd, q(x), q(text), q(eps), W.SD_TURBO, stages=st)
        e = _engine("pix2pix", dt, sd)
        e.finalize(1.0, 1.0, 1.0, -1.0)
        lat = torch.empty(1, 4, 64, 64, device="cuda", dtype=dt)
        out = e.forward(x.to(dt).cuda(), text.to(dt).cuda(), eps.to(dt).cuda(), out_latent=lat)
        torch.cuda.synchronize()
        mine = _stages(e, 0)
        tag = "cfg2_pix2pix_" + ("bf16" if dt == torch.bfloat16 else "fp16")
        refs = {"skip0": st["skips"][0], "skip3": st["skips"][3], "latent": st["latent"], "model_pred": st["model_pred"],
                "pre_clamp": st["pre_clamp"]}
        for name, rr in refs.items():
            stage_report(tag, name, mine[name], rr, bounds[name])
        stage_report(tag, "x_denoised", lat, st["x_denoised"], bounds["x_denoised"])
        stage_report(tag, "image", out, ref, 7e-2 if dt == torch.bfloat16 else 1e-2)
        e.close()
    _flush_bands()
