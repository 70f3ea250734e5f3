"""-m gpu: the teacher-forced layer audit (tests/layer_audit.py) on the engine.

Each case runs one forward with keep_stages = 2, asserts that the audit covers every kept stage and every prepared weight,
holds every layer (on the engine's own inputs and prepared operands) and every prepared weight to its float64 bound, and
checks that the output image is bit-identical to a keep_stages = 0 forward on the same inputs.  The float64 references run
on the GPU.  Each case prints the worst err/bound and mean-ulp per layer family."""
import os
import time

import pytest
import torch

import layer_audit as LA

pytestmark = pytest.mark.gpu

bf, hf = torch.bfloat16, torch.float16


def _engine(kind, cfg, dt, sd, keep, catfuse=True):
    import i2it
    saved = os.environ.pop("I2IT_NO_CATFUSE", None)
    try:
        if not catfuse:
            os.environ["I2IT_NO_CATFUSE"] = "1"
        e = i2it.Engine(dt, i2it.CYCLEGAN if kind == "cyclegan" else i2it.PIX2PIX, cfg=cfg, keep_stages=keep)
    finally:
        os.environ.pop("I2IT_NO_CATFUSE", None)
        if saved is not None:
            os.environ["I2IT_NO_CATFUSE"] = saved
    e.load_state_dict(sd)
    return e


def _inputs(kind, cfg, B, H, W, tb, dt, seed=1):
    g = torch.Generator().manual_seed(seed)
    if kind == "pix2pix":
        x = (torch.rand(B, 1, H, W, generator=g) < 0.08).float().expand(-1, 3, -1, -1).contiguous()
    else:
        x = torch.rand(B, 3, H, W, generator=g) * 2 - 1
    text = torch.randn(tb, 77, cfg["cross_dim"], generator=g)
    eps = torch.randn(B, 4, H // 8, W // 8, generator=g)
    noise = torch.randn(B, 4, H // 8, W // 8, generator=g)
    c = lambda t: t.to(dt).cuda().contiguous()
    return c(x), c(text), c(eps), c(noise)


def run_case(tag, kind, cfg, sd, dt, B, H, W, tb=1, r=None, direction="a2b", cached=False, catfuse=True):
    import i2it
    t0 = time.time()
    spec = LA.Spec(sd, cfg, kind, direction, r=r)
    fold = (1.0, 1.0, 1.0, -1.0) if r is None else (r, r, r, r)
    spec.lw_unet, spec.lw_vae, spec.skip_gamma, spec.twin_r = fold
    x, text, eps, noise = _inputs(kind, cfg, B, H, W, tb, dt)
    noise = noise if r is not None else None
    d = i2it.B2A if direction == "b2a" else i2it.A2B
    outs = []
    for keep in (2, 0):
        e = _engine(kind, cfg, dt, sd, keep, catfuse)
        for a, s in spec.adapter_scales.items():
            e.set_adapter_scale(a, s)
        e.finalize(*fold)
        if cached:
            e.set_text(text)
        out = e.forward(x, None if cached else text, eps, noise, 1.0 if r is None else r, direction=d)
        torch.cuda.synchronize()
        outs.append(out)
        if keep == 2:
            src = LA.EngineSource(e, dict(x=x, text=text, eps=eps, noise=noise, image=out))
            with torch.no_grad():
                a = LA.Audit(src, spec, dt).run()
            print(f"\n[{tag}] {len(a.results)} checks, {len(a.src.stage_names())} stages, {len(a.keys_seen)} prepared weights\n"
                  + a.report())
            a.assert_ok()
            del src, a
        e.close()
        del e
        torch.cuda.empty_cache()
    assert torch.equal(outs[0], outs[1]), f"{tag}: keep_stages = 2 changed the output image"
    print(f"[{tag}] wall {time.time() - t0:.1f} s")


@pytest.fixture(scope="module")
def tiny():
    import weights as W
    return W.TINY, W.make_state_dict("pix2pix", W.TINY, seed=0, perturb_norm=True)


@pytest.mark.parametrize("dt", [bf, hf], ids=["bf16", "fp16"])
def test_tiny_pix2pix_deterministic(tiny, dt):
    cfg, sd = tiny
    run_case(f"tiny det {dt}", "pix2pix", cfg, sd, dt, 2, 64, 64, tb=2)


def test_tiny_odd_latent_maps(tiny):
    """72x104: 9x13 latent, odd maps through the stride-2 convs (pad to even) and nearest upsampling to the skip sizes."""
    cfg, sd = tiny
    run_case("tiny 72x104", "pix2pix", cfg, sd, bf, 2, 72, 104)


def test_tiny_pix2pix_stochastic():
    """r = 0.4 re-folds LoRA, skip gamma and the TwinConv blend; the latent blends the noise map."""
    import weights as W
    sd = W.make_state_dict("pix2pix", W.TINY, seed=0, perturb_norm=True, twin=True)
    run_case("tiny stochastic", "pix2pix", W.TINY, sd, bf, 2, 64, 64, r=0.4)


@pytest.mark.parametrize("cached", [False, True], ids=["inline_text", "set_text"])
def test_tiny_cyclegan_b2a(cached):
    """three UNet adapters, the b2a VAE, per-image prompts; then the prompt's K / V^T cached by i2it_set_text."""
    import weights as W
    sd = W.make_state_dict("cyclegan", W.TINY, seed=0, perturb_norm=True)
    run_case(f"tiny cyclegan b2a cached={cached}", "cyclegan", W.TINY, sd, hf, 2, 64, 64, tb=2, direction="b2a", cached=cached)


def test_tiny_concat_copies(tiny):
    """I2IT_NO_CATFUSE: the UNet concatenations built by copy kernels."""
    cfg, sd = tiny
    run_case("tiny no-catfuse", "pix2pix", cfg, sd, bf, 2, 64, 64, catfuse=False)


@pytest.fixture(scope="module")
def sdturbo():
    import weights as W
    return W.SD_TURBO, W.make_state_dict("pix2pix", W.SD_TURBO, seed=0)


@pytest.mark.parametrize("dt", [bf, hf], ids=["bf16", "fp16"])
def test_sdturbo_256(sdturbo, dt):
    """SD-Turbo widths: heads 5 / 10 / 20, GroupNorm over the 2560 / 1920 / 960 / 640-channel concatenations."""
    cfg, sd = sdturbo
    run_case(f"sd-turbo 256 {dt}", "pix2pix", cfg, sd, dt, 2, 256, 256)


def test_sdturbo_512(sdturbo):
    """512x512: the VAE attention runs unfused over 4096 tokens."""
    cfg, sd = sdturbo
    run_case("sd-turbo 512 bf16", "pix2pix", cfg, sd, bf, 1, 512, 512)
