"""CPU: the layer audit (tests/layer_audit.py) accepts a correctly rounded pipeline and names the layer of each injected error.

The emulated source computes every layer in float64 from the previous rounded stage and rounds once; its prepared weights
are round16 of the float64 fold in the engine layout.  Each injected error below is one the end-to-end stage bounds can miss:
the audit must fail on exactly the layer or prepared weight that carries it, and nowhere else (teacher forcing)."""
import pytest
import torch

import kref
import layer_audit as LA

DT = torch.bfloat16
S = 32                                   # 32x32 image: 4x4 latent, odd UNet maps (1x1) and upsample_to sizes on the path


def _inputs(cfg, B=1, seed=1, r=None):
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(B, 3, S, S, generator=g) * 2 - 1).to(DT)
    text = torch.randn(1, 77, cfg["cross_dim"], generator=g).to(DT)
    eps = torch.randn(B, 4, S // 8, S // 8, generator=g).to(DT)
    noise = torch.randn(B, 4, S // 8, S // 8, generator=g).to(DT) if r is not None else None
    return dict(x=x, text=text, eps=eps, noise=noise, image=None)


def _spec(sd, r=None):
    import weights as W
    if r is None:
        return LA.Spec(sd, W.TINY)
    return LA.Spec(sd, W.TINY, r=r, lw_unet=r, lw_vae=r, skip_gamma=r, twin_r=r)


def _audit(spec, r=None, stage_hook=None, weight_hook=None):
    src = LA.EmulatedSource(_inputs(spec.cfg, r=r))
    with torch.no_grad():
        LA.Audit(src, spec, DT, emulate=True, stage_hook=stage_hook, weight_hook=weight_hook).run()
        return LA.Audit(src, spec, DT).run()


def _failed(a):
    return sorted(n for _, n, _ in a.failures())


@pytest.fixture(scope="module")
def sd_det():
    import weights as W
    return W.make_state_dict("pix2pix", W.TINY, seed=0, perturb_norm=True)


@pytest.fixture(scope="module")
def sd_twin():
    import weights as W
    return W.make_state_dict("pix2pix", W.TINY, seed=0, perturb_norm=True, twin=True)


def test_audit_passes_on_emulated_pipeline(sd_det):
    a = _audit(_spec(sd_det))
    print("\n" + a.report())
    a.assert_ok()
    assert not any(a.completeness.values())
    fam = {f for f, _, _ in a.results}
    assert {"conv", "linear", "groupnorm", "layernorm", "attention", "concat", "upsample", "latent", "ddpm", "weight"} <= fam


def test_audit_passes_on_emulated_stochastic_pipeline(sd_twin):
    a = _audit(_spec(sd_twin, 0.4), r=0.4)
    a.assert_ok()
    assert "unet.conv_in.conv_in_pretrained|twin" in a.src.prepared_keys()


def test_completeness_catches_an_unaudited_stage(sd_det):
    spec = _spec(sd_det)
    src = LA.EmulatedSource(_inputs(spec.cfg))
    with torch.no_grad():
        LA.Audit(src, spec, DT, emulate=True).run()
        src.order.append("unet.some_new_layer")
        with pytest.raises(LA.AuditError, match="some_new_layer"):
            LA.Audit(src, spec, DT).run()


# ---------------------------------------------------------------------------------------------------------------------
# injected errors: each must fail on exactly the named layer / prepared weight
# ---------------------------------------------------------------------------------------------------------------------
def test_conv1_bias_without_time_embedding(sd_det):
    key = "unet.down_blocks.1.resnets.0.conv1"
    spec = _spec(sd_det)

    def hook(k, w, b, a):
        return (w, a.P(k + ".bias").float()) if k == key else (w, b)
    assert _failed(_audit(spec, weight_hook=hook)) == [key]


def test_skip_conv_at_gamma_one_in_a_gamma_04_fold(sd_twin):
    key = "vae.decoder.skip_conv_2"
    spec = _spec(sd_twin, 0.4)

    def hook(k, w, b, a):
        return (a.layout(a.fold64(k), w.shape[2]).to(DT), b) if k == key else (w, b)
    assert _failed(_audit(spec, r=0.4, weight_hook=hook)) == [key]


def test_cross_attention_with_the_neighbouring_blocks_k(sd_det):
    name = "unet.down_blocks.0.attentions.1.transformer_blocks.0.attn2"
    other = "unet.down_blocks.0.attentions.0.transformer_blocks.0.attn2.to_k"

    def hook(n, v, a):
        if n != name:
            return v
        B, C, H, W = v.shape
        q = a.src.stages[name + ".to_q"].double().permute(0, 2, 3, 1).reshape(B, H * W, C)
        k = a.src.stages[other].double().permute(0, 2, 3, 1).reshape(1, 77, C)
        vv = a.src.stages[name + ".to_v"].double()[:, :77, 0, :]
        o = kref.attention64(q, k, vv, 1)[0]
        return kref.round16(o.reshape(B, H, W, C).permute(0, 3, 1, 2), DT)
    assert _failed(_audit(_spec(sd_det), stage_hook=hook)) == [name]


def test_lora_adapter_dropped_from_one_weight(sd_det):
    key = "unet.down_blocks.1.attentions.0.proj_in"

    def hook(k, w, b, a):
        return (a.layout(a.P(k + ".weight"), w.shape[2]).to(DT), b) if k == key else (w, b)
    assert _failed(_audit(_spec(sd_det), weight_hook=hook)) == [key]


def test_unet_concat_with_halves_swapped(sd_det):
    name = "unet.up_blocks.1.resnets.2.concat"
    h_c = sd_det["unet.up_blocks.1.resnets.1.conv2.weight"].shape[0]

    def hook(n, v, a):
        return torch.cat([v[:, h_c:], v[:, :h_c]], dim=1) if n == name else v
    assert _failed(_audit(_spec(sd_det), stage_hook=hook)) == [name]


def test_subpixel_phase_with_transposed_taps(sd_det):
    key = "vae.decoder.up_blocks.1.upsamplers.0.conv|subpixel"

    def hook(k, w, b, a):
        if k != key:
            return w, b
        w = w.clone()
        w[4 + 1], w[4 + 2] = w[4 + 2].clone(), w[4 + 1].clone()    # phase (0,1): taps (ty,tx) = (0,1) <-> (1,0)
        return w, b
    assert _failed(_audit(_spec(sd_det), weight_hook=hook)) == [key]


def test_groupnorm_with_the_wrong_epsilon(sd_det):
    """decoder.conv_in scaled down 1000x: its output variance (~1e-7) is where eps 1e-5 instead of 1e-6 shows."""
    sd = {k: (v * 1e-3 if k.startswith("vae.decoder.conv_in.") and "lora_A" not in k else v) for k, v in sd_det.items()}
    name = "vae.decoder.mid_block.resnets.0.norm1"

    def hook(n, v, a):
        if n != name:
            return v
        x = a.S("vae.decoder.conv_in")
        ref, _ = kref.group_norm64(x, a.P(n + ".weight"), a.P(n + ".bias"), 1e-5, True, DT)
        return kref.round16(ref.permute(0, 3, 1, 2), DT)
    assert _failed(_audit(_spec(sd), stage_hook=hook)) == [name]


def test_nonzero_cin_pad_column(sd_det):
    key = "unet.conv_in"                                           # 4 latent channels padded to 8

    def hook(k, w, b, a):
        if k != key:
            return w, b
        w = w.clone()
        w[4, 7, 5] = 0.25
        return w, b
    a = _audit(_spec(sd_det), weight_hook=hook)
    assert _failed(a) == [key]
    assert "padding" in [c for _, n, c in a.failures()][0].extra


def test_attention_bound_follows_the_engines_path():
    """The subnormal set of the attention bound (kref.py header) is the flash one where the engine ran a flash kernel:
    every d = 64 layer unless the engine was created with I2IT_NO_FLASH, the one-head d = 512 layer above 8192 keys."""
    class Src:
        def __init__(self, flash):
            self.flash, self.inputs = flash, dict(x=torch.zeros(1, 3, S, S))

    import weights as W
    on, off = LA.Audit(Src(True), LA.Spec({}, W.TINY), DT), LA.Audit(Src(False), LA.Spec({}, W.TINY), DT)
    assert on.flash_path(5, 64, 4096) and on.flash_path(1, 64, 1)
    assert not on.flash_path(1, 512, 8192) and on.flash_path(1, 512, 8193)
    assert not any(off.flash_path(h, d, n) for h, d, n in ((5, 64, 4096), (1, 512, 8193)))
    assert not LA.Audit(LA.EmulatedSource(Src(True).inputs), LA.Spec({}, W.TINY), DT).flash_path(5, 64, 4096)
