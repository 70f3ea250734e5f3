"""ORACLE — TEST INFRASTRUCTURE ONLY.  Never imported by the product path.

CPU restatement (pure PyTorch functional, fp32 by default) of the one hot path this
repository accelerates:

    VAE.encode -> one SD-Turbo UNet step (t=999) -> DDPM closed-form x0 -> VAE.decode

as executed by the reference wrappers
    src/pix2pix_turbo.py:186-219   (Pix2Pix_Turbo.forward)
    src/cyclegan_turbo.py:199-207  (CycleGAN_Turbo.forward_with_networks)
    src/model.py:14-54             (patched VAE encoder/decoder forwards)

PARITY UNPINNED: the arithmetic lives in diffusers==0.25.1 / peft, which are pinned in
environment.yaml:31-33 but are NOT vendored in the reference repository and are not
installed here; the reference ships no tests or golden vectors for the path.
This file therefore restates the *published* diffusers 0.25.1 algorithm (AutoencoderKL,
UNet2DConditionModel, DDPMScheduler, peft LoRA) and is pinned by:
  * exact parameter-count checksums (UNet 865,910,724; VAE 83,653,863; skip convs 491,520),
  * the analytic scheduler constants (alpha_bar_999 = 0.0046600951),
  * algebraic identities (LoRA folded == unfolded, TwinConv folded == blended, gamma=1
    stochastic == deterministic, zero lora_B == base model) — see tests/test_oracle.py.

Weights are a flat ``dict[str, Tensor]`` in diffusers/peft key naming with a model prefix
("unet.", "vae.", "vae_b2a."); LoRA branches are kept UN-merged here
(y = W x + b + sum_a s_a * B_a(A_a x)) so that the product's load-time fold is testable.
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import this.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

SD = Dict[str, torch.Tensor]

# SD-Turbo hyper-parameters (HF config.json of stabilityai/sd-turbo; hard-coded because the hub is
# unreachable offline).  A reduced config with the same structure is used by fast tests.
SD_TURBO = dict(
    unet_channels=(320, 640, 1280, 1280),
    unet_heads=(5, 10, 20, 20),          # "attention_head_dim" in the HF config are head COUNTS
    unet_layers_per_block=2,
    cross_dim=1024,
    temb_dim=1280,
    unet_groups=32,
    vae_channels=(128, 256, 512, 512),
    vae_layers_per_block=2,
    vae_groups=32,
    latent_channels=4,
    scaling_factor=0.18215,
)

# ----------------------------------------------------------------------------------------------
# scheduler  (reference: src/model.py:7-11 -> diffusers DDPMScheduler, 1 step, "trailing")
# ----------------------------------------------------------------------------------------------

def alphas_cumprod(num_train_timesteps: int = 1000, beta_start: float = 0.00085,
                   beta_end: float = 0.012) -> torch.Tensor:
    """scaled_linear betas as in diffusers DDPMScheduler.__init__ (fp32 throughout)."""
    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
    return torch.cumprod(1.0 - betas, dim=0)


def ddpm_step_x0(model_pred: torch.Tensor, sample: torch.Tensor, t: int = 999,
                 math_dtype: Optional[torch.dtype] = torch.float32) -> torch.Tensor:
    """DDPMScheduler.step for the single trailing step (t=999, prev_t=-1).

    prev alpha_bar = 1 => coefficient of x0 is 1 and of the current sample is 0, so
    prev_sample = x0 = (x - sqrt(1-abar)*eps_hat)/sqrt(abar)  (+ 1e-10-scale variance noise that
    the reference draws and that is numerically nil; it is omitted here).
    math_dtype=float32 mirrors Pix2Pix_Turbo (1-D timesteps tensor promotes the step to fp32,
    src/pix2pix_turbo.py:162,200-201); math_dtype=None mirrors CycleGAN_Turbo (0-dim timestep keeps
    the activation dtype with three roundings, src/cyclegan_turbo.py:205).
    """
    ac = alphas_cumprod()[t]
    sa, s1 = ac.sqrt(), (1.0 - ac).sqrt()
    if math_dtype is not None:
        x0 = (sample.to(math_dtype) - s1.to(math_dtype) * model_pred.to(math_dtype)) / sa.to(math_dtype)
        return x0.to(model_pred.dtype)
    dt = model_pred.dtype
    return (sample - s1.to(dt) * model_pred) / sa.to(dt)


# ----------------------------------------------------------------------------------------------
# LoRA-aware primitive layers (peft tuners/lora/layer.py: Linear.forward / Conv2d.forward)
# ----------------------------------------------------------------------------------------------

def _base(sd: SD, name: str, what: str) -> Optional[torch.Tensor]:
    for k in (f"{name}.{what}", f"{name}.base_layer.{what}"):
        if k in sd:
            return sd[k]
    return None


def _adapters(sd: SD, name: str) -> List[str]:
    pre = f"{name}.lora_A."
    return sorted({k[len(pre):].rsplit(".", 1)[0] for k in sd if k.startswith(pre)})


def linear(sd: SD, name: str, x: torch.Tensor, scales: Dict[str, float]) -> torch.Tensor:
    w, b = _base(sd, name, "weight"), _base(sd, name, "bias")
    y = F.linear(x, w, b)
    for a in _adapters(sd, name):
        s = scales.get(a, 0.0)
        if s != 0.0:
            y = y + F.linear(F.linear(x, sd[f"{name}.lora_A.{a}.weight"]), sd[f"{name}.lora_B.{a}.weight"]) * s
    return y


def conv2d(sd: SD, name: str, x: torch.Tensor, scales: Dict[str, float], stride: int = 1,
           padding: int = 0) -> torch.Tensor:
    w, b = _base(sd, name, "weight"), _base(sd, name, "bias")
    y = F.conv2d(x, w, b, stride=stride, padding=padding)
    for a in _adapters(sd, name):
        s = scales.get(a, 0.0)
        if s != 0.0:
            # peft Conv2d LoRA: lora_A = Conv(cin->r, k, same stride/pad, no bias); lora_B = Conv1x1(r->cout)
            h = F.conv2d(x, sd[f"{name}.lora_A.{a}.weight"], None, stride=stride, padding=padding)
            y = y + F.conv2d(h, sd[f"{name}.lora_B.{a}.weight"], None) * s
    return y


def group_norm(sd: SD, name: str, x: torch.Tensor, groups: int, eps: float) -> torch.Tensor:
    return F.group_norm(x, groups, sd[f"{name}.weight"], sd[f"{name}.bias"], eps)


def layer_norm(sd: SD, name: str, x: torch.Tensor) -> torch.Tensor:
    return F.layer_norm(x, (x.shape[-1],), sd[f"{name}.weight"], sd[f"{name}.bias"], 1e-5)


def sdpa(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int) -> torch.Tensor:
    """diffusers AttnProcessor2_0: softmax(q k^T / sqrt(d)) v, no mask, q/k/v are [B, N, heads*d]."""
    B, Nq, C = q.shape
    d = C // heads
    q = q.view(B, Nq, heads, d).transpose(1, 2)
    k = k.view(B, -1, heads, d).transpose(1, 2)
    v = v.view(B, -1, heads, d).transpose(1, 2)
    w = torch.softmax((q @ k.transpose(-1, -2)).float() * (1.0 / math.sqrt(d)), dim=-1).to(q.dtype)
    return (w @ v).transpose(1, 2).reshape(B, Nq, C)


# ----------------------------------------------------------------------------------------------
# VAE (diffusers models/vae.py Encoder/Decoder, models/resnet.py ResnetBlock2D with temb=None,
#      models/attention_processor.py Attention with 1 head) + reference patches src/model.py:14-54
# ----------------------------------------------------------------------------------------------

def _vae_resnet(sd, p, x, cfg, scales):
    g = cfg["vae_groups"]
    h = F.silu(group_norm(sd, f"{p}.norm1", x, g, 1e-6))
    h = conv2d(sd, f"{p}.conv1", h, scales, padding=1)
    h = F.silu(group_norm(sd, f"{p}.norm2", h, g, 1e-6))
    h = conv2d(sd, f"{p}.conv2", h, scales, padding=1)
    if _base(sd, f"{p}.conv_shortcut", "weight") is not None:
        x = conv2d(sd, f"{p}.conv_shortcut", x, scales)
    return x + h                                                     # output_scale_factor = 1


def _vae_attn(sd, p, x, cfg, scales):
    B, C, H, W = x.shape
    r = x
    t = group_norm(sd, f"{p}.group_norm", x.view(B, C, H * W), cfg["vae_groups"], 1e-6).transpose(1, 2)
    q, k, v = (linear(sd, f"{p}.to_{n}", t, scales) for n in "qkv")
    o = linear(sd, f"{p}.to_out.0", sdpa(q, k, v, 1), scales)
    return o.transpose(1, 2).reshape(B, C, H, W) + r


def _vae_mid(sd, p, x, cfg, scales):
    x = _vae_resnet(sd, f"{p}.resnets.0", x, cfg, scales)
    x = _vae_attn(sd, f"{p}.attentions.0", x, cfg, scales)
    return _vae_resnet(sd, f"{p}.resnets.1", x, cfg, scales)


def vae_encode(sd: SD, prefix: str, x: torch.Tensor, eps: torch.Tensor, cfg=SD_TURBO,
               scales: Optional[Dict[str, float]] = None, stages: Optional[dict] = None):
    """my_vae_encoder_fwd (src/model.py:14-27) + AutoencoderKL.encode + latent_dist.sample() * sf.

    Returns (latent [B,4,H/8,W/8], skips[4]); skips are the INPUTS of down blocks 0..3 (model.py:18-20).
    ``eps`` replaces the global-RNG randn of DiagonalGaussianDistribution.sample (SURVEY fact 5)."""
    scales = scales or {}
    e = f"{prefix}encoder"
    ch = cfg["vae_channels"]
    s = conv2d(sd, f"{e}.conv_in", x, scales, padding=1)
    skips = []
    for i in range(len(ch)):
        skips.append(s)
        for j in range(cfg["vae_layers_per_block"]):
            s = _vae_resnet(sd, f"{e}.down_blocks.{i}.resnets.{j}", s, cfg, scales)
        if i < len(ch) - 1:
            s = F.pad(s, (0, 1, 0, 1))                                # Downsample2D, padding=0 variant
            s = conv2d(sd, f"{e}.down_blocks.{i}.downsamplers.0.conv", s, scales, stride=2)
    s = _vae_mid(sd, f"{e}.mid_block", s, cfg, scales)
    s = F.silu(group_norm(sd, f"{e}.conv_norm_out", s, cfg["vae_groups"], 1e-6))
    s = conv2d(sd, f"{e}.conv_out", s, scales, padding=1)
    moments = conv2d(sd, f"{prefix}quant_conv", s, scales)
    mean, logvar = moments.chunk(2, dim=1)
    logvar = logvar.clamp(-30.0, 20.0)
    z = mean + torch.exp(0.5 * logvar) * eps
    if stages is not None:
        stages.update(mean=mean, logvar=logvar, skips=skips)
    return z * cfg["scaling_factor"], skips


def vae_decode(sd: SD, prefix: str, z: torch.Tensor, skips, gamma: float = 1.0, cfg=SD_TURBO,
               scales: Optional[Dict[str, float]] = None, stages: Optional[dict] = None):
    """AutoencoderKL.decode(z) with my_vae_decoder_fwd (src/model.py:30-54); returns the PRE-clamp image."""
    scales = scales or {}
    d = f"{prefix}decoder"
    ch = cfg["vae_channels"]
    s = conv2d(sd, f"{prefix}post_quant_conv", z, scales)
    s = conv2d(sd, f"{d}.conv_in", s, scales, padding=1)
    s = _vae_mid(sd, f"{d}.mid_block", s, cfg, scales)
    for i in range(len(ch)):
        s = s + conv2d(sd, f"{d}.skip_conv_{i + 1}", skips[::-1][i] * gamma, scales)   # model.py:40-42
        for j in range(cfg["vae_layers_per_block"] + 1):
            s = _vae_resnet(sd, f"{d}.up_blocks.{i}.resnets.{j}", s, cfg, scales)
        if i < len(ch) - 1:
            s = F.interpolate(s, scale_factor=2.0, mode="nearest")
            s = conv2d(sd, f"{d}.up_blocks.{i}.upsamplers.0.conv", s, scales, padding=1)
    s = F.silu(group_norm(sd, f"{d}.conv_norm_out", s, cfg["vae_groups"], 1e-6))
    s = conv2d(sd, f"{d}.conv_out", s, scales, padding=1)
    if stages is not None:
        stages["pre_clamp"] = s
    return s


# ----------------------------------------------------------------------------------------------
# UNet2DConditionModel (diffusers models/unet_2d_condition.py, unet_2d_blocks.py, transformer_2d.py,
# attention.py, embeddings.py) for the SD-Turbo config
# ----------------------------------------------------------------------------------------------

def timestep_embedding(t: int, dim: int, dtype=torch.float32) -> torch.Tensor:
    """Timesteps(flip_sin_to_cos=True, freq_shift=0): [cos | sin] of t*exp(-ln(1e4) i/half)."""
    half = dim // 2
    f = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32) / half)
    a = float(t) * f
    return torch.cat([torch.cos(a), torch.sin(a)])[None].to(dtype)


def _unet_resnet(sd, p, x, emb_act, cfg, scales):
    g = cfg["unet_groups"]
    h = F.silu(group_norm(sd, f"{p}.norm1", x, g, 1e-5))
    h = conv2d(sd, f"{p}.conv1", h, scales, padding=1)
    h = h + linear(sd, f"{p}.time_emb_proj", emb_act, scales)[:, :, None, None]
    h = F.silu(group_norm(sd, f"{p}.norm2", h, g, 1e-5))
    h = conv2d(sd, f"{p}.conv2", h, scales, padding=1)
    if _base(sd, f"{p}.conv_shortcut", "weight") is not None:
        x = conv2d(sd, f"{p}.conv_shortcut", x, scales)
    return x + h


def _transformer(sd, p, x, text, heads, cfg, scales):
    B, C, H, W = x.shape
    r = x
    t = group_norm(sd, f"{p}.norm", x, cfg["unet_groups"], 1e-6)     # Transformer2DModel.norm: eps 1e-6, no SiLU
    t = t.permute(0, 2, 3, 1).reshape(B, H * W, C)
    t = linear(sd, f"{p}.proj_in", t, scales)
    b = f"{p}.transformer_blocks.0"
    n = layer_norm(sd, f"{b}.norm1", t)
    a = sdpa(linear(sd, f"{b}.attn1.to_q", n, scales), linear(sd, f"{b}.attn1.to_k", n, scales),
             linear(sd, f"{b}.attn1.to_v", n, scales), heads)
    t = t + linear(sd, f"{b}.attn1.to_out.0", a, scales)
    n = layer_norm(sd, f"{b}.norm2", t)
    a = sdpa(linear(sd, f"{b}.attn2.to_q", n, scales), linear(sd, f"{b}.attn2.to_k", text, scales),
             linear(sd, f"{b}.attn2.to_v", text, scales), heads)
    t = t + linear(sd, f"{b}.attn2.to_out.0", a, scales)
    n = layer_norm(sd, f"{b}.norm3", t)
    hg = linear(sd, f"{b}.ff.net.0.proj", n, scales)
    hh, gg = hg.chunk(2, dim=-1)
    t = t + linear(sd, f"{b}.ff.net.2", hh * F.gelu(gg), scales)     # GEGLU, erf GELU
    t = linear(sd, f"{p}.proj_out", t, scales)
    return t.reshape(B, H, W, C).permute(0, 3, 1, 2) + r


def unet_forward(sd: SD, prefix: str, z: torch.Tensor, text: torch.Tensor, cfg=SD_TURBO,
                 scales: Optional[Dict[str, float]] = None, twin_r: Optional[float] = None, t: int = 999):
    """eps_hat = UNet(z, t, text)  (call sites: src/pix2pix_turbo.py:199,212; src/cyclegan_turbo.py:204)."""
    scales = scales or {}
    u = prefix.rstrip(".")
    ch, heads, L = cfg["unet_channels"], cfg["unet_heads"], cfg["unet_layers_per_block"]
    B = z.shape[0]
    if text.shape[0] == 1 and B > 1:
        text = text.expand(B, -1, -1)
    te = timestep_embedding(t, ch[0], z.dtype)
    emb = linear(sd, f"{u}.time_embedding.linear_2",
                 F.silu(linear(sd, f"{u}.time_embedding.linear_1", te, scales)), scales)
    emb_act = F.silu(emb)
    if f"{u}.conv_in.conv_in_pretrained.weight" in sd:               # TwinConv, src/pix2pix_turbo.py:16-26
        x1 = conv2d(sd, f"{u}.conv_in.conv_in_pretrained", z, scales, padding=1)
        x2 = conv2d(sd, f"{u}.conv_in.conv_in_curr", z, scales, padding=1)
        s = x1 * (1 - twin_r) + x2 * twin_r
    else:
        s = conv2d(sd, f"{u}.conv_in", z, scales, padding=1)
    res = [s]
    nb = len(ch)
    for i in range(nb):
        for j in range(L):
            s = _unet_resnet(sd, f"{u}.down_blocks.{i}.resnets.{j}", s, emb_act, cfg, scales)
            if i < nb - 1:
                s = _transformer(sd, f"{u}.down_blocks.{i}.attentions.{j}", s, text, heads[i], cfg, scales)
            res.append(s)
        if i < nb - 1:
            s = conv2d(sd, f"{u}.down_blocks.{i}.downsamplers.0.conv", s, scales, stride=2, padding=1)
            res.append(s)
    s = _unet_resnet(sd, f"{u}.mid_block.resnets.0", s, emb_act, cfg, scales)
    s = _transformer(sd, f"{u}.mid_block.attentions.0", s, text, heads[-1], cfg, scales)
    s = _unet_resnet(sd, f"{u}.mid_block.resnets.1", s, emb_act, cfg, scales)
    rheads = heads[::-1]
    # diffusers UNet2DConditionModel.forward: if any latent dim is not a multiple of 2**num_upsamplers, every non-final up block
    # is told the spatial size of the next skip connection (`upsample_size = down_block_res_samples[-1].shape[2:]`) and
    # Upsample2D interpolates to that size instead of by a factor 2 (models/resnet.py Upsample2D.forward: output_size)
    forward_upsample_size = any(d % (2 ** (nb - 1)) != 0 for d in z.shape[-2:])
    for i in range(nb):
        for j in range(L + 1):
            s = torch.cat([s, res.pop()], dim=1)
            s = _unet_resnet(sd, f"{u}.up_blocks.{i}.resnets.{j}", s, emb_act, cfg, scales)
            if i > 0:
                s = _transformer(sd, f"{u}.up_blocks.{i}.attentions.{j}", s, text, rheads[i], cfg, scales)
        if i < nb - 1:
            if forward_upsample_size:
                s = F.interpolate(s, size=tuple(res[-1].shape[2:]), mode="nearest")
            else:
                s = F.interpolate(s, scale_factor=2.0, mode="nearest")
            s = conv2d(sd, f"{u}.up_blocks.{i}.upsamplers.0.conv", s, scales, padding=1)
    assert not res
    s = F.silu(group_norm(sd, f"{u}.conv_norm_out", s, cfg["unet_groups"], 1e-5))
    return conv2d(sd, f"{u}.conv_out", s, scales, padding=1)


# ----------------------------------------------------------------------------------------------
# the two wrappers' forward recipes
# ----------------------------------------------------------------------------------------------

def pix2pix_forward(sd: SD, c_t: torch.Tensor, text: torch.Tensor, eps: torch.Tensor, cfg=SD_TURBO,
                    deterministic: bool = True, r: float = 1.0, noise_map: Optional[torch.Tensor] = None,
                    lora_alpha_unet: float = 8.0, rank_unet: int = 8, lora_alpha_vae: float = 8.0,
                    rank_vae: int = 4, lora_weight: float = 1.0, decoder_gamma: float = 1.0,
                    stages: Optional[dict] = None) -> torch.Tensor:
    """Pix2Pix_Turbo.forward (src/pix2pix_turbo.py:186-219).  Returns the clamped image [B,3,H,W].

    deterministic: LoRA runtime weights / decoder.gamma are whatever state the module is in
    (``lora_weight``, ``decoder_gamma``; 1 after construction).  stochastic: both become ``r``
    (:206-207,:217), unet_input = enc*r + noise*(1-r) (:210), TwinConv blend r (:211)."""
    lw = lora_weight if deterministic else r
    scales = {"default": lora_alpha_unet / rank_unet * lw, "vae_skip": lora_alpha_vae / rank_vae * lw}
    st = stages if stages is not None else {}
    enc, skips = vae_encode(sd, "vae.", c_t, eps, cfg, scales, st)
    if deterministic:
        z_in, gamma, twin = enc, decoder_gamma, None
    else:
        z_in, gamma, twin = enc * r + noise_map * (1 - r), r, r
    pred = unet_forward(sd, "unet.", z_in, text, cfg, scales, twin_r=twin)
    x0 = ddpm_step_x0(pred, z_in, 999, torch.float32)
    img = vae_decode(sd, "vae.", x0 / cfg["scaling_factor"], skips, gamma, cfg, scales, st)
    st.update(latent=enc, unet_in=z_in, model_pred=pred, x_denoised=x0)
    return img.clamp(-1, 1)


def cyclegan_forward(sd: SD, x: torch.Tensor, text: torch.Tensor, eps: torch.Tensor, direction: str = "a2b",
                     cfg=SD_TURBO, rank_vae: int = 4, lora_alpha_vae: float = 8.0,
                     stages: Optional[dict] = None) -> torch.Tensor:
    """CycleGAN_Turbo.forward_with_networks (src/cyclegan_turbo.py:199-207) with timesteps=[999]*B and the
    caption embedding broadcast over the batch (SURVEY fact 8).  UNet adapters have lora_alpha == rank
    (scale 1, :66-68); the VAE adapter keeps peft's default alpha 8 (scale 8/rank_vae, :101)."""
    assert direction in ("a2b", "b2a")
    vp = "vae." if direction == "a2b" else "vae_b2a."
    scales = {"default_encoder": 1.0, "default_decoder": 1.0, "default_others": 1.0,
              "vae_skip": lora_alpha_vae / rank_vae}
    st = stages if stages is not None else {}
    enc, skips = vae_encode(sd, vp, x, eps, cfg, scales, st)
    enc = enc.to(x.dtype)
    pred = unet_forward(sd, "unet.", enc, text, cfg, scales)
    x0 = ddpm_step_x0(pred, enc, 999, None if x.dtype != torch.float32 else torch.float32)
    img = vae_decode(sd, vp, x0 / cfg["scaling_factor"], skips, 1.0, cfg, scales, st)
    st.update(latent=enc, model_pred=pred, x_denoised=x0)
    return img.clamp(-1, 1)


# ----------------------------------------------------------------------------------------------
# algebra used by the product at load time, restated here so tests can check the fold itself
# ----------------------------------------------------------------------------------------------

def fold_lora(sd: SD, name: str, scales: Dict[str, float]) -> torch.Tensor:
    """W' = W + sum_a s_a * (B_a @ A_a)   (Linear)   /   W'[o,i,:,:] += s_a * sum_r B[o,r] A[r,i,:,:] (Conv)."""
    w = _base(sd, name, "weight").float().clone()
    for a in _adapters(sd, name):
        s = scales.get(a, 0.0)
        A, Bm = sd[f"{name}.lora_A.{a}.weight"].float(), sd[f"{name}.lora_B.{a}.weight"].float()
        if w.dim() == 2:
            w += s * (Bm @ A)
        else:
            w += s * torch.einsum("or,rikl->oikl", Bm[:, :, 0, 0], A)
    return w
