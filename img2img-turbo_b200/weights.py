"""Weight inventory + seeded random initialisation in diffusers/peft key naming.

The reference builds its networks with ``from_pretrained("stabilityai/sd-turbo")`` and then installs
LoRA adapters / skip convs (src/pix2pix_turbo.py:32-45,131-155;
src/cyclegan_turbo.py:48-106).  Offline there are no SD-Turbo weights, so the
``pretrained_name=None, pretrained_path=None`` branch (pix2pix_turbo.py:131) is the one every
BASELINE config uses: PyTorch default layer init for the base model, LoRA "gaussian" init for
lora_A, skip convs = 1e-5.  ``lora_B`` is drawn N(0, 0.02^2) instead of the default zeros so the
load-time fold is actually exercised (BASELINE.md section 3).

Key layout: "<model>.<diffusers key>" with model in {"unet", "vae", "vae_b2a"}; LoRA-wrapped layers carry
"X.lora_A.<adapter>.weight" / "X.lora_B.<adapter>.weight" next to the base "X.weight"/"X.bias"
(the loader also accepts peft's "X.base_layer.weight").
"""
from __future__ import annotations

import math
from typing import Dict, Iterator, List, Optional, Tuple

import torch

SD_TURBO = dict(
    unet_channels=(320, 640, 1280, 1280),
    unet_heads=(5, 10, 20, 20),
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

# A structurally identical but narrow network for fast CPU/GPU parity tests.
TINY = dict(
    unet_channels=(64, 128, 256, 256),
    unet_heads=(1, 2, 4, 4),
    unet_layers_per_block=2,
    cross_dim=128,
    temb_dim=256,
    unet_groups=32,
    vae_channels=(64, 64, 128, 128),
    vae_layers_per_block=2,
    vae_groups=32,
    latent_channels=4,
    scaling_factor=0.18215,
)

# LoRA target lists of the random-init branch (src/pix2pix_turbo.py:137-147)
TARGETS_VAE = ["conv1", "conv2", "conv_in", "conv_shortcut", "conv", "conv_out",
               "skip_conv_1", "skip_conv_2", "skip_conv_3", "skip_conv_4",
               "to_k", "to_q", "to_v", "to_out.0"]
TARGETS_UNET = ["to_k", "to_q", "to_v", "to_out.0", "conv", "conv1", "conv2", "conv_shortcut", "conv_out",
                "proj_in", "proj_out", "ff.net.2", "ff.net.0.proj"]
# substring patterns of CycleGAN-Turbo's initialize_unet (src/cyclegan_turbo.py:53)
GREP_CYCLEGAN = ["to_k", "to_q", "to_v", "to_out.0", "conv", "conv1", "conv2", "conv_in", "conv_shortcut",
                 "conv_out", "proj_out", "proj_in", "ff.net.2", "ff.net.0.proj"]

Spec = Tuple[str, str, tuple]   # (key without model prefix, kind, shape); kind in conv|linear|norm


def _resnet(p, cin, cout, temb=None) -> Iterator[Spec]:
    yield f"{p}.norm1", "norm", (cin,)
    yield f"{p}.conv1", "conv", (cout, cin, 3, 3)
    if temb:
        yield f"{p}.time_emb_proj", "linear", (cout, temb)
    yield f"{p}.norm2", "norm", (cout,)
    yield f"{p}.conv2", "conv", (cout, cout, 3, 3)
    if cin != cout:
        yield f"{p}.conv_shortcut", "conv", (cout, cin, 1, 1)


def _vae_attn(p, c) -> Iterator[Spec]:
    yield f"{p}.group_norm", "norm", (c,)
    for n in ("to_q", "to_k", "to_v", "to_out.0"):
        yield f"{p}.{n}", "linear", (c, c)


def vae_specs(cfg) -> List[Spec]:
    ch, L, lat = cfg["vae_channels"], cfg["vae_layers_per_block"], cfg["latent_channels"]
    out: List[Spec] = [("encoder.conv_in", "conv", (ch[0], 3, 3, 3))]
    prev = ch[0]
    for i, c in enumerate(ch):
        for j in range(L):
            out += _resnet(f"encoder.down_blocks.{i}.resnets.{j}", prev, c)
            prev = c
        if i < len(ch) - 1:
            out.append((f"encoder.down_blocks.{i}.downsamplers.0.conv", "conv", (c, c, 3, 3)))
    out += _resnet("encoder.mid_block.resnets.0", prev, prev)
    out += _vae_attn("encoder.mid_block.attentions.0", prev)
    out += _resnet("encoder.mid_block.resnets.1", prev, prev)
    out += [("encoder.conv_norm_out", "norm", (prev,)), ("encoder.conv_out", "conv", (2 * lat, prev, 3, 3)),
            ("quant_conv", "conv", (2 * lat, 2 * lat, 1, 1)), ("post_quant_conv", "conv", (lat, lat, 1, 1))]
    rch = ch[::-1]
    prev = rch[0]
    out.append(("decoder.conv_in", "conv", (prev, lat, 3, 3)))
    out += _resnet("decoder.mid_block.resnets.0", prev, prev)
    out += _vae_attn("decoder.mid_block.attentions.0", prev)
    out += _resnet("decoder.mid_block.resnets.1", prev, prev)
    for i, c in enumerate(rch):
        for j in range(L + 1):
            out += _resnet(f"decoder.up_blocks.{i}.resnets.{j}", prev, c)
            prev = c
        if i < len(ch) - 1:
            out.append((f"decoder.up_blocks.{i}.upsamplers.0.conv", "conv", (c, c, 3, 3)))
    out += [("decoder.conv_norm_out", "norm", (prev,)), ("decoder.conv_out", "conv", (3, prev, 3, 3))]
    return out


def skip_conv_shapes(cfg):
    """(cin, cout) of decoder.skip_conv_1..4 (src/pix2pix_turbo.py:40-43): skips reversed -> up-block inputs."""
    ch = cfg["vae_channels"]
    skip_c = [ch[0]] + list(ch[:-1])            # channels of encoder skips 0..3 (inputs of down blocks)
    rch = ch[::-1]
    up_in = [rch[0]] + list(rch[:-1])           # input channels of decoder up blocks 0..3
    return [(skip_c[::-1][i], up_in[i]) for i in range(len(ch))]


def _xformer(p, c, cross) -> Iterator[Spec]:
    yield f"{p}.norm", "norm", (c,)
    yield f"{p}.proj_in", "linear", (c, c)
    b = f"{p}.transformer_blocks.0"
    yield f"{b}.norm1", "norm", (c,)
    for n in ("to_q", "to_k", "to_v"):
        yield f"{b}.attn1.{n}", "linear_nobias", (c, c)
    yield f"{b}.attn1.to_out.0", "linear", (c, c)
    yield f"{b}.norm2", "norm", (c,)
    yield f"{b}.attn2.to_q", "linear_nobias", (c, c)
    yield f"{b}.attn2.to_k", "linear_nobias", (c, cross)
    yield f"{b}.attn2.to_v", "linear_nobias", (c, cross)
    yield f"{b}.attn2.to_out.0", "linear", (c, c)
    yield f"{b}.norm3", "norm", (c,)
    yield f"{b}.ff.net.0.proj", "linear", (8 * c, c)
    yield f"{b}.ff.net.2", "linear", (c, 4 * c)
    yield f"{p}.proj_out", "linear", (c, c)


def unet_specs(cfg, twin: bool = False) -> List[Spec]:
    ch, L, T, X, lat = (cfg["unet_channels"], cfg["unet_layers_per_block"], cfg["temb_dim"],
                        cfg["cross_dim"], cfg["latent_channels"])
    out: List[Spec] = [("time_embedding.linear_1", "linear", (T, ch[0])),
                       ("time_embedding.linear_2", "linear", (T, T))]
    if twin:
        out += [("conv_in.conv_in_pretrained", "conv", (ch[0], lat, 3, 3)),
                ("conv_in.conv_in_curr", "conv", (ch[0], lat, 3, 3))]
    else:
        out.append(("conv_in", "conv", (ch[0], lat, 3, 3)))
    nb = len(ch)
    skips = [ch[0]]
    prev = ch[0]
    for i, c in enumerate(ch):
        for j in range(L):
            out += _resnet(f"down_blocks.{i}.resnets.{j}", prev, c, T)
            prev = c
            if i < nb - 1:
                out += _xformer(f"down_blocks.{i}.attentions.{j}", c, X)
            skips.append(c)
        if i < nb - 1:
            out.append((f"down_blocks.{i}.downsamplers.0.conv", "conv", (c, c, 3, 3)))
            skips.append(c)
    out += _resnet("mid_block.resnets.0", prev, prev, T)
    out += _xformer("mid_block.attentions.0", prev, X)
    out += _resnet("mid_block.resnets.1", prev, prev, T)
    rch = ch[::-1]
    for i, c in enumerate(rch):
        for j in range(L + 1):
            out += _resnet(f"up_blocks.{i}.resnets.{j}", prev + skips.pop(), c, T)
            prev = c
            if i > 0:
                out += _xformer(f"up_blocks.{i}.attentions.{j}", c, X)
        if i < nb - 1:
            out.append((f"up_blocks.{i}.upsamplers.0.conv", "conv", (c, c, 3, 3)))
    assert not skips
    out += [("conv_norm_out", "norm", (prev,)), ("conv_out", "conv", (lat, prev, 3, 3))]
    return out


def param_count(specs: List[Spec]) -> int:
    n = 0
    for _, kind, shape in specs:
        numel = math.prod(shape)
        if kind == "norm":
            n += 2 * numel
        elif kind == "linear_nobias":
            n += numel
        else:
            n += numel + shape[0]
    return n


def _suffix_match(key: str, targets: List[str]) -> bool:
    """peft target_modules list semantics: exact name or '.<target>' suffix."""
    return any(key == t or key.endswith("." + t) for t in targets)


def unet_adapter_for(key: str, model_kind: str) -> Optional[str]:
    """Which LoRA adapter wraps UNet layer ``key`` (None = not wrapped)."""
    if model_kind == "pix2pix":
        return "default" if _suffix_match(key, TARGETS_UNET) else None
    # CycleGAN: substring grep over parameter names, skipping biases and norms (cyclegan_turbo.py:54-65)
    n = key + ".weight"
    if "norm" in n or not any(p in n for p in GREP_CYCLEGAN):
        return None
    if "down_blocks" in n or "conv_in" in n:
        return "default_encoder"
    if "up_blocks" in n:
        return "default_decoder"
    return "default_others"


def make_state_dict(kind: str = "pix2pix", cfg=SD_TURBO, seed: int = 0, twin: bool = False,
                    lora_rank_unet: int = 8, lora_rank_vae: int = 4, lora_b_std: float = 0.02,
                    perturb_norm: bool = False, dtype=torch.float32) -> Dict[str, torch.Tensor]:
    """Seeded CPU random init of every tensor on the path (deterministic across machines for a given torch)."""
    assert kind in ("pix2pix", "cyclegan")
    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}

    def uni(shape, bound):
        return torch.empty(shape, dtype=dtype).uniform_(-bound, bound, generator=g)

    def nrm(shape, std, mean=0.0):
        return torch.empty(shape, dtype=dtype).normal_(mean, std, generator=g)

    def add_layer(model, key, k, shape, adapter, rank):
        name = f"{model}.{key}"
        if k == "norm":
            sd[name + ".weight"] = nrm(shape, 0.1, 1.0) if perturb_norm else torch.ones(shape, dtype=dtype)
            sd[name + ".bias"] = nrm(shape, 0.05) if perturb_norm else torch.zeros(shape, dtype=dtype)
            return
        fan_in = math.prod(shape[1:])
        bound = 1.0 / math.sqrt(fan_in)
        sd[name + ".weight"] = uni(shape, bound)
        if k != "linear_nobias":
            sd[name + ".bias"] = uni((shape[0],), bound)
        if adapter is not None:
            a_shape = (rank,) + tuple(shape[1:])
            b_shape = (shape[0], rank) + ((1, 1) if len(shape) == 4 else ())
            sd[f"{name}.lora_A.{adapter}.weight"] = nrm(a_shape, 1.0 / rank)
            sd[f"{name}.lora_B.{adapter}.weight"] = nrm(b_shape, lora_b_std)

    for key, k, shape in unet_specs(cfg, twin):
        add_layer("unet", key, k, shape, unet_adapter_for(key, kind), lora_rank_unet)
    vaes = ["vae"] if kind == "pix2pix" else ["vae", "vae_b2a"]
    for model in vaes:
        for key, k, shape in vae_specs(cfg):
            ad = "vae_skip" if (k != "norm" and _suffix_match(key, TARGETS_VAE)) else None
            add_layer(model, key, k, shape, ad, lora_rank_vae)
        for i, (cin, cout) in enumerate(skip_conv_shapes(cfg)):
            name = f"{model}.decoder.skip_conv_{i + 1}"
            sd[name + ".weight"] = torch.full((cout, cin, 1, 1), 1e-5, dtype=dtype)
            sd[f"{name}.lora_A.vae_skip.weight"] = nrm((lora_rank_vae, cin, 1, 1), 1.0 / lora_rank_vae)
            sd[f"{name}.lora_B.vae_skip.weight"] = nrm((cout, lora_rank_vae, 1, 1), lora_b_std)
    return sd
