"""Drop-in mirror of src/cyclegan_turbo.py (CycleGAN_Turbo, VAE_encode, VAE_decode) over libi2it.

Same constructor kwargs / attributes / forward signatures, so src/inference_unpaired.py runs unchanged
(`model.eval()`, `model.unet.enable_xformers_memory_efficient_attention()`, `model.half()`,
`model(x_t, direction=..., caption=...)`).  The whole of forward_with_networks (cyclegan_turbo.py:199-207) is one
i2it_forward call; batches > 1 work (the reference indexes timesteps[i] of a length-1 tensor and is B=1-only).
"""
from __future__ import annotations

import os
import sys
import warnings
from types import SimpleNamespace

import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import i2it  # noqa: E402
import weights as W  # noqa: E402
import _host  # noqa: E402
from _host import NetHandle, TurboBase, load_sd_turbo_base  # noqa: E402
from model import download_url  # noqa: E402

PRETRAINED = {   # name -> (url, caption, direction)   reference cyclegan_turbo.py:126-149
    "day_to_night": ("https://www.cs.cmu.edu/~img2img-turbo/models/day2night.pkl", "driving in the night", "a2b"),
    "night_to_day": ("https://www.cs.cmu.edu/~img2img-turbo/models/night2day.pkl", "driving in the day", "b2a"),
    "clear_to_rainy": ("https://www.cs.cmu.edu/~img2img-turbo/models/clear2rainy.pkl", "driving in heavy rain", "a2b"),
    "rainy_to_clear": ("https://www.cs.cmu.edu/~img2img-turbo/models/rainy2clear.pkl", "driving in the day", "b2a"),
}


class VAE_encode(nn.Module):
    """Direction-selecting encoder handle (reference :15-27).  Encoding itself is fused into i2it_forward."""

    def __init__(self, vae, vae_b2a=None, owner=None):
        super().__init__()
        self.__dict__["vae"], self.__dict__["vae_b2a"], self.__dict__["owner"] = vae, vae_b2a, owner

    def forward(self, x, direction):
        assert direction in ["a2b", "b2a"]
        raise RuntimeError("VAE_encode is fused with the UNet step and the decoder inside libi2it; call "
                           "CycleGAN_Turbo.forward / forward_with_networks")


class VAE_decode(nn.Module):
    """Direction-selecting decoder handle (reference :30-45)."""

    def __init__(self, vae, vae_b2a=None, owner=None):
        super().__init__()
        self.__dict__["vae"], self.__dict__["vae_b2a"], self.__dict__["owner"] = vae, vae_b2a, owner

    def forward(self, x, direction):
        assert direction in ["a2b", "b2a"]
        raise RuntimeError("VAE_decode is fused into libi2it; call CycleGAN_Turbo.forward / forward_with_networks")


class CycleGAN_Turbo(TurboBase):
    MODEL_KIND = i2it.CYCLEGAN

    def __init__(self, pretrained_name=None, pretrained_path=None, ckpt_folder="checkpoints", lora_rank_unet=8,
                 lora_rank_vae=4, *, cfg=None, seed=0, lora_b_std=0.02, perturb_norm=False, text_stack=None,
                 use_cuda_graph=True, keep_stages=False, synthetic_caption=None, synthetic_direction=None,
                 allow_synthetic_weights=False):
        super().__init__()
        self._init_common(cfg, None, text_stack, use_cuda_graph, keep_stages)
        ckpt = None
        self.caption, self.direction = None, None
        if pretrained_name is not None:
            if pretrained_name not in PRETRAINED:
                raise ValueError(f"unknown pretrained_name {pretrained_name!r}")
            url, self.caption, self.direction = PRETRAINED[pretrained_name]
            os.makedirs(ckpt_folder, exist_ok=True)
            outf = os.path.join(ckpt_folder, os.path.basename(url))
            try:
                download_url(url, outf)
                ckpt = torch.load(outf, map_location="cpu")
            except Exception as ex:
                # A named pretrained model on random weights produces garbage images: refuse unless explicitly asked for
                # (offline synthetic benchmarks pass allow_synthetic_weights=True and keep the caption/direction).
                if not allow_synthetic_weights:
                    raise RuntimeError(f"could not load the {pretrained_name!r} checkpoint from {url} ({type(ex).__name__}: {ex}); "
                                       "pass allow_synthetic_weights=True to run the named configuration on seeded random "
                                       "weights (benchmarks only)") from ex
                warnings.warn(f"checkpoint {url} unreachable ({type(ex).__name__}); using seeded random weights "
                              "(allow_synthetic_weights=True)")
        elif pretrained_path is not None:
            ckpt = torch.load(pretrained_path, map_location="cpu")
        else:
            # the reference has no random-init branch for this class; offline synthetic benchmarks need one
            self.caption, self.direction = synthetic_caption, synthetic_direction
        if ckpt is not None:
            lora_rank_unet, lora_rank_vae = ckpt["rank_unet"], ckpt["rank_vae"]
        self._sd = W.make_state_dict("cyclegan", self._cfg, seed=seed, lora_rank_unet=lora_rank_unet,
                                     lora_rank_vae=lora_rank_vae, lora_b_std=lora_b_std, perturb_norm=perturb_norm)
        have_base = load_sd_turbo_base(self._sd, ["unet", "vae", "vae_b2a"]) if self._cfg is W.SD_TURBO else False
        if ckpt is not None:
            if not have_base:
                warnings.warn("SD-Turbo base weights are not available offline: checkpoint tensors are applied on top of a "
                              "seeded random base (set $I2IT_SD_TURBO_DIR for real outputs)")
            self.load_ckpt_from_state_dict(ckpt)
        # lora_alpha == rank for the three UNet adapters (:66-68) -> scale 1; VAE adapter keeps peft's default alpha 8
        self._adapter_scales = {"default_encoder": 1.0, "default_decoder": 1.0, "default_others": 1.0,
                                "vae_skip": 8.0 / lora_rank_vae}
        self.unet, self.vae, self.vae_b2a = NetHandle(self, "unet."), NetHandle(self, "vae."), NetHandle(self, "vae_b2a.")
        for v in (self.vae, self.vae_b2a):
            v.decoder = SimpleNamespace(gamma=1, ignore_skip=False)
            v.config = SimpleNamespace(scaling_factor=self._cfg["scaling_factor"])
        self.vae_enc = VAE_encode(self.vae, self.vae_b2a, owner=self)
        self.vae_dec = VAE_decode(self.vae, self.vae_b2a, owner=self)

    # ---- checkpoint format written by train_cyclegan_turbo.py:293-307, read at cyclegan_turbo.py:162-190 ----
    def load_ckpt_from_state_dict(self, sd):
        # adapters exist only where the checkpoint has them (reference :163-183 builds the LoraConfigs from the checkpoint's
        # target lists): drop the seeded ones first so no layer keeps a random, never-trained adapter
        for k in [k for k in self._sd if ".lora_A." in k or ".lora_B." in k]:
            del self._sd[k]
        for part, adapter in (("sd_encoder", "default_encoder"), ("sd_decoder", "default_decoder"), ("sd_other", "default_others")):
            for k, v in sd[part].items():
                k2 = k.replace(".lora_A.weight", f".lora_A.{adapter}.weight").replace(".lora_B.weight", f".lora_B.{adapter}.weight")
                self._sd["unet." + k2] = v.detach().float().cpu()
        for part in ("sd_vae_enc", "sd_vae_dec"):
            for k, v in sd[part].items():          # keys already carry "vae." / "vae_b2a." (VAE_encode/VAE_decode state dicts)
                self._sd[k.replace(".base_layer.", ".")] = v.detach().float().cpu()
        self._invalidate()

    def load_ckpt_from_url(self, url, ckpt_folder):
        os.makedirs(ckpt_folder, exist_ok=True)
        outf = os.path.join(ckpt_folder, os.path.basename(url))
        download_url(url, outf)
        self.load_ckpt_from_state_dict(torch.load(outf, map_location="cpu"))

    def _set_adapter_weights(self, prefix, names, weights):
        pass   # all three adapters stay active with weight 1 (reference :72,181)

    def _run(self, x, direction, text_emb, eps=None):
        assert direction in ["a2b", "b2a"]
        dt = self.compute_dtype
        in_dtype = x.dtype
        B, _, H, Wd = x.shape
        xd = self._prep(x, dt)
        if eps is None:
            eps = torch.randn((B, 4, H // 8, Wd // 8), device=_host.DEVICE, dtype=dt)   # latent_dist.sample()
        eps = self._prep(eps, dt)
        text = self._prep(text_emb, dt)
        if text.shape[0] not in (1, B):
            raise ValueError("caption embedding batch must be 1 or match the image batch")
        eng = self._finalize(1.0, 1.0, 1.0, -1.0)
        out = self._staged_forward(eng, xd, text, eps, direction=i2it.A2B if direction == "a2b" else i2it.B2A)
        return out if in_dtype == dt else out.to(in_dtype)

    @staticmethod
    def forward_with_networks(x, direction, vae_enc, unet, vae_dec, sched, timesteps, text_emb, eps=None):
        """Reference :199-207.  `vae_enc` must be the VAE_encode of a CycleGAN_Turbo built by this module; the UNet,
        scheduler and decoder that run are that model's (fused on device)."""
        assert direction in ["a2b", "b2a"]
        owner = getattr(vae_enc, "owner", None)
        if owner is None:
            raise RuntimeError("forward_with_networks needs the VAE_encode handle of an i2it CycleGAN_Turbo")
        return owner._run(x, direction, text_emb, eps)

    @staticmethod
    def get_traininable_params(unet, vae_a2b, vae_b2a):
        raise NotImplementedError("training is outside this build's scope (inference hot path only)")

    def forward(self, x_t, direction=None, caption=None, caption_emb=None, *, eps=None):
        if direction is None:
            assert self.direction is not None
            direction = self.direction
        if caption is None and caption_emb is None:
            assert self.caption is not None
            caption = self.caption
        if caption_emb is not None:
            caption_enc = caption_emb
        else:
            caption_enc = self._encode_text(caption)
        return self.forward_with_networks(x_t, direction, self.vae_enc, self.unet, self.vae_dec, self.sched, self.timesteps,
                                          caption_enc, eps)

    def forward_u8(self, images_u8, direction=None, caption=None, caption_emb=None, *, eps=None):
        """uint8 HWC boundary (SURVEY 8f #3): [B,H,W,3] uint8 -> [B,H,W,3] uint8 CUDA tensor.  Fuses ToTensor + Normalize([0.5],[0.5])
        (inference_unpaired.py:45-47) and ToPILImage()(out*0.5+0.5) (:53) around the same fused forward."""
        if direction is None:
            assert self.direction is not None
            direction = self.direction
        if caption is None and caption_emb is None:
            assert self.caption is not None
            caption = self.caption
        assert direction in ["a2b", "b2a"]
        dt = self.compute_dtype
        text = self._prep(caption_emb if caption_emb is not None else self._encode_text(caption), dt)
        x = images_u8.to(device=_host.DEVICE, non_blocking=True).contiguous()
        B, H, Wd, _ = x.shape
        if eps is None:
            eps = torch.randn((B, 4, H // 8, Wd // 8), device=_host.DEVICE, dtype=dt)
        eps = self._prep(eps, dt)
        eng = self._finalize(1.0, 1.0, 1.0, -1.0)
        return self._staged_forward(eng, x, text, eps, direction=i2it.A2B if direction == "a2b" else i2it.B2A,
                                    u8_mode=i2it.IN_NORMALIZE)
