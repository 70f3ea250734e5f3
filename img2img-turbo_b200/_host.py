"""Host-side plumbing shared by the two reference-API mirrors (pix2pix_turbo.py / cyclegan_turbo.py).

Nothing here computes on the image path: it builds/loads state dicts, encodes prompts with the stock
transformers CLIP text tower (adjacent to, not on, the accelerated path — SURVEY.md section 8f #1), and drives
libi2it through i2it.Engine.
"""
from __future__ import annotations

import hashlib
import os
import warnings
from types import SimpleNamespace
from typing import Dict, List, Optional

import torch

import i2it
import weights as W

SD_TURBO_DIR_ENV = "I2IT_SD_TURBO_DIR"      # optional local snapshot of stabilityai/sd-turbo (offline boxes)
DEVICE = "cuda"      # where the wrappers stage tensors (the engine runs on the current CUDA device)


def _cur_dev() -> int:
    return torch.cuda.current_device() if torch.cuda.is_available() else -1


# ------------------------------------------------------------------------------------------------
# scheduler mirror: make_1step_sched() of src/model.py:7-11, as closed-form constants
# ------------------------------------------------------------------------------------------------
class OneStepDDPM:
    """DDPMScheduler(scaled_linear 0.00085->0.012, 1000 steps, trailing, 1 inference step) reduced to t=999."""

    def __init__(self):
        betas = torch.linspace(0.00085 ** 0.5, 0.012 ** 0.5, 1000, dtype=torch.float32) ** 2
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.timesteps = torch.tensor([999]).long()
        self.config = SimpleNamespace(num_train_timesteps=1000, prediction_type="epsilon", timestep_spacing="trailing")

    def set_timesteps(self, n, device=None):
        assert n == 1, "the one-step path only supports a single inference step"

    def step(self, model_output, timestep, sample, return_dict=True):
        """Closed form x0 (prev alpha_bar = 1).  Provided for API parity; the engine fuses this step on device."""
        ac = self.alphas_cumprod[int(timestep)].to(torch.float32)
        x0 = (sample.float() - (1 - ac).sqrt() * model_output.float()) / ac.sqrt()
        return SimpleNamespace(prev_sample=x0, pred_original_sample=x0)


# ------------------------------------------------------------------------------------------------
# tokenizer / text encoder (stock transformers; falls back to seeded random init offline)
# ------------------------------------------------------------------------------------------------
class HashTokenizer:
    """Offline stand-in used ONLY when no CLIP tokenizer files are reachable: deterministic word hashing into the
    CLIP vocabulary with BOS/EOS and max_length padding.  Keeps the call signature the wrappers use."""
    model_max_length = 77
    bos, eos, vocab = 49406, 49407, 49408

    def __call__(self, text, max_length=77, padding="max_length", truncation=True, return_tensors="pt"):
        texts = [text] if isinstance(text, str) else list(text)
        rows = []
        for t in texts:
            ids = [int(hashlib.md5(w.encode()).hexdigest(), 16) % (self.bos - 1) + 1 for w in t.lower().split()]
            ids = [self.bos] + ids[: max_length - 2] + [self.eos]
            rows.append(ids + [self.eos] * (max_length - len(ids)))
        return SimpleNamespace(input_ids=torch.tensor(rows, dtype=torch.long))


def build_text_stack(cross_dim: int = 1024, seed: int = 1234):
    """(tokenizer, text_encoder).  Mirrors src/pix2pix_turbo.py:32-33."""
    from transformers import CLIPTextConfig, CLIPTextModel
    local = os.environ.get(SD_TURBO_DIR_ENV)
    srcs = ([local] if local else []) + ["stabilityai/sd-turbo"]
    for src in srcs:
        try:
            from transformers import AutoTokenizer
            tok = AutoTokenizer.from_pretrained(src, subfolder="tokenizer")
            enc = CLIPTextModel.from_pretrained(src, subfolder="text_encoder")
            return tok, enc
        except Exception:
            continue
    warnings.warn("stabilityai/sd-turbo tokenizer/text_encoder unreachable (offline): using a seeded random-init CLIP text "
                  "tower and a hash tokenizer — fine for synthetic benchmarks, meaningless for real prompts")
    if cross_dim == 1024:
        cfg = CLIPTextConfig(vocab_size=49408, hidden_size=1024, intermediate_size=4096, num_hidden_layers=23,
                             num_attention_heads=16, max_position_embeddings=77, hidden_act="gelu", projection_dim=512)
    else:   # reduced configs used by tests
        cfg = CLIPTextConfig(vocab_size=49408, hidden_size=cross_dim, intermediate_size=2 * cross_dim, num_hidden_layers=2,
                             num_attention_heads=max(1, cross_dim // 64), max_position_embeddings=77, hidden_act="gelu")
    st = torch.random.get_rng_state()
    torch.manual_seed(seed)
    enc = CLIPTextModel(cfg)
    torch.random.set_rng_state(st)
    return HashTokenizer(), enc


# ------------------------------------------------------------------------------------------------
# light-weight stand-ins for the diffusers module objects the reference exposes as .unet / .vae
# ------------------------------------------------------------------------------------------------
class NetHandle:
    """What `model.unet` / `model.vae` are here: a view of the state dict plus the handful of methods the
    reference's callers use (.eval(), .train(), .requires_grad_(), .to(), .cuda(), .state_dict(),
    .enable_xformers_memory_efficient_attention())."""

    def __init__(self, owner, prefix: str):
        self._owner, self._prefix = owner, prefix
        self.training = False

    def state_dict(self) -> Dict[str, torch.Tensor]:
        p = self._prefix
        return {k[len(p):]: v for k, v in self._owner._sd.items() if k.startswith(p)}

    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        for k, v in sd.items():
            self._owner._sd[self._prefix + k] = v.detach().float().cpu()
        self._owner._invalidate()

    def named_parameters(self):
        return iter(self.state_dict().items())

    def parameters(self):
        return iter(self.state_dict().values())

    def eval(self):
        self.training = False
        return self

    def train(self, mode: bool = True):
        self.training = mode
        return self

    def requires_grad_(self, flag: bool = True):
        return self

    def to(self, *a, **k):
        return self

    def cuda(self, *a, **k):
        return self

    def enable_xformers_memory_efficient_attention(self, *a, **k):
        # src/inference_unpaired.py:36 calls this; attention here is already a fused tensor-core path
        return self

    def set_adapters(self, names, weights=None):
        self._owner._set_adapter_weights(self._prefix, names, weights)


class TurboBase(torch.nn.Module):
    """Common engine management for the two wrappers."""
    MODEL_KIND = i2it.PIX2PIX

    def _init_common(self, cfg, dtype, text_stack, use_cuda_graph=True, keep_stages=False):
        # I2IT_CFG=tiny: reduced-width network when the caller cannot pass `cfg` (e.g. an unmodified inference script under test);
        # the default is always the SD-Turbo geometry
        if cfg is None and os.environ.get("I2IT_CFG") == "tiny":
            cfg = W.TINY
        self._cfg = cfg or W.SD_TURBO
        self._dtype = dtype                      # None until .half()/.bfloat16()/.to(dtype); engine default bf16
        self._engine: Optional[i2it.Engine] = None
        self._engine_key = None
        self._final_key = None
        self._use_graph, self._keep_stages = use_cuda_graph, keep_stages
        self._text_cache: Dict[object, torch.Tensor] = {}
        if text_stack is None:
            text_stack = build_text_stack(self._cfg["cross_dim"])
        self.tokenizer, self.text_encoder = text_stack
        if self.text_encoder is not None:
            self.text_encoder.requires_grad_(False)
        self.sched = OneStepDDPM()
        self.timesteps = torch.tensor([999]).long()

    # ---- dtype handling: the reference calls model.half() (src/inference_paired.py:34-35) ----
    def half(self):
        self._dtype = torch.float16
        return self

    def bfloat16(self):
        self._dtype = torch.bfloat16
        return self

    def float(self):
        self._dtype = None
        return self

    def to(self, *args, **kwargs):
        for a in list(args) + list(kwargs.values()):
            if a in (torch.float16, torch.bfloat16):
                self._dtype = a
            elif a == torch.float32:
                self._dtype = None
        return self

    def cuda(self, device=None):
        return self

    @property
    def compute_dtype(self) -> torch.dtype:
        """fp16/bf16 as requested; an fp32 model (no .half()) computes in bf16 with fp32 accumulation (warned once: the
        reference computes in fp32 there, e.g. inference_paired.py without --use_fp16)."""
        if self._dtype is None and not self.__dict__.get("_warned_fp32"):
            self.__dict__["_warned_fp32"] = True
            warnings.warn("model was not cast to half/bfloat16: libi2it computes in bf16 with fp32 accumulation where the "
                          "reference would compute in fp32 (outputs are returned in the input dtype but carry bf16-level "
                          "rounding); call .half() or .to(torch.bfloat16) to make the choice explicit")
        return self._dtype or torch.bfloat16

    def _invalidate(self):
        self._engine_key = None
        self._final_key = None
        self.__dict__["_text_bound"] = None

    # ---- engine lifecycle -------------------------------------------------------------------------
    def _get_engine(self) -> i2it.Engine:
        key = (self.compute_dtype, _cur_dev())
        if self._engine is None or self._engine_key != key:
            if self._engine is not None:
                self._engine.close()
            te = self._text_encoder_spec()
            eng = i2it.Engine(self.compute_dtype, self.MODEL_KIND, cfg=self._cfg, keep_stages=self._keep_stages,
                              use_cuda_graph=self._use_graph, **({"text_heads": te["heads"], "text_act": te["act"]} if te else {}))
            eng.load_state_dict(self._sd)
            if te:      # the CLIP text tower runs on the engine too (SURVEY 8f #1): same tensors, transformers key names
                eng.load_state_dict({"text_encoder." + k: v for k, v in self.text_encoder.state_dict().items()})
            self._text_on_engine = bool(te)
            for name, s in self._adapter_scales.items():
                eng.set_adapter_scale(name, s)
            self._engine, self._engine_key, self._final_key = eng, key, None
        return self._engine

    def _finalize(self, lw_unet: float, lw_vae: float, gamma: float, twin_r: float):
        eng = self._get_engine()
        key = (float(lw_unet), float(lw_vae), float(gamma), float(twin_r))
        if self._final_key != key:
            eng.finalize(*key)
            self._final_key = key
            self.__dict__["_text_bound"] = None
        return eng

    # ---- text ----------------------------------------------------------------------------------------
    def _text_encoder_spec(self):
        """{"heads", "act", "hidden"} if the text encoder is a CLIP text tower libi2it can run (64-wide heads, gelu / quick_gelu,
        width <= 1280), else None (the stock transformers module is called instead)."""
        enc = self.text_encoder
        c = getattr(enc, "config", None)
        if enc is None or c is None or os.environ.get("I2IT_TORCH_TEXT"):
            return None
        try:
            hidden, heads, act = int(c.hidden_size), int(c.num_attention_heads), str(c.hidden_act)
        except Exception:
            return None
        if heads * 64 != hidden or hidden > 1280 or act not in ("gelu", "quick_gelu") or int(c.max_position_embeddings) != 77:
            return None
        return {"heads": heads, "act": act, "hidden": hidden}

    def _encode_text(self, prompt=None, tokens=None, device=None) -> torch.Tensor:
        """caption_enc = text_encoder(tokens)[0]; cached per distinct prompt / token tensor."""
        if prompt is not None:
            key = ("p", prompt if isinstance(prompt, str) else tuple(prompt), self.compute_dtype)
        else:
            key = ("t", tuple(tokens.flatten().tolist()), tuple(tokens.shape), self.compute_dtype)
        hit = self._text_cache.get(key)
        if hit is not None:
            return hit
        if prompt is not None:
            tokens = self.tokenizer(prompt, max_length=self.tokenizer.model_max_length, padding="max_length",
                                    truncation=True, return_tensors="pt").input_ids
        device = device or DEVICE
        eng = self._get_engine() if (device == "cuda" and self._text_encoder_spec()) else None
        if eng is not None and getattr(self, "_text_on_engine", False):
            # text_encoder(tokens)[0] on the engine: same tensors, hand-written kernels (no torch modules on this path)
            if self._final_key is None:      # the tower has no LoRA: any fold state will do, but the engine wants one
                self._finalize(1.0, 1.0, 1.0, -1.0)
            emb = eng.encode_text(tokens, self._text_encoder_spec()["hidden"])
        else:
            enc = self.text_encoder.to(device)
            with torch.no_grad():
                emb = enc(tokens.to(device))[0]
            emb = emb.to(self.compute_dtype).contiguous()
        if len(self._text_cache) > 64:
            self._text_cache.clear()
        self._text_cache[key] = emb
        return emb

    def _bind_text(self, eng, text):
        """Project the prompt's cross-attention K / V^T once per (prompt, folded weights): i2it_set_text.  `text` tensors come
        from the per-prompt cache (_encode_text), so identity + version is a sufficient change detector."""
        key = (id(eng), self._final_key, id(text), text._version, tuple(text.shape))
        if self.__dict__.get("_text_bound") != key:
            eng.set_text(text)
            self.__dict__["_text_bound"] = key
            self.__dict__["_text_ref"] = text      # keep it alive: id() must not be recycled while the key is cached

    def _staged_forward(self, eng, x, text, eps, noise=None, r=1.0, direction=i2it.A2B, u8_mode=None):
        """Run the engine through persistent device staging buffers (per shape/dtype): the captured CUDA graph bakes the IO
        pointers in, so stable addresses mean every call replays the same graph.  Costs two small device-to-device copies;
        the result is returned in a fresh tensor (never aliased across calls).  The text embedding is not an input of the
        graph: its projections are cached on the engine (_bind_text)."""
        self._bind_text(eng, text)
        key = (tuple(x.shape), x.dtype, eps.dtype, noise is not None, _cur_dev())
        st = self.__dict__.setdefault("_stage", {}).get(key)
        if st is None:
            st = {"x": torch.empty_like(x), "eps": torch.empty_like(eps), "out": torch.empty_like(x),
                  "noise": torch.empty_like(eps) if noise is not None else None}
            if len(self._stage) > 8:
                self._stage.clear()
            self._stage[key] = st
        st["x"].copy_(x, non_blocking=True)
        st["eps"].copy_(eps, non_blocking=True)
        if noise is not None:
            st["noise"].copy_(noise, non_blocking=True)
        if u8_mode is None:
            eng.forward(st["x"], None, st["eps"], noise_map=st["noise"], r=float(r), direction=direction, out=st["out"])
        else:
            eng.forward_u8(st["x"], u8_mode, None, st["eps"], noise_map=st["noise"], r=float(r), direction=direction, out=st["out"])
        return st["out"].clone()

    @staticmethod
    def _prep(t: Optional[torch.Tensor], dtype) -> Optional[torch.Tensor]:
        if t is None:
            return None
        return t.to(device=DEVICE, dtype=dtype).contiguous()


def load_sd_turbo_base(sd: Dict[str, torch.Tensor], which: List[str]) -> bool:
    """Overlay real SD-Turbo base weights from a local snapshot ($I2IT_SD_TURBO_DIR/{unet,vae}/*.safetensors) if present.
    Returns False (leaving the seeded random base) when unavailable — the offline case of every BASELINE config."""
    root = os.environ.get(SD_TURBO_DIR_ENV)
    if not root:
        return False
    try:
        from safetensors.torch import load_file
    except Exception:
        return False
    ok = True
    old_attn = {"query": "to_q", "key": "to_k", "value": "to_v", "proj_attn": "to_out.0"}
    for model in which:
        sub = "unet" if model == "unet" else "vae"
        path = os.path.join(root, sub, "diffusion_pytorch_model.safetensors")
        if not os.path.exists(path):
            ok = False
            continue
        for k, v in load_file(path).items():
            parts = k.split(".")
            parts = [old_attn.get(p, p) if "attentions" in k else p for p in parts]   # pre-0.14 VAE attention key names
            sd[f"{model}." + ".".join(parts)] = v.float()
    return ok
