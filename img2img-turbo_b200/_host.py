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
# resize geometry of the CLIs' host pre-processing (src/my_utils/training_utils.py build_transform)
# ------------------------------------------------------------------------------------------------
def image_prep_geometry(image_prep: str, H: int, W: int):
    """(resize, crop) of forward_u8 that equals build_transform(image_prep) on an H x W PIL image: resize (H, W) of the
    LANCZOS Resize, crop (top, left, height, width) of the CenterCrop or None.  Sizes follow torchvision: Resize(512) gives
    the short side 512 and the long side int(512 * long / short); CenterCrop puts the window at int(round((h - 512) / 2)).
    Raises ValueError for the random-crop training transforms and unknown names."""
    if image_prep in ("resize_512x512", "resize_512"):
        return (512, 512), None
    if image_prep in ("resize_256x256", "resize_256"):
        return (256, 256), None
    if image_prep == "no_resize":
        return (H, W), None
    if image_prep == "resized_crop_512":
        if W <= H:
            rs = (int(512 * H / W), 512)
        else:
            rs = (512, int(512 * W / H))
        return rs, (int(round((rs[0] - 512) / 2.0)), int(round((rs[1] - 512) / 2.0)), 512, 512)
    raise ValueError(f"image_prep {image_prep!r} has no deterministic resize geometry (random crops are training-only)")


def ragged_geometries(sizes, image_prep: Optional[str] = None, resize=None):
    """(H, W, geometries) of a ragged uint8 batch of images of `sizes` [(H_i, W_i), ...]: image i goes through
    image_prep_geometry(image_prep, H_i, W_i), or a LANCZOS resize to `resize` (H, W) when image_prep is None, and its output
    comes back at (H_i, W_i).  H x W is the network size they share; raises ValueError when they would not share one."""
    if len(sizes) == 0:
        raise ValueError("a ragged batch needs at least one image")
    geoms, net = [], set()
    for h, w in sizes:
        h, w = int(h), int(w)
        rs, crop = image_prep_geometry(image_prep, h, w) if image_prep is not None else (tuple(int(v) for v in resize), None)
        net.add(tuple(crop[2:]) if crop is not None else tuple(rs))
        geoms.append({"resize": tuple(rs), "crop": crop, "out_size": (h, w)})
    if len(net) != 1:
        raise ValueError(f"the images of a ragged batch must share one network size; {image_prep or resize} gives {sorted(net)}")
    H, W = net.pop()
    return H, W, geoms


def paired_geometry(H: int, W: int):
    """resize (H, W) of src/inference_paired.py:38-41: LANCZOS to the multiple of 8 below each side."""
    return H - H % 8, W - W % 8


# ------------------------------------------------------------------------------------------------
# light-weight stand-ins for the diffusers module objects the reference exposes as .unet / .vae
# ------------------------------------------------------------------------------------------------
def weight_record(sd: Dict[str, torch.Tensor]) -> Dict[str, tuple]:
    """What weight_update compares against: key -> (the tensor registered on the engine, its version counter then)."""
    return {k: (v, v._version) for k, v in sd.items()}


def _shares_storage(a: torch.Tensor, b: torch.Tensor) -> bool:
    return a.untyped_storage().data_ptr() == b.untyped_storage().data_ptr()


def weight_update(loaded: Optional[Dict[str, tuple]], sd: Dict[str, torch.Tensor]) -> Optional[List[str]]:
    """How a live engine that holds `loaded` (weight_record of the tensors registered on it) takes the state dict `sd`: the
    keys whose tensors changed, to register again in place before a refold, or None when it needs a new engine (no engine
    yet, a key added or removed, a shape changed).  A TwinConv added or removed changes the keys.

    A recorded tensor may alias what the caller holds (state_dict() hands out the stored tensors, and an fp32 CPU tensor is
    stored as is), so its values are not a record of what was registered: a tensor modified in place since (its version
    moved) counts as changed, and so does any other tensor on its storage.  Only a different tensor on other storage is
    compared by value with an unmodified record."""
    if loaded is None or loaded.keys() != sd.keys():
        return None
    changed = []
    for k, v in sd.items():
        old, version = loaded[k]
        if tuple(v.shape) != tuple(old.shape):
            return None
        if old._version != version:
            changed.append(k)
        elif v is old:
            continue
        elif _shares_storage(v, old) or v.dtype != old.dtype or not torch.equal(v, old):
            changed.append(k)
    return changed


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
        self._owner._reload()

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
    # forward plans an engine keeps (least recently run evicted first): a demo or a folder loop over many image sizes stays
    # bounded; an evicted size is rebuilt with identical outputs when it returns
    MAX_PLANS = 16

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

    def _reload(self):
        """Take the state dict's new tensors.  A live engine that holds the same keys and shapes registers only the tensors
        that changed and refolds in place, keeping its plans and CUDA graphs; anything else builds a new engine."""
        live = self._engine is not None and self._engine_key is not None
        changed = weight_update(self.__dict__.get("_loaded"), self._sd) if live else None
        if changed is None:
            self._invalidate()
            return
        if not changed:
            return
        try:
            self._engine.load_state_dict({k: self._sd[k] for k in changed})
            self._loaded = weight_record(self._sd)
            if self._final_key is not None:
                self._engine.refold(*self._final_key)
                self.__dict__["_text_bound"] = None
        except Exception:
            self._invalidate()
            raise

    # ---- engine lifecycle -------------------------------------------------------------------------
    def _get_engine(self) -> i2it.Engine:
        key = (self.compute_dtype, _cur_dev())
        if self._engine is None or self._engine_key != key:
            if self._engine is not None:
                self._engine.close()
            te = self._text_encoder_spec()
            eng = i2it.Engine(self.compute_dtype, self.MODEL_KIND, cfg=self._cfg, keep_stages=self._keep_stages,
                              use_cuda_graph=self._use_graph, max_plans=self.MAX_PLANS,
                              **({"text_heads": te["heads"], "text_act": te["act"]} if te else {}))
            eng.load_state_dict(self._sd)
            self._loaded = weight_record(self._sd)
            if te:      # the CLIP text tower runs on the engine too (SURVEY 8f #1): same tensors, transformers key names
                eng.load_state_dict({"text_encoder." + k: v for k, v in self.text_encoder.state_dict().items()})
            self._text_on_engine = bool(te)
            for name, s in self._adapter_scales.items():
                eng.set_adapter_scale(name, s)
            self._engine, self._engine_key, self._final_key = eng, key, None
        return self._engine

    def release_plans(self):
        """Give back the device memory of every forward plan (the shared workspace included).  Weights, prompt caches and the
        staging buffers stay; the next forward of each shape rebuilds its plan."""
        if self._engine is not None:
            self._engine.release_plans()

    def _finalize(self, lw_unet: float, lw_vae: float, gamma: float, twin_r: float):
        eng = self._get_engine()
        key = (float(lw_unet), float(lw_vae), float(gamma), float(twin_r))
        if self._final_key != key:
            prev = self._final_key
            if prev is not None and (prev[3] < 0) == (key[3] < 0):
                eng.refold(*key)          # the same weights in the same buffers: plans and CUDA graphs stay
            else:
                eng.finalize(*key)
            self._final_key = key
            self.__dict__["_text_bound"] = None
        return eng

    # ---- text ----------------------------------------------------------------------------------------
    def _text_encoder_spec(self):
        """{"heads", "act", "hidden"} if the text encoder is a CLIP text tower libi2it can run (64-wide heads, gelu / quick_gelu,
        width <= 1280, 77 positions, LayerNorm eps 1e-5 as the engine's layernorm launches use), else None (the stock
        transformers module is called instead)."""
        enc = self.text_encoder
        c = getattr(enc, "config", None)
        if enc is None or c is None or os.environ.get("I2IT_TORCH_TEXT"):
            return None
        try:
            hidden, heads, act = int(c.hidden_size), int(c.num_attention_heads), str(c.hidden_act)
            ln_eps = float(c.layer_norm_eps)
        except Exception:
            return None
        if heads * 64 != hidden or hidden > 1280 or act not in ("gelu", "quick_gelu") or int(c.max_position_embeddings) != 77:
            return None
        if ln_eps != 1e-5:
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

    @staticmethod
    def _u8_geometry(shape, resize, crop, out_size):
        """(H, W, geometry) of a uint8 forward on [B, H, W, 3] images: the network size and the forward_u8 keywords (None
        without a resize, crop or output size)."""
        if resize is None and crop is None and out_size is None:
            return shape[1], shape[2], None
        rs, cr, out = i2it.resize_geometry((shape[1], shape[2]), resize, crop, out_size)
        return cr[2], cr[3], {"resize": rs, "crop": cr, "out_size": out}

    def _staged_forward(self, eng, x, text, eps, noise=None, r=1.0, direction=i2it.A2B, u8_mode=None, geometry=None,
                        variations=False, ragged=None):
        """Run the engine through persistent device staging buffers (per shape/dtype): the captured CUDA graph bakes the IO
        pointers in, so stable addresses mean every call replays the same graph.  Costs two small device-to-device copies;
        the result is returned in a fresh tensor (never aliased across calls).  The text embedding is not an input of the
        graph: its projections are cached on the engine (_bind_text).  `geometry`: forward_u8 resize keywords.
        variations: x is one image and the eps.shape[0] outputs are its variations (forward_variations).
        ragged: x is a list of uint8 images of their own sizes and `ragged` their forward_u8 geometries (forward_u8_ragged)."""
        if ragged is not None:
            return self._ragged_forward(eng, x, text, eps, noise, r, direction, u8_mode, ragged)
        self._bind_text(eng, text)
        gkey = tuple(sorted(geometry.items())) if geometry else None
        n = eps.shape[0] if variations else x.shape[0]
        key = (tuple(x.shape), x.dtype, eps.dtype, noise is not None, _cur_dev(), gkey) + ((n,) if variations else ())
        st = self.__dict__.setdefault("_stage", {}).get(key)
        if st is None:
            out = x.new_empty((n,) + tuple(x.shape[1:]) if geometry is None else (n,) + geometry["out_size"] + (3,))
            st = {"x": torch.empty_like(x), "eps": torch.empty_like(eps), "out": out,
                  "noise": torch.empty_like(eps) if noise is not None else None}
            if len(self._stage) > 8:
                self._stage.clear()
            self._stage[key] = st
        st["x"].copy_(x, non_blocking=True)
        st["eps"].copy_(eps, non_blocking=True)
        if noise is not None:
            st["noise"].copy_(noise, non_blocking=True)
        if isinstance(direction, list):          # one direction per image: CycleGAN's mixed-direction forward
            eng.forward_mixed(st["x"], None, st["eps"], direction, out=st["out"])
        elif u8_mode is None:
            fwd = eng.forward_variations if variations else eng.forward
            fwd(st["x"], None, st["eps"], noise_map=st["noise"], r=float(r), direction=direction, out=st["out"])
        else:
            fwd = eng.forward_u8_variations if variations else eng.forward_u8
            fwd(st["x"], u8_mode, None, st["eps"], noise_map=st["noise"], r=float(r), direction=direction, out=st["out"],
                **(geometry or {}))
        return st["out"].clone()

    def _ragged_forward(self, eng, images, text, eps, noise, r, direction, u8_mode, geometries):
        """forward_u8_ragged on a list of images.  Only eps and the noise map go through persistent staging: the graph bakes
        their pointers in.  The images and the fresh outputs sit in the call's descriptors, so they need no copy."""
        self._bind_text(eng, text)
        key = ("ragged", tuple(eps.shape), eps.dtype, noise is not None, _cur_dev())
        st = self.__dict__.setdefault("_stage", {}).get(key)
        if st is None:
            st = {"eps": torch.empty_like(eps), "noise": torch.empty_like(eps) if noise is not None else None}
            if len(self._stage) > 8:
                self._stage.clear()
            self._stage[key] = st
        st["eps"].copy_(eps, non_blocking=True)
        if noise is not None:
            st["noise"].copy_(noise, non_blocking=True)
        if isinstance(direction, list):
            return eng.forward_u8_ragged_mixed(images, u8_mode, None, st["eps"], direction, geometries=geometries)
        return eng.forward_u8_ragged(images, u8_mode, None, st["eps"], noise_map=st["noise"], r=float(r), direction=direction,
                                     geometries=geometries)

    @staticmethod
    def _variation_count(n, text, noise_map, eps) -> int:
        """n of a variations call: from n=, eps, a noise_map or prompt batch other than 1 (a batch of 1 is shared by all
        variations); every one of them that is given must agree.  1 when none is."""
        got = {"n": n, "eps": None if eps is None else eps.shape[0],
               "noise_map": noise_map.shape[0] if noise_map is not None and noise_map.shape[0] != 1 else None,
               "prompt": text.shape[0] if text.shape[0] != 1 else None}
        got = {k: int(v) for k, v in got.items() if v is not None}
        if len(set(got.values())) > 1:
            raise ValueError(f"the number of variations differs between arguments: {got}")
        n = next(iter(got.values()), 1)
        if n < 1:
            raise ValueError(f"the number of variations must be >= 1, got {n}")
        return n

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
