"""ctypes binding of libi2it.so (the C ABI declared in include/i2it.h).

PyTorch is plumbing here: it owns device memory and streams; every FLOP of the image path runs inside
libi2it's sm_90a kernels.  There is NO fallback: if the library is missing or the device is not an
H100, construction raises.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, Optional, Sequence

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libi2it.so")

F16, BF16, F32 = 0, 1, 2
PIX2PIX, CYCLEGAN = 0, 1
A2B, B2A = 0, 1
ACT_NONE, ACT_CLAMP1, ACT_GEGLU, ACT_GELU, ACT_QUICKGELU = 0, 1, 2, 3, 4   # epilogue activations (tapgemm TgAct)
IN_UNIT, IN_NORMALIZE, IN_SKETCH = 0, 1, 2      # uint8 input transforms (ForwardDesc.in_mode)

_TORCH2DT = {torch.float16: F16, torch.bfloat16: BF16, torch.float32: F32}
_DT2TORCH = {F16: torch.float16, BF16: torch.bfloat16}

# every symbol include/i2it.h declares (tests check the library exports all of them)
SYMBOLS = [
    "i2it_default_config", "i2it_create", "i2it_destroy", "i2it_last_error", "i2it_set_weight",
    "i2it_set_adapter_scale", "i2it_finalize_weights", "i2it_workspace_bytes", "i2it_forward",
    "i2it_set_text", "i2it_encode_text", "i2it_prep_launch_count", "i2it_debug_fast_div", "i2it_launch_count", "i2it_profile", "i2it_read_stage", "i2it_op_conv2d", "i2it_op_group_norm", "i2it_op_layer_norm",
    "i2it_op_attention", "i2it_op_upsample2x", "i2it_op_conv2d_ex", "i2it_op_launches", "i2it_op_vt_proj",
    "i2it_op_upsample_to", "i2it_stage_names", "i2it_prepared_keys", "i2it_read_prepared", "i2it_text_stage_names",
    "i2it_op_resize_u8", "i2it_debug_resample_coeffs",
    "i2it_set_max_plans", "i2it_release_plans", "i2it_memory_stats_get", "i2it_debug_poison_workspace",
    "i2it_debug_tapgemm_override", "i2it_op_resize_u8_ragged", "i2it_debug_ragged_tables", "i2it_debug_graph_captures",
    "i2it_refold_weights", "i2it_debug_refold_info",
    "i2it_mixed_size_check", "i2it_op_conv2d_sel",
]
TEXT_TOKEN_EMB = "text_encoder.text_model.embeddings.token_embedding.weight"
TEXT_POS_EMB = "text_encoder.text_model.embeddings.position_embedding.weight"


def check_tokens(tokens: torch.Tensor, vocab: int, ntok: int):
    """Raise ValueError unless `tokens` is [B, ntok] with every id in [0, vocab).  The text tower reads B * ntok ids and
    writes B * ntok rows whatever the tensor's shape, and its embedding kernel clamps ids: both checks must come first."""
    if tokens.dim() != 2 or tokens.shape[0] < 1 or tokens.shape[1] != ntok:
        raise ValueError(f"text tokens must be [B, {ntok}] (the position table's length), got {list(tokens.shape)}")
    if tokens.dtype.is_floating_point or tokens.dtype.is_complex or tokens.dtype == torch.bool:
        raise ValueError(f"text tokens must be integer ids, got {tokens.dtype}")
    lo, hi = int(tokens.min()), int(tokens.max())
    if lo < 0 or hi >= vocab:
        raise ValueError(f"token ids must lie in [0, {vocab}), got ids from {lo} to {hi}")


class ConvDesc(C.Structure):
    """i2it_conv_desc (include/i2it.h)."""
    _fields_ = [
        ("x", C.c_void_p), ("N", C.c_int), ("H", C.c_int), ("W", C.c_int), ("Cin", C.c_int), ("ldx", C.c_int),
        ("w", C.c_void_p), ("bias", C.c_void_p), ("Cout", C.c_int), ("ksize", C.c_int), ("stride", C.c_int),
        ("asym_pad", C.c_int), ("residual", C.c_void_p), ("ldr", C.c_int), ("act", C.c_int),
        ("out", C.c_void_p), ("ldo", C.c_int), ("out_fp32", C.c_int),
        ("x2", C.c_void_p), ("C2", C.c_int), ("ld2", C.c_int), ("w2", C.c_void_p),
        ("up2x", C.c_int), ("tokens", C.c_int),
        ("gn_y", C.c_void_p), ("ldg", C.c_int), ("gn_silu", C.c_int), ("gn_eps", C.c_float), ("gn_gamma", C.c_void_p),
        ("gn_beta", C.c_void_p),
    ]


class ResizeDesc(C.Structure):
    """i2it_resize_desc (include/i2it.h); sizes are rows x columns."""
    _fields_ = [(n, C.c_int) for n in ("in_H", "in_W", "resize_H", "resize_W", "crop_y", "crop_x", "out_H", "out_W")]


class ForwardDesc(C.Structure):
    """i2it_forward_desc (include/i2it.h): one image forward; unset fields are zero (unused)."""
    _fields_ = [
        ("batch", C.c_int), ("H", C.c_int), ("W", C.c_int), ("direction", C.c_int), ("directions", C.POINTER(C.c_int)),
        ("shared_input", C.c_int), ("x", C.c_void_p), ("x_u8", C.c_void_p), ("x_u8_list", C.POINTER(C.c_void_p)),
        ("in_mode", C.c_int), ("geometry", C.POINTER(ResizeDesc)), ("max_side", C.c_int),
        ("text_emb", C.c_void_p), ("text_batch", C.c_int), ("eps", C.c_void_p), ("noise_map", C.c_void_p), ("r", C.c_float),
        ("out", C.c_void_p), ("out_u8", C.c_void_p), ("out_u8_list", C.POINTER(C.c_void_p)), ("out_latent", C.c_void_p),
    ]


def resize_geometry(in_hw, resize=None, crop=None, out_size=None):
    """Complete the LANCZOS geometry of a uint8 forward on an image of in_hw = (H, W): resize (H, W) defaults to the input
    size, crop (top, left, height, width) to the whole resized image, out_size (H, W) to the crop's size.  Returns
    ((resize_H, resize_W), (top, left, H, W), (out_H, out_W)); the network runs on the H x W window."""
    rs = tuple(int(v) for v in (resize if resize is not None else in_hw))
    cr = tuple(int(v) for v in (crop if crop is not None else (0, 0) + rs))
    out = tuple(int(v) for v in (out_size if out_size is not None else cr[2:]))
    if len(rs) != 2 or len(cr) != 4 or len(out) != 2:
        raise ValueError("resize and out_size are (H, W), crop is (top, left, height, width)")
    return rs, cr, out


def ragged_max_side(sizes) -> int:
    """Default capacity of a ragged forward: the largest of `sizes` rounded up to a multiple of 1024, at least 4096, so an
    ordinary stream of uploads runs on one plan per batch size."""
    return max(4096, -(-max(int(v) for v in sizes) // 1024) * 1024)


def _ragged_descs(geometries, in_hws):
    """(H, W, ResizeDesc array) of a ragged call: geometries[i] holds image i's forward_u8 keywords (resize, crop, out_size;
    each may be absent or None); every crop must have the same size, the network's."""
    if len(geometries) != len(in_hws):
        raise ValueError(f"{len(in_hws)} images but {len(geometries)} geometries")
    descs, net = (ResizeDesc * len(in_hws))(), set()
    for i, (hw, g) in enumerate(zip(in_hws, geometries)):
        rs, cr, osz = resize_geometry(hw, g.get("resize"), g.get("crop"), g.get("out_size"))
        net.add(cr[2:])
        descs[i] = ResizeDesc(hw[0], hw[1], rs[0], rs[1], cr[0], cr[1], osz[0], osz[1])
    if len(net) != 1:
        raise ValueError(f"a ragged batch runs one network size; its geometries give {sorted(net)}")
    H, W = net.pop()
    return H, W, descs


def ragged_table_ints(geometries, in_hws, max_side: int):
    """(used, bound): coefficient-table ints a ragged forward on these images uploads, and what its plan reserves (host only)."""
    H, W, descs = _ragged_descs(geometries, in_hws)
    used, bound = C.c_longlong(0), C.c_longlong(0)
    if load_library().i2it_debug_ragged_tables(descs, len(in_hws), H, W, int(max_side), C.byref(used), C.byref(bound)) != 0:
        raise ValueError("the ragged forward would reject these geometries")
    return used.value, bound.value


def resample_coeffs(in_size: int, out_size: int):
    """Tables of one LANCZOS pass exactly as the resample kernels get them (host only, no GPU):
    (ksize, bounds [out][2] = (first input index, taps), 22-bit coefficients [out][ksize])."""
    lib = load_library()
    ksize = lib.i2it_debug_resample_coeffs(in_size, out_size, None, None, 0)
    if ksize < 0:
        raise ValueError(f"bad resample sizes {in_size} -> {out_size}")
    bounds = (C.c_int * (2 * out_size))()
    coeffs = (C.c_int * (out_size * ksize))()
    if lib.i2it_debug_resample_coeffs(in_size, out_size, bounds, coeffs, out_size * ksize) != ksize:
        raise RuntimeError("i2it_debug_resample_coeffs failed")
    return ksize, [tuple(bounds[2 * i: 2 * i + 2]) for i in range(out_size)], \
        [list(coeffs[i * ksize: (i + 1) * ksize]) for i in range(out_size)]


class MemoryStats(C.Structure):
    """i2it_memory_stats (include/i2it.h)."""
    _fields_ = [
        ("arena_bytes", C.c_size_t), ("plan_bytes", C.c_size_t), ("plans", C.c_int),
        ("plan_builds", C.c_int), ("plan_evictions", C.c_int),
    ]


class Config(C.Structure):
    _fields_ = [
        ("dtype", C.c_int), ("model_kind", C.c_int), ("device", C.c_int),
        ("unet_channels", C.c_int * 4), ("unet_heads", C.c_int * 4),
        ("cross_dim", C.c_int), ("temb_dim", C.c_int), ("vae_channels", C.c_int * 4),
        ("scaling_factor", C.c_float), ("keep_stages", C.c_int), ("use_cuda_graph", C.c_int),
        ("text_heads", C.c_int), ("text_act", C.c_int),
    ]


_lib = None


def load_library(path: Optional[str] = None):
    """dlopen libi2it.so and declare prototypes.  Fails loudly when the extension is not built."""
    global _lib
    if _lib is not None:
        return _lib
    path = path or os.environ.get("I2IT_LIB", LIB_PATH)
    if not os.path.exists(path):
        raise RuntimeError(
            f"libi2it.so not found at {path}: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C img2img-turbo_b200/csrc`).  There is no CPU/PyTorch fallback for the image path.")
    lib = C.CDLL(path)
    vp, ci, cf = C.c_void_p, C.c_int, C.c_float
    lib.i2it_default_config.argtypes = [C.POINTER(Config)]
    lib.i2it_create.argtypes = [C.POINTER(Config), C.POINTER(vp)]
    lib.i2it_destroy.argtypes = [vp]
    lib.i2it_destroy.restype = None
    lib.i2it_last_error.argtypes = [vp]
    lib.i2it_last_error.restype = C.c_char_p
    lib.i2it_set_weight.argtypes = [vp, C.c_char_p, vp, C.POINTER(C.c_int64), ci, ci, ci]
    lib.i2it_set_adapter_scale.argtypes = [vp, C.c_char_p, cf]
    lib.i2it_finalize_weights.argtypes = [vp, cf, cf, cf, cf]
    lib.i2it_workspace_bytes.argtypes = [vp, ci, ci, ci, C.POINTER(C.c_size_t)]
    lib.i2it_forward.argtypes = [vp, C.POINTER(ForwardDesc), vp]
    lib.i2it_set_text.argtypes = [vp, vp, ci, vp]
    lib.i2it_encode_text.argtypes = [vp, vp, ci, vp, vp]
    lib.i2it_prep_launch_count.argtypes = [vp, C.POINTER(ci)]
    lib.i2it_debug_fast_div.argtypes = [C.c_longlong, ci, ci]
    lib.i2it_debug_fast_div.restype = C.c_longlong
    lib.i2it_launch_count.argtypes = [vp, ci, ci, ci, ci, C.POINTER(ci)]
    lib.i2it_profile.argtypes = [vp, ci, C.c_char_p, C.c_size_t, vp]
    lib.i2it_read_stage.argtypes = [vp, C.c_char_p, vp, C.c_size_t, C.POINTER(ci)]
    lib.i2it_op_conv2d.argtypes = [vp, vp, ci, ci, ci, ci, ci, vp, vp, ci, ci, ci, ci, vp, ci, ci, vp, ci, ci, vp]
    lib.i2it_op_group_norm.argtypes = [vp, vp, ci, ci, ci, ci, vp, vp, cf, ci, vp, ci, vp]
    lib.i2it_op_layer_norm.argtypes = [vp, vp, ci, ci, ci, vp, vp, cf, vp, ci, vp]
    lib.i2it_op_conv2d_ex.argtypes = [vp, C.POINTER(ConvDesc), vp]
    lib.i2it_op_launches.argtypes = [vp, C.c_char_p, C.c_size_t]
    lib.i2it_op_attention.argtypes = [vp, vp, ci, vp, ci, vp, ci, ci, ci, ci, ci, ci, ci, ci, vp, ci, vp]
    lib.i2it_op_vt_proj.argtypes = [vp, vp, ci, ci, ci, ci, vp, vp, ci, vp, vp]
    lib.i2it_op_upsample2x.argtypes = [vp, vp, ci, ci, ci, ci, vp, vp]
    lib.i2it_op_upsample_to.argtypes = [vp, vp, ci, ci, ci, ci, ci, ci, vp, vp]
    lib.i2it_stage_names.argtypes = [vp, C.c_char_p, C.c_size_t]
    lib.i2it_text_stage_names.argtypes = [vp, C.c_char_p, C.c_size_t]
    lib.i2it_prepared_keys.argtypes = [vp, C.c_char_p, C.c_size_t]
    lib.i2it_read_prepared.argtypes = [vp, C.c_char_p, vp, C.c_size_t, vp, C.c_size_t, C.POINTER(ci)]
    lib.i2it_op_resize_u8.argtypes = [vp, vp, ci, ci, ci, vp, ci, ci, vp]
    lib.i2it_debug_resample_coeffs.argtypes = [ci, ci, C.POINTER(ci), C.POINTER(ci), ci]
    lib.i2it_set_max_plans.argtypes = [vp, ci]
    lib.i2it_release_plans.argtypes = [vp]
    lib.i2it_memory_stats_get.argtypes = [vp, C.POINTER(MemoryStats)]
    lib.i2it_debug_poison_workspace.argtypes = [vp, ci]
    lib.i2it_debug_tapgemm_override.argtypes = [vp, ci, ci, ci]
    lib.i2it_op_resize_u8_ragged.argtypes = [vp, C.POINTER(vp), C.POINTER(ci), C.POINTER(vp), C.POINTER(ci), ci, ci, vp]
    lib.i2it_debug_ragged_tables.argtypes = [C.POINTER(ResizeDesc), ci, ci, ci, ci, C.POINTER(C.c_longlong),
                                             C.POINTER(C.c_longlong)]
    lib.i2it_debug_graph_captures.argtypes = [vp, C.POINTER(ci)]
    lib.i2it_refold_weights.argtypes = [vp, cf, cf, cf, cf]
    lib.i2it_debug_refold_info.argtypes = [vp, C.c_char_p, C.c_size_t]
    lib.i2it_mixed_size_check.argtypes = [ci, ci, C.c_char_p, C.c_size_t]
    lib.i2it_op_conv2d_sel.argtypes = [vp, C.POINTER(ConvDesc), vp, vp, vp, C.POINTER(ci), vp]
    for name in SYMBOLS:
        fn = getattr(lib, name)
        if name not in ("i2it_destroy", "i2it_last_error"):
            fn.restype = ci
    _lib = lib
    return lib


def _ptr(t: Optional[torch.Tensor]):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _ptrs(ts):
    return (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def _check_u8_images(images, what):
    for x in images:
        if not (x.dim() == 3 and x.shape[2] == 3 and x.dtype == torch.uint8 and x.is_cuda and x.is_contiguous()):
            raise ValueError(f"{what}: every image must be a contiguous uint8 CUDA tensor [H, W, 3], got "
                             f"{x.dtype} {list(x.shape)}{'' if x.is_cuda else ' on the CPU'}")


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def mixed_size_check(H: int, W: int) -> str:
    """Why a mixed-direction forward refuses the network size H x W, or "" when it accepts it (i2it_mixed_size_check: every
    VAE tile must hold rows of one image).  Host only."""
    buf = C.create_string_buffer(1024)
    load_library().i2it_mixed_size_check(int(H), int(W), buf, 1024)
    return buf.value.decode()


def directions_array(directions, n: int):
    """The C array of a mixed-direction call: n values, each A2B (0) or B2A (1).  Raises ValueError otherwise."""
    dirs = list(directions)
    if len(dirs) != n:
        raise ValueError(f"{n} images but {len(dirs)} directions")
    for i, d in enumerate(dirs):
        if isinstance(d, bool) or not isinstance(d, int) or d not in (A2B, B2A):
            raise ValueError(f"direction {d!r} of image {i} is neither A2B (0) nor B2A (1)")
    return (C.c_int * n)(*dirs)


class Engine:
    """One engine per (device, stream).  Thin, typed wrapper over the C handle."""

    def __init__(self, dtype: torch.dtype = torch.bfloat16, model_kind: int = PIX2PIX, cfg: Optional[dict] = None,
                 device: Optional[int] = None, keep_stages: int = 0, use_cuda_graph: bool = True,
                 text_heads: int = 0, text_act: str = "gelu", max_plans: int = 0):
        if not torch.cuda.is_available():
            raise RuntimeError("libi2it needs a CUDA device (H100 / sm_90a); no CPU fallback exists")
        self.lib = load_library()
        self.dtype = dtype
        c = Config()
        self.lib.i2it_default_config(C.byref(c))
        c.dtype = _TORCH2DT[dtype]
        c.model_kind = model_kind
        c.device = torch.cuda.current_device() if device is None else device
        c.keep_stages = int(keep_stages)                     # 1: named checkpoints, 2: every layer output
        c.use_cuda_graph = int(use_cuda_graph)
        c.text_heads = int(text_heads)                       # 0: hidden / 64
        c.text_act = 1 if text_act == "quick_gelu" else 0
        if cfg is not None:
            for i in range(4):
                c.unet_channels[i] = cfg["unet_channels"][i]
                c.unet_heads[i] = cfg["unet_heads"][i]
                c.vae_channels[i] = cfg["vae_channels"][i]
            c.cross_dim = cfg["cross_dim"]
            c.temb_dim = cfg["temb_dim"]
            c.scaling_factor = cfg["scaling_factor"]
        self.cross_dim = c.cross_dim
        self.device = c.device
        self._h = C.c_void_p(0)
        rc = self.lib.i2it_create(C.byref(c), C.byref(self._h))
        if rc != 0:
            raise RuntimeError("i2it_create failed: " + self.lib.i2it_last_error(C.c_void_p(0)).decode())
        # i2it_create reads I2IT_NO_FLASH: without it d = 64 attention runs flash_attn, and d = 512 flash_attn512 above 8192 keys
        self.flash = os.environ.get("I2IT_NO_FLASH") is None
        if max_plans:
            self.set_max_plans(max_plans)

    def _check(self, rc: int, what: str):
        if rc != 0:
            raise RuntimeError(f"{what} failed: " + self.lib.i2it_last_error(self._h).decode())

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self.lib.i2it_destroy(self._h)
            self._h = C.c_void_p(0)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- weights -------------------------------------------------------------------------------
    def load_state_dict(self, sd: Dict[str, torch.Tensor]):
        for k, v in sd.items():
            t = v.detach()
            if t.dtype not in _TORCH2DT:
                t = t.float()
            t = t.contiguous()
            shape = (C.c_int64 * t.dim())(*t.shape)
            self._check(self.lib.i2it_set_weight(self._h, k.encode(), _ptr(t), shape, t.dim(), _TORCH2DT[t.dtype],
                                                 int(t.is_cuda)), f"i2it_set_weight({k})")
            if k == TEXT_TOKEN_EMB:              # encode_text checks token ids and the output width against these
                self._text_vocab, self._text_hidden = int(t.shape[0]), int(t.shape[1])
            elif k == TEXT_POS_EMB:
                self._text_ntok = int(t.shape[0])

    def set_adapter_scale(self, adapter: str, alpha_over_r: float):
        self._check(self.lib.i2it_set_adapter_scale(self._h, adapter.encode(), alpha_over_r), "i2it_set_adapter_scale")

    def finalize(self, lora_weight_unet: float = 1.0, lora_weight_vae: float = 1.0, skip_gamma: float = 1.0,
                 twin_r: float = -1.0):
        self._text_batch = None          # cached text projections die with the folded weights
        self._check(self.lib.i2it_finalize_weights(self._h, lora_weight_unet, lora_weight_vae, skip_gamma, twin_r),
                    "i2it_finalize_weights")

    def refold(self, lora_weight_unet: float = 1.0, lora_weight_vae: float = 1.0, skip_gamma: float = 1.0,
               twin_r: float = -1.0):
        """Fold again in place (i2it_refold_weights): new scalars, or tensors re-registered with their shapes since the last
        fold.  Plans and their CUDA graphs stay; the set_text cache is dropped, as after finalize."""
        self._check(self.lib.i2it_refold_weights(self._h, lora_weight_unet, lora_weight_vae, skip_gamma, twin_r),
                    "i2it_refold_weights")
        self._text_batch = None          # a refused refold keeps the cache, as the engine does

    # ---- the hot path ----------------------------------------------------------------------------
    def set_text(self, text_emb: torch.Tensor):
        """Cache the cross-attention K / V^T of a prompt embedding [1|B,77,cross]; later forwards pass text_emb=None."""
        if not (text_emb.is_cuda and text_emb.is_contiguous() and text_emb.dtype == self.dtype):
            raise ValueError("libi2it operands must be contiguous CUDA tensors in the engine dtype")
        if text_emb.dim() != 3 or text_emb.shape[1:] != (77, self.cross_dim):
            raise ValueError(f"text_emb must be [1|B,77,{self.cross_dim}]")
        self._check(self.lib.i2it_set_text(self._h, _ptr(text_emb), text_emb.shape[0], _stream()), "i2it_set_text")
        self._text_batch = text_emb.shape[0]

    def encode_text(self, tokens: torch.Tensor, hidden: int) -> torch.Tensor:
        """CLIP text tower on the engine: tokens [B,77] (any integer dtype) -> last_hidden_state [B,77,hidden] in the engine dtype.
        Needs the `text_encoder.*` tensors in the loaded state dict.  Raises ValueError, before any launch, unless tokens is
        [B, position-table length] with ids in [0, vocab) and `hidden` is the tower's width."""
        vocab, ntok = getattr(self, "_text_vocab", None), getattr(self, "_text_ntok", None)
        if vocab is None or ntok is None:
            raise ValueError("encode_text needs the text_encoder.* tensors (load_state_dict) first")
        check_tokens(tokens, vocab, ntok)
        if hidden != self._text_hidden:
            raise ValueError(f"hidden must be the text tower's width {self._text_hidden}, got {hidden}")
        ids = tokens.to(device="cuda", dtype=torch.int32).contiguous()
        out = torch.empty(ids.shape[0], ids.shape[1], hidden, device="cuda", dtype=self.dtype)
        self._check(self.lib.i2it_encode_text(self._h, _ptr(ids), ids.shape[0], _ptr(out), _stream()), "i2it_encode_text")
        return out

    def _check_operands(self, B, H, W, text_emb, eps, others):
        for t in (text_emb, eps) + tuple(others):
            if t is not None:
                if not (t.is_cuda and t.is_contiguous() and t.dtype == self.dtype):
                    raise ValueError("libi2it operands must be contiguous CUDA tensors in the engine dtype")
        if text_emb is not None:
            if text_emb.shape[1:] != (77, self.cross_dim) or text_emb.shape[0] not in (1, B):
                raise ValueError(f"text_emb must be [1|B,77,{self.cross_dim}]")
            tb = text_emb.shape[0]
        else:
            tb = getattr(self, "_text_batch", None)
            if tb is None:
                raise ValueError("text_emb=None needs a previous set_text()")
        if eps.shape != (B, 4, H // 8, W // 8):
            raise ValueError("eps must be [B,4,H/8,W/8]")
        return tb

    def _forward(self, n, H, W, text_emb, tb, eps, out_latent, **fields):
        """One i2it_forward call on n images (or variations) of an H x W network; `fields` fill the rest of its ForwardDesc."""
        d = ForwardDesc(batch=n, H=H, W=W, text_emb=_ptr(text_emb), text_batch=tb, eps=_ptr(eps), out_latent=_ptr(out_latent),
                        **fields)
        self._check(self.lib.i2it_forward(self._h, C.byref(d), _stream()), "i2it_forward")

    def forward(self, x: torch.Tensor, text_emb: Optional[torch.Tensor], eps: torch.Tensor,
                noise_map: Optional[torch.Tensor] = None, r: float = 1.0, direction: int = A2B,
                out: Optional[torch.Tensor] = None, out_latent: Optional[torch.Tensor] = None) -> torch.Tensor:
        B, Cc, H, W = x.shape
        assert Cc == 3, "image must be [B,3,H,W]"
        tb = self._check_operands(B, H, W, text_emb, eps, (x, noise_map, out, out_latent))
        if out is None:
            out = torch.empty_like(x)
        self._forward(B, H, W, text_emb, tb, eps, out_latent, direction=direction, x=_ptr(x), noise_map=_ptr(noise_map),
                      r=float(r), out=_ptr(out))
        return out

    def forward_u8(self, x_u8: torch.Tensor, in_mode: int, text_emb: Optional[torch.Tensor], eps: torch.Tensor,
                   noise_map: Optional[torch.Tensor] = None, r: float = 1.0, direction: int = A2B,
                   out: Optional[torch.Tensor] = None, out_latent: Optional[torch.Tensor] = None, *,
                   resize=None, crop=None, out_size=None) -> torch.Tensor:
        """uint8 HWC boundary: x_u8 [B,H,W,3] uint8 CUDA -> [B,H,W,3] uint8 CUDA (pre/post-processing fused on device).

        With a geometry (see resize_geometry) the PIL LANCZOS resizes around the forward run on device too: x_u8 is resized to
        `resize` (H, W), the network runs on the `crop` (top, left, height, width) window, and its output image is resized to
        `out_size` (H, W).  eps / noise_map / out_latent then have the crop's size."""
        B, Hi, Wi, Cc = x_u8.shape
        assert Cc == 3 and x_u8.dtype == torch.uint8 and x_u8.is_cuda and x_u8.is_contiguous(), "image must be uint8 CUDA [B,H,W,3]"
        rs, (cy, cx, H, W), osz = resize_geometry((Hi, Wi), resize, crop, out_size)
        tb = self._check_operands(B, H, W, text_emb, eps, (noise_map, out_latent))
        if out is None:
            out = torch.empty(B, osz[0], osz[1], 3, dtype=torch.uint8, device=x_u8.device)
        assert out.dtype == torch.uint8 and out.is_cuda and out.is_contiguous() and out.shape == (B, osz[0], osz[1], 3)
        # without resize / crop / out_size this is the identity geometry, which runs the plan of the plain uint8 forward
        g = ResizeDesc(Hi, Wi, rs[0], rs[1], cy, cx, osz[0], osz[1])
        self._forward(B, H, W, text_emb, tb, eps, out_latent, direction=direction, x_u8=_ptr(x_u8), in_mode=int(in_mode),
                      geometry=C.pointer(g), noise_map=_ptr(noise_map), r=float(r), out_u8=_ptr(out))
        return out

    def forward_variations(self, x1: torch.Tensor, text_emb: Optional[torch.Tensor], eps: torch.Tensor,
                           noise_map: Optional[torch.Tensor] = None, r: float = 1.0, direction: int = A2B,
                           out: Optional[torch.Tensor] = None, out_latent: Optional[torch.Tensor] = None) -> torch.Tensor:
        """n = eps.shape[0] variations of ONE image x1 [1,3,H,W]: eps / noise_map / out / out_latent have batch n, text_emb
        batch 1 or n.  The VAE encoder runs once; output i equals image i of forward() on x1 repeated n times, bit for bit."""
        B, Cc, H, W = x1.shape
        if B != 1 or Cc != 3:
            raise ValueError(f"forward_variations takes one image [1,3,H,W], got {list(x1.shape)}")
        n = eps.shape[0]
        tb = self._check_operands(n, H, W, text_emb, eps, (x1, noise_map, out, out_latent))
        if out is None:
            out = torch.empty(n, 3, H, W, device=x1.device, dtype=x1.dtype)
        self._forward(n, H, W, text_emb, tb, eps, out_latent, direction=direction, shared_input=1, x=_ptr(x1),
                      noise_map=_ptr(noise_map), r=float(r), out=_ptr(out))
        return out

    def forward_u8_variations(self, x_u8_1: torch.Tensor, in_mode: int, text_emb: Optional[torch.Tensor], eps: torch.Tensor,
                              noise_map: Optional[torch.Tensor] = None, r: float = 1.0, direction: int = A2B,
                              out: Optional[torch.Tensor] = None, out_latent: Optional[torch.Tensor] = None, *,
                              resize=None, crop=None, out_size=None) -> torch.Tensor:
        """forward_u8 on ONE image x_u8_1 [1,H,W,3] with n = eps.shape[0] outputs [n,out_H,out_W,3] (see forward_variations);
        the resize / crop / out_size geometry is forward_u8's.  The input resize runs once, the output resize per output."""
        B, Hi, Wi, Cc = x_u8_1.shape
        assert Cc == 3 and x_u8_1.dtype == torch.uint8 and x_u8_1.is_cuda and x_u8_1.is_contiguous(), \
            "image must be uint8 CUDA [1,H,W,3]"
        if B != 1:
            raise ValueError(f"forward_u8_variations takes one image [1,H,W,3], got {list(x_u8_1.shape)}")
        n = eps.shape[0]
        rs, (cy, cx, H, W), osz = resize_geometry((Hi, Wi), resize, crop, out_size)
        tb = self._check_operands(n, H, W, text_emb, eps, (noise_map, out_latent))
        if out is None:
            out = torch.empty(n, osz[0], osz[1], 3, dtype=torch.uint8, device=x_u8_1.device)
        assert out.dtype == torch.uint8 and out.is_cuda and out.is_contiguous() and out.shape == (n, osz[0], osz[1], 3)
        g = ResizeDesc(Hi, Wi, rs[0], rs[1], cy, cx, osz[0], osz[1])
        self._forward(n, H, W, text_emb, tb, eps, out_latent, direction=direction, shared_input=1, x_u8=_ptr(x_u8_1),
                      in_mode=int(in_mode), geometry=C.pointer(g), noise_map=_ptr(noise_map), r=float(r), out_u8=_ptr(out))
        return out

    def forward_u8_ragged(self, images: Sequence[torch.Tensor], in_mode: int, text_emb: Optional[torch.Tensor],
                          eps: torch.Tensor, noise_map: Optional[torch.Tensor] = None, r: float = 1.0, direction: int = A2B, *,
                          geometries, max_side: Optional[int] = None, outs: Optional[Sequence[torch.Tensor]] = None,
                          out_latent: Optional[torch.Tensor] = None):
        """forward_u8 on n = len(images) uint8 images of their own sizes ([H_i, W_i, 3] contiguous CUDA tensors) in one forward
        at batch n.  geometries[i] is image i's forward_u8 keywords as a dict (resize, crop, out_size); every crop has the
        network size H x W, and eps / noise_map / out_latent are [n, 4, H/8, W/8].  Returns the n outputs [out_H_i, out_W_i, 3]
        (or fills `outs`).  Output i equals forward_u8(images[i][None], ..., **geometries[i]) with eps[i], byte for byte.

        max_side: the plan's capacity, at least every in / resize / out dimension; None takes ragged_max_side of the call's
        dimensions, so a stream of calls with the same n reuses one plan and one graph."""
        return self._forward_u8_ragged("forward_u8_ragged", images, in_mode, text_emb, eps, geometries, max_side, outs,
                                       out_latent, noise_map=noise_map, r=r, direction=direction)

    def forward_mixed(self, x: torch.Tensor, text_emb: Optional[torch.Tensor], eps: torch.Tensor, directions,
                      out: Optional[torch.Tensor] = None, out_latent: Optional[torch.Tensor] = None) -> torch.Tensor:
        """CycleGAN forward of a batch that mixes both directions (ForwardDesc.directions): image i through vae (directions[i]
        == A2B) or vae_b2a (B2A).  Output i equals image i of forward(..., direction=directions[i]) byte for byte; one plan and
        one CUDA graph serve every mix.  A refused size raises ValueError with the engine's rule (mixed_size_check)."""
        B, Cc, H, W = x.shape
        assert Cc == 3, "image must be [B,3,H,W]"
        dirs = directions_array(directions, B)
        why = mixed_size_check(H, W)
        if why:
            raise ValueError("mixed-direction forward: " + why)
        tb = self._check_operands(B, H, W, text_emb, eps, (x, out, out_latent))
        if out is None:
            out = torch.empty_like(x)
        self._forward(B, H, W, text_emb, tb, eps, out_latent, directions=dirs, x=_ptr(x), out=_ptr(out))
        return out

    def forward_u8_ragged_mixed(self, images: Sequence[torch.Tensor], in_mode: int, text_emb: Optional[torch.Tensor],
                                eps: torch.Tensor, directions, *, geometries, max_side: Optional[int] = None,
                                outs: Optional[Sequence[torch.Tensor]] = None, out_latent: Optional[torch.Tensor] = None):
        """forward_u8_ragged with a direction per image (ForwardDesc.directions): uploads of any size, both directions,
        one plan.  Output i equals forward_u8(images[i][None], ..., direction=directions[i], **geometries[i]) byte for byte."""
        return self._forward_u8_ragged("forward_u8_ragged_mixed", images, in_mode, text_emb, eps, geometries, max_side, outs,
                                       out_latent, directions=directions)

    def _forward_u8_ragged(self, what, images, in_mode, text_emb, eps, geometries, max_side, outs, out_latent, *,
                           noise_map=None, r=0.0, direction=A2B, directions=None):
        """The body of forward_u8_ragged and forward_u8_ragged_mixed (directions given: a mixed batch, which has no noise_map)."""
        n = len(images)
        _check_u8_images(images, what)
        dirs = directions_array(directions, n) if directions is not None else None
        H, W, descs = _ragged_descs(geometries, [tuple(x.shape[:2]) for x in images])
        if dirs is not None:
            why = mixed_size_check(H, W)
            if why:
                raise ValueError("mixed-direction forward: " + why)
        if eps.shape[0] != n:
            raise ValueError(f"{n} images but eps has batch {eps.shape[0]}")
        tb = self._check_operands(n, H, W, text_emb, eps, (noise_map, out_latent))
        if max_side is None:
            max_side = ragged_max_side([v for d in descs for v in (d.in_H, d.in_W, d.resize_H, d.resize_W, d.out_H, d.out_W)])
        if outs is None:
            outs = [torch.empty(d.out_H, d.out_W, 3, dtype=torch.uint8, device=images[0].device) for d in descs]
        if len(outs) != n or any(tuple(o.shape) != (d.out_H, d.out_W, 3) or o.dtype != torch.uint8 or not o.is_cuda
                                 or not o.is_contiguous() for o, d in zip(outs, descs)):
            raise ValueError("outs must be n contiguous uint8 CUDA tensors [out_H_i, out_W_i, 3]")
        self._forward(n, H, W, text_emb, tb, eps, out_latent, direction=direction, directions=dirs, x_u8_list=_ptrs(images),
                      in_mode=int(in_mode), geometry=descs, max_side=int(max_side), noise_map=_ptr(noise_map), r=float(r),
                      out_u8_list=_ptrs(outs))
        return list(outs)

    def graph_captures(self) -> int:
        """CUDA graphs this engine has captured (a replayed forward captures none)."""
        n = C.c_int(0)
        self._check(self.lib.i2it_debug_graph_captures(self._h, C.byref(n)), "i2it_debug_graph_captures")
        return n.value

    def prep_launch_count(self) -> int:
        n = C.c_int(0)
        self._check(self.lib.i2it_prep_launch_count(self._h, C.byref(n)), "i2it_prep_launch_count")
        return n.value

    def launch_count(self, B: int, H: int, W: int, direction: int = A2B) -> int:
        n = C.c_int(0)
        self._check(self.lib.i2it_launch_count(self._h, B, H, W, direction, C.byref(n)), "i2it_launch_count")
        return n.value

    def profile(self, reps: int = 3):
        """Per-launch timings of the last forward's plan: list of dicts (kind, ms, flops, bytes, shape)."""
        import json
        cap = 1 << 22
        buf = C.create_string_buffer(cap)
        self._check(self.lib.i2it_profile(self._h, reps, buf, cap, _stream()), "i2it_profile")
        return json.loads(buf.value.decode())

    def workspace_bytes(self, B: int, H: int, W: int) -> int:
        n = C.c_size_t(0)
        self._check(self.lib.i2it_workspace_bytes(self._h, B, H, W, C.byref(n)), "i2it_workspace_bytes")
        return n.value

    # ---- plan cache ------------------------------------------------------------------------------
    def set_max_plans(self, max_plans: int):
        """Keep at most `max_plans` forward plans (0: no limit); the least recently run one is evicted first and rebuilt,
        with identical outputs, when its shape returns.  The last forward's plan is never evicted."""
        self._check(self.lib.i2it_set_max_plans(self._h, int(max_plans)), "i2it_set_max_plans")

    def release_plans(self):
        """Drop every forward plan and unmap the shared workspace (prepared weights and the set_text cache are kept)."""
        self._check(self.lib.i2it_release_plans(self._h), "i2it_release_plans")

    def memory_stats(self) -> dict:
        """{"arena_bytes", "plan_bytes", "plans", "plan_builds", "plan_evictions"}: the workspace shared by the forward plans,
        the plans' own persistent bytes, the resident plans and the build / eviction counters."""
        s = MemoryStats()
        self._check(self.lib.i2it_memory_stats_get(self._h, C.byref(s)), "i2it_memory_stats_get")
        return {name: getattr(s, name) for name, _ in MemoryStats._fields_}

    def _debug_poison_workspace(self, value: int = 0xFF):
        """Fill the shared workspace with `value` (tests: no forward may read workspace it did not write)."""
        self._check(self.lib.i2it_debug_poison_workspace(self._h, int(value)), "i2it_debug_poison_workspace")

    def _debug_tapgemm_override(self, bn: int = 0, stages: int = 0, grid: int = 0):
        """Force tapgemm's tile width, ring depth and persistent grid in the op_* calls that follow (0: the engine's choice;
        forward plans never read it).  An op whose launch cannot take a value raises with the legal range."""
        self._check(self.lib.i2it_debug_tapgemm_override(self._h, int(bn), int(stages), int(grid)),
                    "i2it_debug_tapgemm_override")

    def read_stage(self, name: str, max_elems: int = 1 << 26, image: Optional[int] = None) -> torch.Tensor:
        """fp32 NCHW copy of a named stage of the last forward (keep_stages engines); image=i reads one image of the batch."""
        if image is not None:
            name = f"{name}@{int(image)}"
        dims = (C.c_int * 4)()
        buf = torch.empty(max_elems, dtype=torch.float32, device="cuda")
        self._check(self.lib.i2it_read_stage(self._h, name.encode(), _ptr(buf), max_elems, dims), f"i2it_read_stage({name})")
        n, c, h, w = list(dims)
        return buf[: n * c * h * w].view(n, c, h, w).clone()

    def _json(self, fn, what, cap=1 << 22):
        import json
        buf = C.create_string_buffer(cap)
        self._check(fn(self._h, buf, cap), what)
        return json.loads(buf.value.decode())

    def stage_names(self):
        """[(name, (N, C, H, W))] of every stage the last forward kept, in build order."""
        return [(s["name"], tuple(s["dims"])) for s in self._json(self.lib.i2it_stage_names, "i2it_stage_names")]

    def text_stage_names(self):
        """[(name, (N, C, H, W))] of every stage the last encode_text kept, in build order (read them with read_stage)."""
        return [(s["name"], tuple(s["dims"])) for s in self._json(self.lib.i2it_text_stage_names, "i2it_text_stage_names")]

    def _debug_refold_info(self) -> dict:
        """What the last refold rebuilt: {"recipes": prepared-weight keys in fold order, "jobs", "gemv_jobs", "bytes": the
        algorithmic bytes those jobs read and write}."""
        return self._json(self.lib.i2it_debug_refold_info, "i2it_debug_refold_info")

    def prepared_keys(self):
        """Cache keys of every prepared weight (plain layer names, "+sc", ".qk", "|twin", "|im2col", "|subpixel", "identity|n")."""
        return self._json(self.lib.i2it_prepared_keys, "i2it_prepared_keys")

    def read_prepared(self, key: str):
        """A prepared weight as the kernels read it: ([taps, rows, cin_pad] in the engine dtype, fp32 bias [rows] or None)."""
        dims = (C.c_int * 4)()
        self._check(self.lib.i2it_read_prepared(self._h, key.encode(), None, 0, None, 0, dims), f"i2it_read_prepared({key})")
        taps, rows, cin_pad, has_bias = list(dims)
        w = torch.empty(taps, rows, cin_pad, device="cuda", dtype=self.dtype)
        b = torch.empty(rows, device="cuda", dtype=torch.float32) if has_bias else None
        self._check(self.lib.i2it_read_prepared(self._h, key.encode(), _ptr(w), w.numel(), _ptr(b), rows if has_bias else 0, dims),
                    f"i2it_read_prepared({key})")
        return w, b

    # ---- diagnostic single ops (NHWC tensors in the engine dtype; weights fp32 CUDA) -----------------
    def op_conv2d(self, x_nhwc, w, bias=None, stride=1, asym_pad=False, residual=None, act=ACT_NONE, out_fp32=False):
        N, H, W, Cin = x_nhwc.shape
        Cout, _, k, _ = w.shape
        oc = Cout // 2 if act == ACT_GEGLU else Cout
        # ceil(H / stride): an odd map is padded to even before a stride-2 conv, as F.conv2d(stride=2, padding=1) sizes it
        out = torch.empty(N, -(-H // stride), -(-W // stride), oc, device="cuda",
                          dtype=torch.float32 if out_fp32 else self.dtype)
        w = w.float().contiguous()
        b = bias.float().contiguous() if bias is not None else None
        self._check(self.lib.i2it_op_conv2d(self._h, _ptr(x_nhwc), N, H, W, Cin, x_nhwc.stride(2), _ptr(w), _ptr(b), Cout, k,
                                            stride, int(asym_pad), _ptr(residual),
                                            residual.stride(2) if residual is not None else 0, act, _ptr(out), oc,
                                            int(out_fp32), _stream()), "i2it_op_conv2d")
        return out

    def op_conv2d_sel(self, x_nhwc, w, bias, w_alt, bias_alt, directions, *, w2_alt=None, **kw):
        """op_conv2d_ex with a second weight set chosen per image (i2it_op_conv2d_sel): image n uses (w_alt, bias_alt, w2_alt)
        where directions[n] == 1.  w2_alt None shares w2.  Keywords as op_conv2d_ex."""
        dirs = directions_array(directions, x_nhwc.shape[0])
        keep = [w_alt.float().contiguous(), bias_alt.float().contiguous() if bias_alt is not None else None,
                w2_alt.float().contiguous() if w2_alt is not None else None]
        return self.op_conv2d_ex(x_nhwc, w, bias, _sel=(keep, dirs), **kw)

    def op_conv2d_ex(self, x_nhwc, w, bias=None, *, stride=1, asym_pad=False, residual=None, act=ACT_NONE, out=None,
                     out_fp32=False, x2=None, w2=None, up2x=False, tokens=False, gn=None, gn_out=None, _sel=None):
        """Every conv variant of the engine (i2it_conv_desc).  NHWC views may be channel slices (pixel stride > C);
        `out` / `gn_out` are optional preallocated views.  gn = (gamma, beta, eps, silu) adds the GroupNorm that consumes the
        output.  Returns out, or (out, groupnorm output) when gn is given."""
        N, H, W, Cin = x_nhwc.shape
        Cout, _, k, _ = w.shape
        oc = Cout // 2 if act == ACT_GEGLU else Cout
        Ho, Wo = (2 * H, 2 * W) if up2x else (-(-H // stride), -(-W // stride))
        dt = torch.float32 if out_fp32 else self.dtype
        if out is None:
            out = torch.empty(N, Ho, Wo, oc, device="cuda", dtype=dt)
        assert out.shape == (N, Ho, Wo, oc) and out.dtype == dt and out.stride(3) == 1
        keep = [w.float().contiguous(), bias.float().contiguous() if bias is not None else None,
                w2.float().contiguous() if w2 is not None else None]
        d = ConvDesc()
        d.x, d.N, d.H, d.W, d.Cin, d.ldx = x_nhwc.data_ptr(), N, H, W, Cin, x_nhwc.stride(2)
        d.w, d.bias, d.Cout, d.ksize, d.stride, d.asym_pad = _ptr(keep[0]), _ptr(keep[1]), Cout, k, stride, int(asym_pad)
        d.residual, d.ldr = _ptr(residual), residual.stride(2) if residual is not None else 0
        d.act, d.out, d.ldo, d.out_fp32 = act, out.data_ptr(), out.stride(2), int(out_fp32)
        if x2 is not None:
            d.x2, d.C2, d.ld2, d.w2 = x2.data_ptr(), x2.shape[3], x2.stride(2), _ptr(keep[2])
        d.up2x, d.tokens = int(up2x), int(tokens)
        g = None
        if gn is not None:
            gamma, beta, eps, silu = gn
            g = gn_out if gn_out is not None else torch.empty(N, Ho, Wo, oc, device="cuda", dtype=self.dtype)
            keep += [gamma.float().contiguous(), beta.float().contiguous()]
            d.gn_y, d.ldg, d.gn_silu, d.gn_eps = g.data_ptr(), g.stride(2), int(silu), float(eps)
            d.gn_gamma, d.gn_beta = _ptr(keep[3]), _ptr(keep[4])
        if _sel is not None:
            (wa, ba, w2a), dirs = _sel
            self._check(self.lib.i2it_op_conv2d_sel(self._h, C.byref(d), _ptr(wa), _ptr(ba), _ptr(w2a), dirs, _stream()),
                        "i2it_op_conv2d_sel")
        else:
            self._check(self.lib.i2it_op_conv2d_ex(self._h, C.byref(d), _stream()), "i2it_op_conv2d_ex")
        return (out, g) if gn is not None else out

    def op_launches(self):
        """Launch list of the last op call: [{"kind", "shape"}...]."""
        import json
        cap = 1 << 16
        buf = C.create_string_buffer(cap)
        self._check(self.lib.i2it_op_launches(self._h, buf, cap), "i2it_op_launches")
        return json.loads(buf.value.decode())

    def op_group_norm(self, x_nhwc, gamma, beta, eps, silu):
        N, H, W, Cc = x_nhwc.shape
        out = torch.empty_like(x_nhwc)
        self._check(self.lib.i2it_op_group_norm(self._h, _ptr(x_nhwc), N, H * W, Cc, x_nhwc.stride(2), _ptr(gamma.float()),
                                                _ptr(beta.float()), eps, int(silu), _ptr(out), Cc, _stream()),
                    "i2it_op_group_norm")
        return out

    def op_layer_norm(self, x, gamma, beta, eps=1e-5):
        rows, Cc = x.shape
        out = torch.empty_like(x)
        self._check(self.lib.i2it_op_layer_norm(self._h, _ptr(x), rows, Cc, x.stride(0), _ptr(gamma.float()), _ptr(beta.float()),
                                                eps, _ptr(out), Cc, _stream()), "i2it_op_layer_norm")
        return out

    def op_attention(self, q, k, vt, heads, causal=False):
        """q [B, Nq, C], k [1|B, Nk, C], vt [1|B, C, ldv >= Nk].  Rows may be strided (q and k as column slices of one fused
        projection), but the C ABI takes one leading dimension per operand: image b must start b * rows * ld elements in."""
        B, Nq, Cc = q.shape
        kvb, Nk, _ = k.shape
        for t, rows in ((q, Nq), (k, Nk), (vt, Cc)):
            if t.stride(2) != 1 or (t.shape[0] > 1 and t.stride(0) != rows * t.stride(1)):
                raise ValueError(f"op_attention: operand of shape {list(t.shape)} has strides {t.stride()}; images must be "
                                 "[rows, ld] blocks with unit column stride")
        out = torch.empty(B, Nq, Cc, device=q.device, dtype=q.dtype)
        self._check(self.lib.i2it_op_attention(self._h, _ptr(q), q.stride(1), _ptr(k), k.stride(1), _ptr(vt), vt.stride(1), B, Nq,
                                               Nk, heads, Cc // heads, kvb, int(causal), _ptr(out), Cc, _stream()),
                    "i2it_op_attention")
        return out

    def op_vt_proj(self, x, w, bias=None):
        """x [B, ntok, Cin] -> (w @ x[b]^T + bias[:, None]) as [B, Cout, round_up(ntok, 8)] (columns past ntok are padding)."""
        B, ntok, Cin = x.shape
        Cout = w.shape[0]
        out = torch.empty(B, Cout, (ntok + 7) // 8 * 8, device="cuda", dtype=self.dtype)
        w = w.float().contiguous()
        b = bias.float().contiguous() if bias is not None else None
        self._check(self.lib.i2it_op_vt_proj(self._h, _ptr(x), B, ntok, Cin, x.stride(1), _ptr(w), _ptr(b), Cout, _ptr(out),
                                             _stream()), "i2it_op_vt_proj")
        return out

    def op_upsample2x(self, x_nhwc):
        N, H, W, Cc = x_nhwc.shape
        out = torch.empty(N, 2 * H, 2 * W, Cc, device="cuda", dtype=self.dtype)
        self._check(self.lib.i2it_op_upsample2x(self._h, _ptr(x_nhwc), N, H, W, Cc, _ptr(out), _stream()), "i2it_op_upsample2x")
        return out

    def op_upsample_to(self, x_nhwc, Ho, Wo):
        N, H, W, Cc = x_nhwc.shape
        out = torch.empty(N, Ho, Wo, Cc, device="cuda", dtype=self.dtype)
        self._check(self.lib.i2it_op_upsample_to(self._h, _ptr(x_nhwc), N, H, W, Cc, Ho, Wo, _ptr(out), _stream()),
                    "i2it_op_upsample_to")
        return out

    def op_resize_u8(self, x, H2, W2):
        """PIL LANCZOS resize of uint8 HWC CUDA images: [B, H, W, 3] -> [B, H2, W2, 3] (synchronous)."""
        B, H, W, Cc = x.shape
        assert Cc == 3 and x.dtype == torch.uint8 and x.is_cuda and x.is_contiguous(), "image must be uint8 CUDA [B,H,W,3]"
        out = torch.empty(B, H2, W2, 3, dtype=torch.uint8, device=x.device)
        self._check(self.lib.i2it_op_resize_u8(self._h, _ptr(x), B, H, W, _ptr(out), H2, W2, _stream()), "i2it_op_resize_u8")
        return out

    def op_resize_u8_ragged(self, images, sizes, max_side: Optional[int] = None):
        """PIL LANCZOS resize of uint8 HWC CUDA images of their own sizes, images[i] [H_i, W_i, 3] -> [sizes[i][0], sizes[i][1], 3],
        in the two ragged launches of forward_u8_ragged (synchronous).  max_side None: ragged_max_side of the sizes."""
        n = len(images)
        _check_u8_images(images, "op_resize_u8_ragged")
        if len(sizes) != n:
            raise ValueError(f"{n} images but {len(sizes)} sizes")
        hw_in = [int(v) for x in images for v in x.shape[:2]]
        hw_out = [int(v) for s in sizes for v in s]
        if max_side is None:
            max_side = ragged_max_side(hw_in + hw_out)
        outs = [torch.empty(int(s[0]), int(s[1]), 3, dtype=torch.uint8, device=images[0].device) for s in sizes]
        self._check(self.lib.i2it_op_resize_u8_ragged(self._h, _ptrs(images), (C.c_int * (2 * n))(*hw_in), _ptrs(outs),
                                                      (C.c_int * (2 * n))(*hw_out), n, int(max_side), _stream()),
                    "i2it_op_resize_u8_ragged")
        return outs
