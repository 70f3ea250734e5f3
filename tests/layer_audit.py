"""Teacher-forced layer audit: every layer of one forward, and every prepared weight, against float64.

The walker follows the graph of oracle/oracle.py (VAE encoder, UNet, DDPM step, VAE decoder) over a *source* that provides

    stage_names()          names of the kept stages, in build order (an engine run with keep_stages = 2)
    read_stage(name)       a stage as an fp32 NCHW tensor (exact copy of the 16-bit values)
    prepared_keys()        every prepared-weight cache key
    read_prepared(key)     ([taps, rows, cin_pad] 16-bit weight, fp32 bias or None), as the kernels read them
    inputs                 dict: x (NCHW image, engine dtype), text (the prompt the forward or i2it_set_text used), eps,
                           noise (or None), image (the forward's output, or None)

For each layer it takes the engine's OWN input stages and prepared operands, computes that single op in float64 with
tests/kref.py and holds the engine's output to the per-element bound of its kernel family, so the error of earlier layers
never carries into a check.  Separately, every prepared weight and bias is compared with the float64 fold of the state
dict in the engine layout.  Every stage name and every prepared key must be audited exactly once (`Audit.run` asserts it).

The same walker, with `emulate=True`, builds a source: each layer is computed in float64 from the previous rounded stage
and rounded once, and each prepared weight is round16 of the float64 fold.  tests/test_layer_audit.py uses it to show that
the audit passes on a correct pipeline and names the layer of each injected error.
"""
from __future__ import annotations

import math
from typing import Callable, Dict, List, Optional

import torch
import torch.nn.functional as F

import kref

EPS24 = kref.EPS24
MEAN_ULP_MIN_ELEMS = 1024       # smaller GEMM outputs are held to the per-element bound only

# checkpoint names that are the same tensor as a layer stage (keep_stages = 1 names): checked bit-equal to the layer
def _aliases(vp: str) -> Dict[str, str]:
    e, d = vp + "encoder", vp + "decoder"
    a = {"skip0": f"{e}.conv_in", "enc_mid": f"{e}.mid_block.resnets.1.conv2", "dec_mid": f"{d}.mid_block.resnets.1.conv2",
         "unet_mid": "unet.mid_block.resnets.1.conv2", "dec_up3": f"{d}.up_blocks.3.resnets.2.conv2"}
    for i in (1, 2, 3):
        a[f"skip{i}"] = f"{e}.down_blocks.{i - 1}.downsamplers.0.conv"
    for i in (0, 1, 2):
        a[f"dec_up{i}"] = f"{d}.up_blocks.{i}.upsamplers.0.conv"
    return a


class Spec:
    """What the forward computed: model kind, config, fold parameters (as given to the engine)."""

    def __init__(self, sd, cfg, kind="pix2pix", direction="a2b", r=None, adapter_scales=None, lw_unet=1.0, lw_vae=1.0,
                 skip_gamma=1.0, twin_r=-1.0):
        self.sd, self.cfg, self.kind, self.direction = sd, cfg, kind, direction
        self.r = r                                   # None: deterministic (no noise blend)
        self.adapter_scales = adapter_scales or ({"default": 1.0, "vae_skip": 2.0} if kind == "pix2pix" else
                                                 {"default_encoder": 1.0, "default_decoder": 1.0, "default_others": 1.0,
                                                  "vae_skip": 2.0})
        self.lw_unet, self.lw_vae, self.skip_gamma, self.twin_r = lw_unet, lw_vae, skip_gamma, twin_r
        self.vp = "vae_b2a." if (kind == "cyclegan" and direction == "b2a") else "vae."


class AuditError(AssertionError):
    pass


class Audit:
    def __init__(self, src, spec: Spec, dtype, emulate=False, stage_hook=None, weight_hook=None):
        self.src, self.spec, self.dt, self.emulate = src, spec, dtype, emulate
        self.sd, self.cfg, self.vp = spec.sd, spec.cfg, spec.vp
        self.dev = src.inputs["x"].device
        self._sd_cache = {}
        self.results = []                       # (family, name, Check-like)
        self.stages_seen: List[str] = []
        self.keys_seen: List[str] = []
        self.stage_hook, self.weight_hook = stage_hook, weight_hook
        self.used_keys = set()
        if emulate:
            src.stages, src.order, src.prepared = {}, [], {}

    # ------------------------------------------------------------------------------------------------ plumbing
    def P(self, name):
        """fp32 state-dict tensor on the audit device, as float64."""
        if name not in self._sd_cache:
            self._sd_cache[name] = self.sd[name].to(self.dev).double()
        return self._sd_cache[name]

    def has(self, name):
        return name in self.sd

    def S(self, name):
        """A stage as float64 NHWC (channel padding kept)."""
        return self.src.read_stage(name).to(self.dev).double().permute(0, 2, 3, 1)

    def W(self, key):
        """A prepared weight: (w [taps, rows, cin_pad] float64, bias float64 or None)."""
        self.used_keys.add(key)
        if self.emulate and key not in self.src.prepared:
            w64, b, _ = self.expected(key)
            w = w64.to(self.dt)
            bb = b.float() if b is not None else None
            if self.weight_hook:
                w, bb = self.weight_hook(key, w, bb, self)
            self.src.prepared[key] = (w, bb)
        w, b = self.src.read_prepared(key)
        return w.to(self.dev).double(), (b.to(self.dev).double() if b is not None else None)

    def conv_w(self, key, cin, k=None):
        """prepared weight in PyTorch layout [rows, cin, k, k] (padding columns dropped) + bias."""
        w, b = self.W(key)
        taps = w.shape[0]
        k = k or int(round(math.sqrt(taps)))
        return w[:, :, :cin].permute(1, 2, 0).reshape(w.shape[1], cin, k, k), b

    def emit(self, family, name, ref_nchw, check: Callable, exact=False, pad_zero=True):
        """Audit: compare stage `name` with the reference.  Emulate: store round16(ref) (the reference itself if exact)."""
        self.stages_seen.append(name)
        if self.emulate:
            v = ref_nchw if exact else kref.round16(ref_nchw, self.dt)
            if self.stage_hook:
                v = self.stage_hook(name, v, self)
            self.src.stages[name] = v if self.dt == torch.float64 else v.float()     # float64: no rounding anywhere
            self.src.order.append(name)
            return
        got = self.src.read_stage(name).to(self.dev).double()
        C = ref_nchw.shape[1]
        extra = None
        if pad_zero and got.shape[1] > C:
            pad = got[:, C:]
            if bool((pad != 0).any()):
                extra = f"{int((pad != 0).sum())} nonzero padding channels"
        got = got[:, :C]
        c = check(got)
        if extra is not None:
            c.ok, c.extra = False, extra
        self.results.append((family, name, c))

    def gemm(self, family, name, ref, mag, K, factor=1.0, pad_zero=True):
        if ref.numel() >= MEAN_ULP_MIN_ELEMS:
            chk = lambda got: kref.check_gemm(name, got, ref, mag, K, self.dt, factor)
        else:   # a handful of correctly rounded elements can average above 0.30 ulp by chance: per-element bound only
            chk = lambda got: kref.Check(name, got, ref, kref.gemm_bound(ref, mag, K, self.dt, factor), self.dt)
        self.emit(family, name, ref, chk, pad_zero=pad_zero)

    def exact(self, family, name, ref):
        self.emit(family, name, ref, lambda got: _Exact(name, got, ref), exact=True)

    # ------------------------------------------------------------------------------------------------ layer kinds
    def conv(self, name, x, key, *, k=3, stride=1, asym=False, res=None, x2=None, key2=None, family="conv"):
        """conv / linear (NHWC x) with optional identity residual and second 1x1 source; output stage `name`."""
        w, b = self.conv_w(key, x.shape[3], k)
        # stride 2 on an odd map: the engine's pad-to-even copy is the zero padding conv64 applies
        ref = kref.conv64(x, w, b, stride=stride, asym=asym)
        mag = kref.conv64(x.abs(), w.abs(), b.abs() if b is not None else None, stride=stride, asym=asym)
        K = x.shape[3] * k * k
        if x2 is not None:
            w2, _ = self.conv_w(key2, x2.shape[3], 1)
            ref, mag, K = ref + kref.conv64(x2, w2), mag + kref.conv64(x2.abs(), w2.abs()), K + x2.shape[3]
        if res is not None:
            r = res.permute(0, 3, 1, 2)
            ref, mag = ref + r, mag + r.abs()
        self.gemm(family, name, ref, mag, K)
        return ref

    def linear(self, name, x, key, res=None, family="linear"):
        return self.conv(name, x, key, k=1, res=res, family=family)

    def group_norm(self, name, x, norm, eps, silu):
        ref, bound = kref.group_norm64(x, self.P(norm + ".weight"), self.P(norm + ".bias"), eps, silu, self.dt)
        ref, bound = ref.permute(0, 3, 1, 2), bound.permute(0, 3, 1, 2)
        self.emit("groupnorm", name, ref, lambda got: kref.check_norm(name, got, ref, bound, self.dt))

    def layer_norm(self, name, x, norm, eps=1e-5):
        ref, bound = kref.layer_norm64(x, self.P(norm + ".weight"), self.P(norm + ".bias"), eps, self.dt)
        ref, bound = ref.permute(0, 3, 1, 2), bound.permute(0, 3, 1, 2)
        self.emit("layernorm", name, ref, lambda got: kref.check_norm(name, got, ref, bound, self.dt))

    def vt(self, name, x_tok, key):
        """V^T projection: stage [B, ldv, 1, C] holds V[b, t, c] at (b, t, 0, c); token padding is not checked."""
        w, b = self.conv_w(key, x_tok.shape[2], 1)
        x = x_tok.unsqueeze(1)                                          # [B, 1, ntok, Cin] as NHWC
        ref = kref.conv64(x, w, b)                                      # [B, C, 1, ntok]
        mag = kref.conv64(x.abs(), w.abs(), b.abs() if b is not None else None)
        t = lambda v: v.permute(0, 3, 2, 1)                             # -> [B, ntok, 1, C]
        self.gemm("linear", name, t(ref), t(mag), x_tok.shape[2], pad_zero=False)

    def read_v(self, name, ntok):
        return self.S(name)[:, 0, :, :ntok].transpose(1, 2)            # NHWC [B, 1, C, ldv] -> V [B, ntok, C]

    def flash_path(self, heads, d, Nk):
        """Whether the source's engine ran this attention on a flash kernel, whose probabilities are relative to the row
        maximum (tests/kref.py header): d = 64 unless the engine was created with I2IT_NO_FLASH, and the one-head d = 512
        attention above 8192 keys.  A source that does not say (the emulated one) gets the unfused set, which contains it."""
        if not getattr(self.src, "flash", False):
            return False
        return d == 64 or (d == 512 and heads == 1 and Nk > 8192)

    def attention(self, name, q, k, v, heads, H, W, causal=False):
        """q [B, Nq, C], k / v [kvB, Nk, C] (the engine's own operands) -> stage [B, C, H, W]."""
        flash = self.flash_path(heads, q.shape[2] // heads, k.shape[1])
        o, pav, e_s, psub = kref.attention64(q, k, v, heads, causal=causal, flash=flash)
        B, C = q.shape[0], q.shape[2]
        sp = lambda t: t.reshape(B, H, W, C).permute(0, 3, 1, 2)
        ref, pav, e_s, psub = sp(o), sp(pav), sp(e_s), sp(psub)
        self.emit("attention", name, ref, lambda got: kref.check_attention(name, got, ref, pav, e_s, psub, k.shape[1], self.dt))

    # ------------------------------------------------------------------------------------------------ blocks
    def vae_resnet(self, p, x, skip=None, skip_key=None):
        self.group_norm(p + ".norm1", x, p + ".norm1", 1e-6, True)
        self.conv(p + ".conv1", self.S(p + ".norm1"), p + ".conv1")
        h = self.S(p + ".conv1")
        self.group_norm(p + ".norm2", h, p + ".norm2", 1e-6, True)
        h = self.S(p + ".norm2")
        if self.has(p + ".conv_shortcut.weight"):
            self.conv(p + ".conv2", h, p + ".conv2+sc", x2=x, key2=p + ".conv_shortcut")
        else:
            self.conv(p + ".conv2", h, p + ".conv2", res=x, x2=skip, key2=skip_key)
        return self.S(p + ".conv2")

    def vae_attn(self, p, x):
        B, H, W, C = x.shape
        self.group_norm(p + ".group_norm", x, p + ".group_norm", 1e-6, False)
        t = self.S(p + ".group_norm")
        self.linear(p + ".qk", t, p + ".qk")
        qk = self.S(p + ".qk").reshape(B, H * W, 2 * C)
        self.vt(p + ".to_v", t.reshape(B, H * W, C), p + ".to_v")
        v = self.read_v(p + ".to_v", H * W)
        self.attention(p, qk[..., :C], qk[..., C:], v, 1, H, W)
        self.linear(p + ".to_out.0", self.S(p), p + ".to_out.0", res=x)
        return self.S(p + ".to_out.0")

    def unet_resnet(self, p, x):
        self.group_norm(p + ".norm1", x, p + ".norm1", 1e-5, True)
        self.conv(p + ".conv1", self.S(p + ".norm1"), p + ".conv1")
        self.group_norm(p + ".norm2", self.S(p + ".conv1"), p + ".norm2", 1e-5, True)
        h = self.S(p + ".norm2")
        if self.has(p + ".conv_shortcut.weight"):
            self.conv(p + ".conv2", h, p + ".conv2+sc", x2=x, key2=p + ".conv_shortcut")
        else:
            self.conv(p + ".conv2", h, p + ".conv2", res=x)
        return self.S(p + ".conv2")

    def xformer(self, p, x, heads, text_batch):
        B, H, W, C = x.shape
        N = H * W
        b = p + ".transformer_blocks.0"
        tok = lambda n: self.S(n).reshape(B, N, -1)
        self.group_norm(p + ".norm", x, p + ".norm", 1e-6, False)
        self.linear(p + ".proj_in", self.S(p + ".norm"), p + ".proj_in")
        t = self.S(p + ".proj_in")
        # self-attention
        self.layer_norm(b + ".norm1", t, b + ".norm1")
        n = self.S(b + ".norm1")
        self.linear(b + ".attn1.qk", n, b + ".attn1.qk")
        qk = tok(b + ".attn1.qk")
        self.vt(b + ".attn1.to_v", n.reshape(B, N, C), b + ".attn1.to_v")
        self.attention(b + ".attn1", qk[..., :C], qk[..., C:], self.read_v(b + ".attn1.to_v", N), heads, H, W)
        self.linear(b + ".attn1.to_out.0", self.S(b + ".attn1"), b + ".attn1.to_out.0", res=t)
        t = self.S(b + ".attn1.to_out.0")
        # cross-attention: K / V^T must be this block's projection of the prompt (inline or cached by i2it_set_text)
        self.layer_norm(b + ".norm2", t, b + ".norm2")
        self.linear(b + ".attn2.to_q", self.S(b + ".norm2"), b + ".attn2.to_q")
        text = self.text.view(text_batch, 1, 77, -1)
        self.linear(b + ".attn2.to_k", text, b + ".attn2.to_k")
        self.vt(b + ".attn2.to_v", text.view(text_batch, 77, -1), b + ".attn2.to_v")
        k = self.S(b + ".attn2.to_k").reshape(text_batch, 77, C)
        self.attention(b + ".attn2", tok(b + ".attn2.to_q"), k, self.read_v(b + ".attn2.to_v", 77), heads, H, W)
        self.linear(b + ".attn2.to_out.0", self.S(b + ".attn2"), b + ".attn2.to_out.0", res=t)
        t = self.S(b + ".attn2.to_out.0")
        # GEGLU feed-forward: the prepared rows interleave (h, g) pairs
        self.layer_norm(b + ".norm3", t, b + ".norm3")
        self.geglu(b + ".ff.net.0.proj", self.S(b + ".norm3"), b + ".ff.net.0.proj")
        self.linear(b + ".ff.net.2", self.S(b + ".ff.net.0.proj"), b + ".ff.net.2", res=t)
        self.linear(p + ".proj_out", self.S(b + ".ff.net.2"), p + ".proj_out", res=x)
        return self.S(p + ".proj_out")

    def geglu(self, name, x, key):
        w, b = self.conv_w(key, x.shape[3], 1)
        ref = kref.conv64(x, w, b)
        mag = kref.conv64(x.abs(), w.abs(), b.abs() if b is not None else None)
        h, g = ref[:, 0::2], ref[:, 1::2]
        mh, mg = mag[:, 0::2], mag[:, 1::2]
        self.gemm("linear", name, h * kref.gelu64(g), mh * kref.gelu64(g).abs() + h.abs() * mg, x.shape[3], factor=2.0)

    def subpixel(self, name, x, key, skip, skip_key):
        """nearest-2x + conv3x3 as four parity convs over the pre-summed taps the engine prepared, + the skip conv."""
        w, b = self.W(key)
        rows, cin = w.shape[1], x.shape[3]
        wsub = w[:, :, :cin].reshape(4, 2, 2, rows, cin).permute(0, 3, 4, 1, 2)      # [phase, rows, cin, ty, tx]
        ref = kref.subpixel_conv64(x, wsub, b)
        mag = kref.subpixel_conv64(x.abs(), wsub.abs(), b.abs())
        w2, _ = self.conv_w(skip_key, skip.shape[3], 1)
        ref, mag = ref + kref.conv64(skip, w2), mag + kref.conv64(skip.abs(), w2.abs())
        self.gemm("conv", name, ref, mag, 4 * cin + skip.shape[3])

    # ------------------------------------------------------------------------------------------------ the graph
    def walk(self):
        inp = self.src.inputs
        self.text = inp["text"].to(self.dev).double()
        vp, e, d = self.vp, self.vp + "encoder", self.vp + "decoder"
        ch = self.cfg["unet_channels"]
        heads = self.cfg["unet_heads"]
        x = inp["x"].to(self.dev)
        B = x.shape[0]
        text_batch = self.text.shape[0]
        # ---- VAE encoder: conv_in over the im2col rows [B, H, W, 32] (k = tap * 3 + c, 27..31 zero)
        xp = F.pad(x.double(), (1, 1, 1, 1))
        H, W = x.shape[2], x.shape[3]
        cols = [xp[:, c, ky:ky + H, kx:kx + W] for ky in range(3) for kx in range(3) for c in range(3)]
        col = torch.stack(cols + [torch.zeros_like(cols[0])] * 5, dim=1)
        self.exact("pack", e + ".conv_in.im2col", col)
        self.conv(e + ".conv_in", self.S(e + ".conv_in.im2col")[..., :27], e + ".conv_in|im2col", k=1)
        s = self.S(e + ".conv_in")
        skips = []
        for i in range(4):
            skips.append(s)
            for j in range(2):
                s = self.vae_resnet(f"{e}.down_blocks.{i}.resnets.{j}", s)
            if i < 3:
                dn = f"{e}.down_blocks.{i}.downsamplers.0.conv"
                self.conv(dn, s, dn, stride=2, asym=True)
                s = self.S(dn)
        s = self.vae_resnet(e + ".mid_block.resnets.0", s)
        s = self.vae_attn(e + ".mid_block.attentions.0", s)
        s = self.vae_resnet(e + ".mid_block.resnets.1", s)
        self.group_norm(e + ".conv_norm_out", s, e + ".conv_norm_out", 1e-6, True)
        self.conv(e + ".conv_out", self.S(e + ".conv_norm_out"), e + ".conv_out")
        self.conv("moments", self.S(e + ".conv_out")[..., :8], vp + "quant_conv", k=1)
        self.latent(self.S("moments"))
        # ---- UNet
        z = self.S("latent")[..., :4]
        if self.has("unet.conv_in.conv_in_pretrained.weight"):
            self.conv("unet.conv_in", z, "unet.conv_in.conv_in_pretrained|twin")
        else:
            self.conv("unet.conv_in", z, "unet.conv_in")
        s = self.S("unet.conv_in")
        res = [s]
        for i in range(4):
            blk = f"unet.down_blocks.{i}"
            for j in range(2):
                s = self.unet_resnet(f"{blk}.resnets.{j}", s)
                if i < 3:
                    s = self.xformer(f"{blk}.attentions.{j}", s, heads[i], text_batch)
                res.append(s)
            if i < 3:
                self.conv(f"{blk}.downsamplers.0.conv", s, f"{blk}.downsamplers.0.conv", stride=2)
                s = self.S(f"{blk}.downsamplers.0.conv")
                res.append(s)
        s = self.unet_resnet("unet.mid_block.resnets.0", s)
        s = self.xformer("unet.mid_block.attentions.0", s, heads[3], text_batch)
        s = self.unet_resnet("unet.mid_block.resnets.1", s)
        for i in range(4):
            blk = f"unet.up_blocks.{i}"
            for j in range(3):
                cat = f"{blk}.resnets.{j}.concat"
                self.exact("concat", cat, torch.cat([s, res.pop()], dim=3).permute(0, 3, 1, 2))
                s = self.unet_resnet(f"{blk}.resnets.{j}", self.S(cat))
                if i > 0:
                    s = self.xformer(f"{blk}.attentions.{j}", s, heads[3 - i], text_batch)
            if i < 3:
                Ho, Wo = res[-1].shape[1], res[-1].shape[2]
                up = f"{blk}.upsamplers.0.nearest"
                self.exact("upsample", up, F.interpolate(s.permute(0, 3, 1, 2), size=(Ho, Wo), mode="nearest"))
                self.conv(f"{blk}.upsamplers.0.conv", self.S(up), f"{blk}.upsamplers.0.conv")
                s = self.S(f"{blk}.upsamplers.0.conv")
        self.group_norm("unet.conv_norm_out", s, "unet.conv_norm_out", 1e-5, True)
        self.conv("model_pred", self.S("unet.conv_norm_out"), "unet.conv_out")
        # ---- DDPM step (bit-exact: the scheduler arithmetic of each wrapper) and the decoder input
        self.exact("ddpm", "dec_in", F.pad(self.ddpm(z, self.S("model_pred")[..., :4]), (0, 0, 0, 0, 0, 4)))
        # ---- VAE decoder
        self.conv(vp + "post_quant_conv", self.S("dec_in")[..., :4], vp + "post_quant_conv", k=1)
        self.conv(d + ".conv_in", self.S(vp + "post_quant_conv")[..., :4], d + ".conv_in")
        s = self.S(d + ".conv_in")
        sk = lambda i: f"{d}.skip_conv_{i + 1}"
        s = self.vae_resnet(d + ".mid_block.resnets.0", s)
        s = self.vae_attn(d + ".mid_block.attentions.0", s)
        s = self.vae_resnet(d + ".mid_block.resnets.1", s, skips[3], sk(0))
        for i in range(4):
            for j in range(3):
                s = self.vae_resnet(f"{d}.up_blocks.{i}.resnets.{j}", s)
            if i < 3:
                u = f"{d}.up_blocks.{i}.upsamplers.0.conv"
                self.subpixel(u, s, u + "|subpixel", skips[2 - i], sk(i + 1))
                s = self.S(u)
        self.group_norm(d + ".conv_norm_out", s, d + ".conv_norm_out", 1e-6, True)
        g = self.S(d + ".conv_norm_out")
        ref = self.conv("pre_clamp", g, d + ".conv_out")
        if inp.get("image") is not None and not self.emulate:   # the final launch writes clamp(conv_out) as NCHW
            w, b = self.conv_w(d + ".conv_out", g.shape[3], 3)
            mag = kref.conv64(g.abs(), w.abs(), b.abs())
            img = inp["image"].to(self.dev).double()
            self.results.append(("conv", "image", kref.check_gemm("image", img, ref.clamp(-1, 1), mag, g.shape[3] * 9, self.dt)))
        # ---- the keep_stages = 1 checkpoints are the same tensors as layer stages
        for a, n in _aliases(vp).items():
            self.stages_seen.append(a)
            if self.emulate:
                self.src.stages[a] = self.src.stages[n]
                self.src.order.append(a)
            elif not torch.equal(self.src.read_stage(a), self.src.read_stage(n)):
                self.results.append(("alias", a, _Fail(a, f"differs from {n}")))

    def latent(self, mom):
        """mean + exp(0.5 clamp(logvar, -30, 20)) eps, times sf; stochastic: round16 of that, blended with the noise map."""
        eps = self.src.inputs["eps"].to(self.dev).double().permute(0, 2, 3, 1)
        mean, lv = mom[..., :4], mom[..., 4:8].clamp(-30.0, 20.0)
        sf = float(torch.tensor(self.cfg["scaling_factor"], dtype=torch.float32))
        std = torch.exp(0.5 * lv)
        v = (mean + std * eps) * sf
        mag = (mean.abs() + std * eps.abs()) * sf
        bound = kref.ulp16(v, self.dt) + 8 * EPS24 * mag
        if self.spec.r is not None:
            r = float(torch.tensor(self.spec.r, dtype=torch.float32))
            noise = self.src.inputs["noise"].to(self.dev).double().permute(0, 2, 3, 1)
            # the kernel rounds the encoded latent to 16 bits before the blend (as the reference does): that rounding may
            # land one 16-bit ulp away from round16(v) next to a tie, scaled by r
            vr = kref.round16(v, self.dt)
            bound = kref.ulp16(vr * r + noise * (1 - r), self.dt) + kref.ulp16(v, self.dt) * r + \
                8 * EPS24 * (vr.abs() * r + noise.abs() * (1 - r)) + 8 * EPS24 * mag * r
            v = vr * r + noise * (1 - r)
        ref = F.pad(v, (0, 4)).permute(0, 3, 1, 2)
        bnd = F.pad(bound, (0, 4), value=1.0).permute(0, 3, 1, 2)
        self.emit("latent", "latent", ref, lambda got: kref.Check("latent", got, ref[:, :got.shape[1]], bnd[:, :got.shape[1]], self.dt))

    def ddpm(self, sample, pred):
        """x0 / sf exactly as the wrappers' scheduler call rounds it (tests/test_gpu_boundary.py), NCHW."""
        from _host import OneStepDDPM
        dt = self.dt
        s, p = sample.to(dt).permute(0, 3, 1, 2), pred.to(dt).permute(0, 3, 1, 2)
        ac = OneStepDDPM().alphas_cumprod.to(self.dev)
        if self.spec.kind == "cyclegan":
            t = torch.tensor([999], device=self.dev).long()[0]
            a = ac[t]
            x0 = torch.stack([(s[i] - (1 - a) ** 0.5 * p[i]) / a ** 0.5 for i in range(s.shape[0])])
        else:
            a = ac[torch.tensor([999], device=self.dev).long()]
            x0 = ((s - (1 - a) ** 0.5 * p) / a ** 0.5).to(dt)
        return (x0 / self.cfg["scaling_factor"]).double()

    # ------------------------------------------------------------------------------------------------ prepared weights
    def fold64(self, name, mag=False):
        """W + sum_a s_a * lw * B_a @ A_a in float64 (PyTorch layout), lw = lw_unet for unet.*, lw_vae otherwise.
        mag: |W| + sum_a |s_a lw| |B_a| @ |A_a|, the scale of the fp32 fold's rounding error."""
        m = (lambda t: t.abs()) if mag else (lambda t: t)
        w = m(self.P(name + ".weight")).clone()
        pre = name + ".lora_A."
        lw = self.spec.lw_unet if name.startswith("unet.") else self.spec.lw_vae
        for a in sorted({k[len(pre):].rsplit(".", 1)[0] for k in self.sd if k.startswith(pre)}):
            s = self.spec.adapter_scales[a] * lw
            if s == 0:
                continue
            A, Bm = m(self.P(f"{pre}{a}.weight")), m(self.P(f"{name}.lora_B.{a}.weight"))
            s = m(torch.tensor(s)).item()
            if w.dim() == 2:
                w = w + s * (Bm @ A)
            else:
                w = w + s * torch.einsum("or,rikl->oikl", Bm[:, :, 0, 0], A)
        return w

    @staticmethod
    def layout(w, cin_pad):
        """[rows, cin(, k, k)] -> engine [taps][rows][cin_pad]."""
        if w.dim() == 2:
            w = w[:, :, None, None]
        rows, cin = w.shape[:2]
        out = w.reshape(rows, cin, -1).permute(2, 0, 1)
        return F.pad(out, (0, cin_pad - cin))

    def temb64(self, p):
        """time_emb_proj(silu(linear_2(silu(linear_1(te))))) in float64, te = oracle.timestep_embedding (fp32), and its bound.
        te itself is defined only to fp32 accuracy of its frequencies: a one-ulp change of f_i moves 999 f_i by ~1e-4, which
        libm and torch disagree on; that sensitivity is part of the bound."""
        import oracle as O
        C0, T = self.cfg["unet_channels"][0], self.cfg["temb_dim"]
        te = O.timestep_embedding(999, C0)[0].to(self.dev).double()
        half = C0 // 2
        f = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float64, device=self.dev) / half)
        dte = (999 * 4 * f * 2.0 ** -24 + 2 * EPS24).repeat(2)
        silu = lambda v: v * torch.sigmoid(v)
        err, x = dte, te
        for n, act in (("unet.time_embedding.linear_1", True), ("unet.time_embedding.linear_2", True), (p + ".time_emb_proj", False)):
            w, b = self.fold64(n), self.P(n + ".bias")
            h = w @ x + b
            e_lin = (w.shape[1] + 8) * EPS24 * (w.abs() @ x.abs() + b.abs()) + w.abs() @ err
            if act:
                x, err = silu(h), 1.1 * e_lin + 4 * EPS24 * silu(h).abs()
            else:
                x, err = h, e_lin
        return x, err

    def expected(self, key, mag=False):
        """(float64 weight in engine layout, reference bias, bias bound or None for exact) of a prepared-weight key.
        mag: the same re-layout of the fold magnitudes (every re-layout sums with non-negative coefficients); no bias."""
        sp = self.spec
        fold = lambda n: self.fold64(n, mag)
        if key.startswith("identity|"):
            n = int(key.split("|")[1])
            return torch.eye(n, dtype=torch.float64, device=self.dev)[None], None, None
        if key.endswith("|twin"):
            pre = key[:-5]
            cur = pre.replace("conv_in_pretrained", "conv_in_curr")
            r = float(torch.tensor(sp.twin_r, dtype=torch.float32))
            w = (1 - r) * fold(pre) + r * fold(cur)
            b = (1 - r) * self.P(pre + ".bias") + r * self.P(cur + ".bias")
            # c0 = 1 - r and both products round in fp32 before the sum
            bb = 4 * EPS24 * ((1 - r) * self.P(pre + ".bias").abs() + r * self.P(cur + ".bias").abs())
            return self.layout(w, _pad8(w.shape[1])), b, bb + 2 * kref.ulp16(b, torch.float32)
        if key.endswith("|im2col"):
            n = key[:-7]
            w = fold(n)                                          # [rows, 3, 3, 3] -> k = tap * 3 + c
            col = F.pad(w.permute(0, 2, 3, 1).reshape(w.shape[0], 27), (0, 5))
            return col[None], self.P(n + ".bias"), None
        if key.endswith("|subpixel"):
            n = key[:-9]
            w = fold(n)
            sub = kref.subpixel_weights(w, torch.float64)              # [4, rows, cin, 2, 2], summed in float64
            out = sub.permute(0, 3, 4, 1, 2).reshape(16, w.shape[0], w.shape[1])
            return F.pad(out, (0, _pad8(w.shape[1]) - w.shape[1])), self.P(n + ".bias"), None
        if key.endswith("+sc"):
            p = key[:-len(".conv2+sc")]
            w = fold(p + ".conv2")
            b = self.P(p + ".conv2.bias") + self.P(p + ".conv_shortcut.bias")
            return self.layout(w, _pad8(w.shape[1])), b, 2 * kref.ulp16(b, torch.float32)
        if key.endswith(".qk"):
            p = key[:-3]
            wq, wk = fold(p + ".to_q"), fold(p + ".to_k")
            w = torch.cat([wq, wk])
            b = torch.cat([self.P(p + ".to_q.bias"), self.P(p + ".to_k.bias")]) if self.has(p + ".to_q.bias") else None
            return self.layout(w, _pad8(w.shape[1])), b, None
        w = fold(key)
        b = self.P(key + ".bias") if self.has(key + ".bias") else None
        if ".skip_conv_" in key:
            w = w * float(torch.tensor(sp.skip_gamma, dtype=torch.float32))
        if key.endswith("ff.net.0.proj"):
            half = w.shape[0] // 2
            idx = torch.empty(w.shape[0], dtype=torch.long, device=self.dev)
            idx[0::2], idx[1::2] = torch.arange(half, device=self.dev), torch.arange(half, 2 * half, device=self.dev)
            w, b = w[idx], b[idx]
        if mag:
            return self.layout(w, _pad8(w.shape[1])), None, None
        bnd = None
        if key.startswith("unet.") and key.endswith(".conv1"):
            t, e = self.temb64(key[:-len(".conv1")])
            b = b + t
            bnd = e + 2 * kref.ulp16(b, torch.float32)
        return self.layout(w, _pad8(w.shape[1])), b, bnd

    def max_rank(self):
        if not hasattr(self, "_max_rank"):
            self._max_rank = max([v.shape[0] for k, v in self.sd.items() if ".lora_A." in k] or [0])
        return self._max_rank

    def cin_of(self, key):
        """input width of the layer behind a key (columns past it, up to cin_pad, are padding)."""
        for suf, base in (("|twin", ""), ("|subpixel", ""), ("+sc", ""), (".qk", ".to_q")):
            if key.endswith(suf):
                return self.sd[key[:-len(suf)] + base + ".weight"].shape[1]
        return self.sd[key + ".weight"].shape[1]

    def check_prepared(self, key):
        w64, bref, bbound = self.expected(key)
        got, gb = self.src.read_prepared(key)
        got, gb = got.to(self.dev).double(), (gb.to(self.dev).double() if gb is not None else None)
        if got.shape != w64.shape:
            return _Fail(key, f"layout {tuple(got.shape)} != {tuple(w64.shape)}")
        # the fp32 fold: up to rank products and sums, the TwinConv / gamma coefficients, four sub-pixel taps
        c = kref.check_weights(key, got, w64, self.dt, fold_err=(self.max_rank() + 8) * EPS24 * self.expected(key, mag=True)[0])
        bad = []
        if key.endswith("|im2col"):
            pad = got[..., 27:]
        elif key.startswith("identity|"):
            pad = torch.zeros(0)
        else:
            pad = got[..., self.cin_of(key):]
        if pad.numel() and bool((pad != 0).any()):
            bad.append(f"{int((pad != 0).sum())} nonzero padding columns")
        if key.startswith("identity|") and not torch.equal(got, w64):
            bad.append("not an exact identity")
        if (bref is None) != (gb is None):
            bad.append(f"bias present: {gb is not None}, expected {bref is not None}")
        elif bref is not None:
            if bbound is None:
                if not torch.equal(gb, bref.float().double()):
                    bad.append(f"bias not bit-equal ({int((gb != bref.float().double()).sum())} elements)")
            else:
                r = ((gb - bref).abs() / bbound).max().item()
                c.bias_worst = r
                if r > 1:
                    i = int(((gb - bref).abs() / bbound).argmax())
                    bad.append(f"bias err/bound {r:.3g} at row {i} (got {gb[i].item():.6g}, ref {bref[i].item():.6g})")
        if bad:
            c.ok, c.extra = False, "; ".join(bad)
        return c

    # ------------------------------------------------------------------------------------------------ driver
    def audited_keys(self, keys):
        """The prepared keys this audit owns: the forward's (the CLIP text tower's are tests/text_audit.py's)."""
        return [k for k in keys if not k.startswith("text_encoder.")]

    def run(self, require_complete=True):
        self.walk()
        keys = sorted(self.used_keys) if self.emulate else self.audited_keys(self.src.prepared_keys())
        for k in keys:
            self.keys_seen.append(k)
            if not self.emulate:
                self.results.append(("weight", k, self.check_prepared(k)))
        if self.emulate:
            self.src.keys = keys
            return self
        # completeness: every stage and every prepared key audited exactly once
        names = self.src.stage_names()
        dup = sorted({n for n in self.stages_seen if self.stages_seen.count(n) > 1})
        missing = [n for n in names if n not in set(self.stages_seen)]
        extra = [n for n in self.stages_seen if n not in set(names)]
        unused = sorted(set(keys) - self.used_keys - {k for k in keys if k.startswith("identity|")})
        self.completeness = dict(duplicate=dup, unaudited=missing, not_kept=extra, unused_keys=unused)
        if require_complete and (dup or missing or extra or unused):
            raise AuditError(f"audit is not complete: {self.completeness}")
        return self

    def failures(self):
        return [(f, n, c) for f, n, c in self.results if not c]

    def report(self):
        """One line per failure, then the worst err/bound and mean-ulp per family."""
        lines = [f"FAIL {f} {c}" + (f" ({c.extra})" if getattr(c, "extra", None) else "") for f, _, c in self.failures()]
        fam = {}
        for f, n, c in self.results:
            w = fam.setdefault(f, [0, 0.0, "", 0.0])
            w[0] += 1
            if c.worst >= w[1]:
                w[1], w[2] = c.worst, n
            w[3] = max(w[3], c.mean_ulp)
        for f, (cnt, worst, n, mu) in sorted(fam.items()):
            lines.append(f"{f:10s} {cnt:4d} checks  worst err/bound {worst:.3f} ({n})  worst mean-ulp {mu:.3f}")
        return "\n".join(lines)

    def assert_ok(self):
        bad = self.failures()
        assert not bad, "layer audit failed:\n" + self.report()


def _pad8(c):
    return (c + 7) // 8 * 8


class _Exact:
    """Bit-exact comparison with the Check interface."""

    def __init__(self, name, got, ref):
        self.name = name
        ref = ref.to(got.dtype)
        self.n_bad = int((got != ref).sum())
        self.numel = got.numel()
        self.worst = 0.0 if self.n_bad == 0 else float("inf")
        self.mean_ulp = 0.0
        self.where = (got != ref).nonzero()[:4].tolist()
        self.ok = self.n_bad == 0

    def __bool__(self):
        return self.ok

    def __str__(self):
        return f"{'PASS' if self.ok else 'FAIL'} [{self.name}] bit-exact: {self.n_bad}/{self.numel} differ" + \
            (f" at {self.where}" if self.n_bad else "")


class _Fail(_Exact):
    def __init__(self, name, why):
        self.name, self.ok, self.worst, self.mean_ulp, self.n_bad, self.numel, self.where = name, False, float("inf"), 0.0, 1, 1, []
        self.extra = why


class EmulatedSource:
    """A source whose stages are the float64 layer references rounded once (Audit(emulate=True) fills it)."""

    def __init__(self, inputs):
        self.inputs = inputs
        self.stages, self.order, self.prepared, self.keys = {}, [], {}, []

    def read_stage(self, name):
        return self.stages[name]

    def stage_names(self):
        return list(self.order)

    def prepared_keys(self):
        return list(self.keys)

    def read_prepared(self, key):
        return self.prepared[key]


class EngineSource:
    """The engine after one forward with keep_stages = 2."""

    def __init__(self, engine, inputs):
        self.e, self.inputs = engine, inputs
        self._cache = {}
        self._dims = dict(engine.stage_names())

    @property
    def flash(self):
        return self.e.flash

    def read_stage(self, name):
        if name not in self._cache:
            N, C, H, W = self._dims[name]
            self._cache[name] = self.e.read_stage(name, max_elems=max(N * C * H * W, 1))
        return self._cache[name]

    def stage_names(self):
        return [n for n, _ in self.e.stage_names()]

    def prepared_keys(self):
        return self.e.prepared_keys()

    def read_prepared(self, key):
        return self.e.read_prepared(key)
