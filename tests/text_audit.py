"""Teacher-forced audit of the CLIP text tower (Engine::encode_text): every layer and every prepared weight against float64.

The walker follows transformers' CLIPTextTransformer (token + position embeddings, pre-LN layers with causal self-attention
and a GELU / quick-GELU MLP, final LayerNorm) over a source in the format of tests/layer_audit.py, whose stages are the
ones an engine with keep_stages = 2 keeps under the transformers state-dict prefixes (T = text_encoder.text_model,
L = T.encoder.layers.{l}):

    T.embeddings                 bit-exact: round16(tok[id] + pos[t]), one fp32 add
    L.layer_norm1, L.layer_norm2 kref.layer_norm64 with the tower's epsilon
    L.self_attn.qk               fused q|k projection                          kref.check_gemm
    L.self_attn.v_proj           V^T [B][C][ldv], as the UNet's to_v stages    kref.check_gemm
    L.self_attn                  causal softmax(Q K^T / 8) V                   kref.check_attention
    L.self_attn.out_proj         + residual                                    kref.check_gemm
    L.mlp.fc1                    + GELU / quick-GELU (factor 2)                kref.check_gemm
    L.mlp.fc2                    + residual                                    kref.check_gemm

The final LayerNorm writes into the caller's buffer: it is checked on the tensor encode_text returned (inputs["out"]).
The tower has no LoRA, so each prepared weight (L.qk, L.self_attn.v_proj, L.self_attn.out_proj, L.mlp.fc1, L.mlp.fc2)
must be bit-equal to round16(W) in the engine layout ([q; k] rows, zero padding columns) and each bias bit-equal to its
fp32 tensor.  Source inputs: tokens [B, 77] and out [B, 77, C] (the returned last_hidden_state).

With emulate=True the walker builds a source instead (each layer in float64 from the previous rounded stage, rounded
once); with dtype float64 nothing is rounded, which pins the walker's composition to CLIPTextModel.double().
"""
from __future__ import annotations

import torch

import kref
import layer_audit as LA

T = "text_encoder.text_model"


class TextSpec:
    """What the tower computes: its "text_encoder."-prefixed fp32 tensors, heads, activation and LayerNorm epsilon."""

    def __init__(self, sd, heads, act="gelu", eps=1e-5):
        self.sd, self.heads, self.act, self.eps = sd, heads, act, eps
        self.layers = 0
        while f"{T}.encoder.layers.{self.layers}.layer_norm1.weight" in sd:
            self.layers += 1

    @classmethod
    def from_model(cls, m):
        """From a transformers CLIPTextModel."""
        c = m.config
        sd = {"text_encoder." + k: v.detach().float().cpu() for k, v in m.state_dict().items()}
        return cls(sd, int(c.num_attention_heads), str(c.hidden_act), float(c.layer_norm_eps))


def clip_model(hidden, layers, heads, inter, act="gelu", seed=0, eps=1e-5):
    """A CLIPTextModel from its config alone (no hub access), with every bias and LayerNorm perturbed away from the default
    init (biases 0, LayerNorms (1, 0)) so that each one is exercised."""
    from transformers import CLIPTextConfig, CLIPTextModel
    cfg = CLIPTextConfig(vocab_size=49408, hidden_size=hidden, intermediate_size=inter, num_hidden_layers=layers,
                         num_attention_heads=heads, max_position_embeddings=77, hidden_act=act, layer_norm_eps=eps)
    torch.manual_seed(seed)
    m = CLIPTextModel(cfg).eval()
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith(".bias"):
                p.normal_(0, 0.02)
            elif "layer_norm" in n and n.endswith(".weight"):
                p.normal_(1.0, 0.1)
    return m


def eos_tokens(B, seed=0, pad=49407):
    """CLIP-style rows: BOS, 5 + 9 b random ids, EOS, then `pad` to 77."""
    g = torch.Generator().manual_seed(seed)
    rows = []
    for b in range(B):
        ids = [49406] + torch.randint(1, 49000, (5 + 9 * b,), generator=g).tolist() + [49407]
        rows.append(ids + [pad] * (77 - len(ids)))
    return torch.tensor(rows, dtype=torch.long)


class TextAudit(LA.Audit):
    def __init__(self, src, spec: TextSpec, dtype, emulate=False, stage_hook=None, weight_hook=None):
        self.src, self.spec, self.dt, self.emulate = src, spec, dtype, emulate
        self.sd = spec.sd
        self.dev = src.inputs["tokens"].device
        self._sd_cache = {}
        self.results = []
        self.stages_seen, self.keys_seen = [], []
        self.stage_hook, self.weight_hook = stage_hook, weight_hook
        self.used_keys = set()
        if emulate:
            src.stages, src.order, src.prepared = {}, [], {}

    # ------------------------------------------------------------------------------------------------ layers
    def embeddings(self, ids):
        """tok[id] + pos[t] as the kernel forms it: one fp32 add, rounded once (float64 emulation: not rounded)."""
        acc = torch.float64 if self.dt == torch.float64 else torch.float32
        tok = self.sd[T + ".embeddings.token_embedding.weight"].to(self.dev).to(acc)
        pos = self.sd[T + ".embeddings.position_embedding.weight"].to(self.dev).to(acc)
        e = (tok[ids] + pos[: ids.shape[1]]).to(self.dt).double()                      # [B, ntok, C]
        self.exact("embedding", T + ".embeddings", e.permute(0, 2, 1).unsqueeze(2))     # NCHW [B, C, 1, ntok]

    def fc1(self, name, x, key):
        w, b = self.conv_w(key, x.shape[3], 1)
        z = kref.conv64(x, w, b)
        mag = kref.conv64(x.abs(), w.abs(), b.abs() if b is not None else None)
        act = kref.quick_gelu64 if self.spec.act == "quick_gelu" else kref.gelu64
        self.gemm("linear", name, act(z), mag, x.shape[3], factor=2.0)               # |GELU'| <= 1.13, |quick-GELU'| <= 1.1

    def final_norm(self, x):
        name = T + ".final_layer_norm"
        B, _, ntok, C = x.shape
        ref, bound = kref.layer_norm64(x, self.P(name + ".weight"), self.P(name + ".bias"), self.spec.eps, self.dt)
        if self.emulate:
            v = kref.round16(ref, self.dt).permute(0, 3, 1, 2)                          # NCHW, as the stage hooks see stages
            if self.stage_hook:
                v = self.stage_hook(name, v, self)
            self.src.inputs["out"] = v[:, :, 0, :].transpose(1, 2).contiguous()
            return
        got = self.src.inputs["out"].to(self.dev).double().reshape(B, ntok, C)
        self.results.append(("layernorm", name, kref.check_norm(name, got, ref.reshape(B, ntok, C), bound.reshape(B, ntok, C),
                                                                self.dt)))

    def walk(self):
        sp = self.spec
        ids = self.src.inputs["tokens"].to(self.dev).long()
        B, ntok = ids.shape
        self.embeddings(ids)
        x = self.S(T + ".embeddings")                                                   # NHWC [B, 1, ntok, C]
        C = x.shape[3]
        for l in range(sp.layers):
            L = f"{T}.encoder.layers.{l}"
            self.layer_norm(L + ".layer_norm1", x, L + ".layer_norm1", sp.eps)
            n = self.S(L + ".layer_norm1")
            self.linear(L + ".self_attn.qk", n, L + ".qk")
            qk = self.S(L + ".self_attn.qk").reshape(B, ntok, 2 * C)
            self.vt(L + ".self_attn.v_proj", n.reshape(B, ntok, C), L + ".self_attn.v_proj")
            v = self.read_v(L + ".self_attn.v_proj", ntok)
            self.attention(L + ".self_attn", qk[..., :C], qk[..., C:], v, sp.heads, 1, ntok, causal=True)
            self.linear(L + ".self_attn.out_proj", self.S(L + ".self_attn"), L + ".self_attn.out_proj", res=x)
            x = self.S(L + ".self_attn.out_proj")
            self.layer_norm(L + ".layer_norm2", x, L + ".layer_norm2", sp.eps)
            self.fc1(L + ".mlp.fc1", self.S(L + ".layer_norm2"), L + ".mlp.fc1")
            self.linear(L + ".mlp.fc2", self.S(L + ".mlp.fc1"), L + ".mlp.fc2", res=x)
            x = self.S(L + ".mlp.fc2")
        self.final_norm(x)

    # ------------------------------------------------------------------------------------------------ prepared weights
    def expected(self, key, mag=False):
        """(float64 weight in engine layout, fp32 bias or None, None): the fused q|k key stacks q_proj over k_proj."""
        if key.endswith(".qk"):
            p = key[:-len(".qk")] + ".self_attn."
            w = torch.cat([self.P(p + "q_proj.weight"), self.P(p + "k_proj.weight")])
            b = torch.cat([self.P(p + "q_proj.bias"), self.P(p + "k_proj.bias")]) if self.has(p + "q_proj.bias") else None
        else:
            w = self.P(key + ".weight")
            b = self.P(key + ".bias") if self.has(key + ".bias") else None
        return self.layout(w, LA._pad8(w.shape[1])), b, None

    def check_prepared(self, key):
        """No fold: the weight (padding columns included) bit-equal to round16(W), the bias bit-equal to its fp32 tensor."""
        w64, bref, _ = self.expected(key)
        got, gb = self.src.read_prepared(key)
        got, gb = got.to(self.dev).double(), (gb.to(self.dev).double() if gb is not None else None)
        if got.shape != w64.shape:
            return LA._Fail(key, f"layout {tuple(got.shape)} != {tuple(w64.shape)}")
        c = LA._Exact(key, got, kref.round16(w64, self.dt))
        if (bref is None) != (gb is None):
            c.ok, c.extra = False, f"bias present: {gb is not None}, expected {bref is not None}"
        elif bref is not None and not torch.equal(gb, bref.float().double()):
            c.ok, c.extra = False, f"bias not bit-equal ({int((gb != bref.float().double()).sum())} elements)"
        if not c.ok:
            c.worst = float("inf")
        return c

    def audited_keys(self, keys):
        return [k for k in keys if k.startswith("text_encoder.")]


class TextEngineSource(LA.EngineSource):
    """The engine after one encode_text with keep_stages = 2 (inputs: tokens, out)."""

    def __init__(self, engine, inputs):
        self.e, self.inputs = engine, inputs
        self._cache = {}
        self._dims = dict(engine.text_stage_names())

    def stage_names(self):
        return [n for n, _ in self.e.text_stage_names()]
