"""CPU: the CLIP text-tower audit (tests/text_audit.py), the token checks of i2it.Engine.encode_text, and the epsilon guard
that keeps a differently configured tower off the engine.

The walker is pinned to transformers first: with rounding switched off its composition of float64 layers must equal
CLIPTextModel.double().  Then the emulated bf16 pipeline must pass the audit, and each injected error, one a whole-tower
mean-error bound can miss, must fail on exactly the layer or prepared weight that carries it (teacher forcing)."""
from types import SimpleNamespace

import pytest
import torch

import kref
import layer_audit as LA
import text_audit as TA

DT = torch.bfloat16
T = TA.T
L0, L1 = f"{T}.encoder.layers.0", f"{T}.encoder.layers.1"


@pytest.fixture(scope="module")
def gelu_tower():
    return TA.clip_model(128, 2, 2, 256, "gelu")


@pytest.fixture(scope="module")
def quick_tower():
    return TA.clip_model(192, 3, 3, 512, "quick_gelu", seed=1)


def _audit(spec, tokens, dt=DT, stage_hook=None, weight_hook=None):
    src = LA.EmulatedSource(dict(tokens=tokens, out=None))
    with torch.no_grad():
        TA.TextAudit(src, spec, dt, emulate=True, stage_hook=stage_hook, weight_hook=weight_hook).run()
        return TA.TextAudit(src, spec, dt).run()


def _failed(a):
    return sorted(n for _, n, _ in a.failures())


@pytest.mark.parametrize("tower", ["gelu_tower", "quick_tower"])
def test_float64_walk_matches_transformers(tower, request):
    m = request.getfixturevalue(tower)
    tokens = TA.eos_tokens(3)
    src = LA.EmulatedSource(dict(tokens=tokens, out=None))
    with torch.no_grad():
        TA.TextAudit(src, TA.TextSpec.from_model(m), torch.float64, emulate=True).run()
        ref = m.double()(tokens)[0]
        m.float()
    got = src.inputs["out"]
    assert got.dtype == torch.float64 and got.shape == ref.shape
    rel = ((got - ref).abs().max() / ref.abs().max()).item()
    assert rel < 1e-12, rel


@pytest.mark.parametrize("tower", ["gelu_tower", "quick_tower"])
def test_audit_passes_on_emulated_pipeline(tower, request):
    spec = TA.TextSpec.from_model(request.getfixturevalue(tower))
    a = _audit(spec, TA.eos_tokens(3))
    print("\n" + a.report())
    a.assert_ok()
    assert not any(a.completeness.values())
    assert len(a.src.stage_names()) == 1 + 8 * spec.layers and len(a.keys_seen) == 5 * spec.layers
    assert {f for f, _, _ in a.results} == {"embedding", "layernorm", "linear", "attention", "weight"}


def test_completeness_catches_an_extra_stage(gelu_tower):
    spec = TA.TextSpec.from_model(gelu_tower)
    src = LA.EmulatedSource(dict(tokens=TA.eos_tokens(2), out=None))
    with torch.no_grad():
        TA.TextAudit(src, spec, DT, emulate=True).run()
        src.order.append(f"{L0}.self_attn.some_new_layer")
        with pytest.raises(LA.AuditError, match="some_new_layer"):
            TA.TextAudit(src, spec, DT).run()


# ---------------------------------------------------------------------------------------------------------------------
# injected errors: each must fail on exactly the named layer / prepared weight
# ---------------------------------------------------------------------------------------------------------------------
def _attention(a, L, heads, mask_diag=1, v_roll=0):
    """Layer L's attention over the stages already built: keys j >= t + mask_diag masked; v_roll shifts V's heads."""
    x = a.S(L + ".self_attn.qk")
    B, _, ntok, C2 = x.shape
    C = C2 // 2
    qk = x.reshape(B, ntok, C2)
    v = a.read_v(L + ".self_attn.v_proj", ntok)
    v = torch.roll(v, -v_roll * (C // heads), dims=2)
    d = C // heads
    q, k = (t.reshape(B, ntok, heads, d).transpose(1, 2) for t in (qk[..., :C], qk[..., C:]))
    s = q @ k.transpose(-1, -2) / d ** 0.5
    s = s.masked_fill(torch.ones(ntok, ntok, dtype=torch.bool).triu(mask_diag), float("-inf"))
    o = (torch.softmax(s, -1) @ v.reshape(B, ntok, heads, d).transpose(1, 2)).transpose(1, 2).reshape(B, ntok, C)
    return kref.round16(o.permute(0, 2, 1).unsqueeze(2), DT)


def _linear(a, x_name, key, act=None, res=None):
    """round16 of a linear layer over stage x_name with the prepared weight `key` (NCHW), optional activation / residual."""
    x = a.S(x_name)
    w, b = a.conv_w(key, x.shape[3], 1)
    y = kref.conv64(x, w, b)
    if act is not None:
        y = act(y)
    if res is not None:
        y = y + a.S(res).permute(0, 3, 1, 2)
    return kref.round16(y, DT)


def test_position_row_off_by_one(gelu_tower):
    spec = TA.TextSpec.from_model(gelu_tower)
    name = T + ".embeddings"

    def hook(n, v, a):
        if n != name:
            return v
        ids = a.src.inputs["tokens"]
        pos = a.sd[T + ".embeddings.position_embedding.weight"]
        rows = torch.tensor([0] + list(range(ids.shape[1] - 1)))                      # t >= 1 reads row t - 1
        e = a.sd[T + ".embeddings.token_embedding.weight"][ids] + pos[rows]
        return e.to(DT).double().permute(0, 2, 1).unsqueeze(2)
    assert _failed(_audit(spec, TA.eos_tokens(2), stage_hook=hook)) == [name]


def test_causal_mask_admits_the_next_key(gelu_tower):
    spec = TA.TextSpec.from_model(gelu_tower)
    name = L1 + ".self_attn"
    hook = lambda n, v, a: _attention(a, L1, spec.heads, mask_diag=2) if n == name else v
    assert _failed(_audit(spec, TA.eos_tokens(2), stage_hook=hook)) == [name]


def test_q_and_k_rows_swapped(gelu_tower):
    spec = TA.TextSpec.from_model(gelu_tower)
    key = L0 + ".qk"

    def hook(k, w, b, a):
        if k != key:
            return w, b
        C = w.shape[1] // 2
        return torch.cat([w[:, C:], w[:, :C]], dim=1), torch.cat([b[C:], b[:C]])
    assert _failed(_audit(spec, TA.eos_tokens(2), weight_hook=hook)) == [key]


def test_v_proj_bias_dropped(gelu_tower):
    spec = TA.TextSpec.from_model(gelu_tower)
    key = L1 + ".self_attn.v_proj"
    hook = lambda k, w, b, a: (w, None) if k == key else (w, b)
    a = _audit(spec, TA.eos_tokens(2), weight_hook=hook)
    assert _failed(a) == [key]
    assert "bias present" in a.failures()[0][2].extra


def test_head_reads_the_next_heads_v(gelu_tower):
    spec = TA.TextSpec.from_model(gelu_tower)
    name = L0 + ".self_attn"
    hook = lambda n, v, a: _attention(a, L0, spec.heads, v_roll=1) if n == name else v
    assert _failed(_audit(spec, TA.eos_tokens(2), stage_hook=hook)) == [name]


def test_quick_gelu_in_one_fc1_of_a_gelu_tower(gelu_tower):
    spec = TA.TextSpec.from_model(gelu_tower)
    name = L1 + ".mlp.fc1"
    hook = lambda n, v, a: _linear(a, L1 + ".layer_norm2", name, act=kref.quick_gelu64) if n == name else v
    assert _failed(_audit(spec, TA.eos_tokens(2), stage_hook=hook)) == [name]


def test_fc2_without_its_residual(quick_tower):
    spec = TA.TextSpec.from_model(quick_tower)
    name = f"{T}.encoder.layers.2.mlp.fc2"
    hook = lambda n, v, a: _linear(a, f"{T}.encoder.layers.2.mlp.fc1", name) if n == name else v
    assert _failed(_audit(spec, TA.eos_tokens(2), stage_hook=hook)) == [name]


def test_layer_norm_with_the_wrong_epsilon(gelu_tower):
    """Token (0, 3): its token and position rows scaled down 1000x, so its embedding's variance (~1e-10) is where eps
    1e-6 instead of 1e-5 shows most (the other embeddings, of variance ~5e-4, move by about 1 %)."""
    spec = TA.TextSpec.from_model(gelu_tower)
    tokens = TA.eos_tokens(2)
    tok, pos = T + ".embeddings.token_embedding.weight", T + ".embeddings.position_embedding.weight"
    sd = dict(spec.sd)
    sd[tok], sd[pos] = sd[tok].clone(), sd[pos].clone()
    sd[tok][tokens[0, 3]] *= 1e-3
    sd[pos][3] *= 1e-3
    spec = TA.TextSpec(sd, spec.heads, spec.act, spec.eps)
    name = L0 + ".layer_norm1"

    def hook(n, v, a):
        if n != name:
            return v
        ref, _ = kref.layer_norm64(a.S(T + ".embeddings"), a.P(n + ".weight"), a.P(n + ".bias"), 1e-6, DT)
        return kref.round16(ref.permute(0, 3, 1, 2), DT)
    assert _failed(_audit(spec, tokens, stage_hook=hook)) == [name]


def test_final_layer_norm_skipped(gelu_tower):
    spec = TA.TextSpec.from_model(gelu_tower)
    name = T + ".final_layer_norm"
    hook = lambda n, v, a: a.src.stages[L1 + ".mlp.fc2"] if n == name else v
    assert _failed(_audit(spec, TA.eos_tokens(2), stage_hook=hook)) == [name]


# ---------------------------------------------------------------------------------------------------------------------
# host-side guards
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(2, 20), (2, 78), (77,), (2, 77, 1)])
def test_token_check_rejects_other_shapes(shape):
    import i2it
    with pytest.raises(ValueError, match="must be"):
        i2it.check_tokens(torch.zeros(shape, dtype=torch.long), 49408, 77)


@pytest.mark.parametrize("bad", [-1, 49408])
def test_token_check_rejects_ids_outside_the_table(bad):
    import i2it
    t = TA.eos_tokens(2)
    t[1, 5] = bad
    with pytest.raises(ValueError, match=r"\[0, 49408\)"):
        i2it.check_tokens(t, 49408, 77)


def test_token_check_accepts_both_ends_of_the_table():
    import i2it
    t = TA.eos_tokens(2)
    t[0, 1], t[1, 1] = 0, 49407
    i2it.check_tokens(t, 49408, 77)
    i2it.check_tokens(t.to(torch.int32), 49408, 77)
    with pytest.raises(ValueError, match="integer"):
        i2it.check_tokens(t.float(), 49408, 77)


def test_text_encoder_spec_requires_the_engines_epsilon():
    """The engine's LayerNorm launches use eps 1e-5: a tower configured otherwise stays on the torch module."""
    from _host import TurboBase
    spec = lambda eps: TurboBase._text_encoder_spec(SimpleNamespace(text_encoder=TA.clip_model(128, 1, 2, 256, eps=eps)))
    assert spec(1e-5) == {"heads": 2, "act": "gelu", "hidden": 128}
    assert spec(1e-6) is None
