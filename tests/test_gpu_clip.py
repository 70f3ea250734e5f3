"""-m gpu: the CLIP text tower on the engine (SURVEY.md section 8f #1) against transformers' CLIPTextModel — the one row whose
oracle IS the reference's own dependency (transformers is importable here), so this parity is pinned: same random-init tensors,
fp32 reference, engine in fp16 / bf16.  `text_encoder(tokens)[0]` is what src/pix2pix_turbo.py:190-196 feeds the
UNet."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _tokens(B, vocab=49408, seed=0):
    g = torch.Generator().manual_seed(seed)
    rows = []
    for b in range(B):
        n = 5 + 9 * b
        ids = [49406] + torch.randint(1, 49000, (n,), generator=g).tolist() + [49407]
        rows.append(ids + [49407] * (77 - len(ids)))               # CLIP pads with EOS
    return torch.tensor(rows, dtype=torch.long)


def _model(hidden, layers, heads, inter, act="gelu", seed=0):
    from transformers import CLIPTextConfig, CLIPTextModel
    cfg = CLIPTextConfig(vocab_size=49408, hidden_size=hidden, intermediate_size=inter, num_hidden_layers=layers,
                         num_attention_heads=heads, max_position_embeddings=77, hidden_act=act)
    torch.manual_seed(seed)
    m = CLIPTextModel(cfg).eval()
    with torch.no_grad():       # default init leaves every LayerNorm at (1, 0) and biases at 0: perturb so they are exercised
        for n, p in m.named_parameters():
            if n.endswith(".bias"):
                p.normal_(0, 0.02)
            elif "layer_norm" in n and n.endswith(".weight"):
                p.normal_(1.0, 0.1)
    return m


def _check(tag, got, ref, rel_bound):
    got, ref = got.float().cpu(), ref.float().cpu()
    assert got.shape == ref.shape and torch.isfinite(got).all()
    err = (got - ref).abs()
    rel = err.mean().item() / (ref.abs().mean().item() + 1e-12)
    band = (err <= 1e-4 + 1e-3 * ref.abs()).float().mean().item()
    print(f"[{tag}] mean|err|={err.mean().item():.3e} ({rel:.2%} of mean|ref|) max={err.max().item():.3e}; in north-star band: {band:.1%}")
    assert rel < rel_bound, (tag, rel)


@pytest.mark.parametrize("dt,bound", [(torch.float16, 4e-3), (torch.bfloat16, 3e-2)])
@pytest.mark.parametrize("shape", ["small", "small_quick", "sd_turbo"])
def test_clip_text_tower_vs_transformers(shape, dt, bound):
    import i2it
    hidden, layers, heads, inter, act = {"small": (128, 2, 2, 256, "gelu"), "small_quick": (192, 3, 3, 512, "quick_gelu"),
                                         "sd_turbo": (1024, 23, 16, 4096, "gelu")}[shape]
    m = _model(hidden, layers, heads, inter, act)
    tok = _tokens(3)
    with torch.no_grad():
        ref = m(tok)[0]                                            # fp32, CPU
    e = i2it.Engine(dt, i2it.PIX2PIX, text_heads=heads, text_act=act)
    e.load_state_dict({"text_encoder." + k: v for k, v in m.state_dict().items()})
    e.finalize(1.0, 1.0, 1.0, -1.0)
    got = e.encode_text(tok, hidden)
    torch.cuda.synchronize()
    _check(f"clip_{shape}_{'fp16' if dt == torch.float16 else 'bf16'}", got, ref, bound * (3 if shape == "sd_turbo" else 1))
    # causality: changing a later token must not change earlier positions (bit for bit)
    tok2 = tok.clone()
    tok2[:, 40:] = 1234
    got2 = e.encode_text(tok2, hidden)
    assert torch.equal(got[:, :40], got2[:, :40]) and not torch.equal(got[:, 40:], got2[:, 40:])
    # batch invariance: a prompt encoded alone == the same prompt inside a batch
    one = e.encode_text(tok[1:2], hidden)
    assert torch.equal(one[0], got[1])
    assert e.prep_launch_count() <= 4


def test_public_api_encodes_prompts_on_the_engine():
    """Pix2Pix_Turbo._encode_text (what forward() calls for `prompt=`) runs the tower through libi2it and matches the wrapped
    transformers module in fp32; the torch module is not called on this path."""
    import weights as W
    from pix2pix_turbo import Pix2Pix_Turbo
    m = Pix2Pix_Turbo(cfg=W.TINY, perturb_norm=True)                # TINY: cross_dim 128 -> a 2-layer, 2-head CLIP stand-in
    m.set_eval(); m.half()
    calls = []
    m.text_encoder.register_forward_hook(lambda *a: calls.append(1))
    emb = m._encode_text("a photo of a bird")
    assert m._text_on_engine and not calls and emb.shape == (1, 77, 128) and emb.dtype == torch.float16
    tokens = m.tokenizer("a photo of a bird", max_length=77, padding="max_length", truncation=True, return_tensors="pt").input_ids
    with torch.no_grad():
        ref = m.text_encoder.float().cpu()(tokens)[0]
    calls.clear()                                                  # (that was this test calling the torch module)
    _check("clip_public_api_fp16", emb, ref, 4e-3)
    x = (torch.rand(1, 1, 64, 64) < 0.08).float().expand(-1, 3, -1, -1).contiguous()
    y = m(x.cuda().half(), "a photo of a bird")
    assert torch.isfinite(y.float()).all() and not calls
