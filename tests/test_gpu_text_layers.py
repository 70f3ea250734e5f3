"""-m gpu: the teacher-forced audit of the CLIP text tower (tests/text_audit.py) on the engine.

Each case encodes tokens with keep_stages = 2, asserts that the audit covers every kept text stage and every
text_encoder.* prepared weight, holds every layer (on the engine's own inputs and prepared operands) to its float64 bound
and every prepared weight to bit equality, and checks that the output is bit-identical to a keep_stages = 0 engine on the
same tokens.  The float64 references run on the GPU.  Each case prints the worst err/bound and mean-ulp per layer family."""
import time

import pytest
import torch

import layer_audit as LA
import text_audit as TA

pytestmark = pytest.mark.gpu

bf, hf = torch.bfloat16, torch.float16
SHAPES = {"small": (128, 2, 2, 256, "gelu"), "small_quick": (192, 3, 3, 512, "quick_gelu"), "sd_turbo": (1024, 23, 16, 4096, "gelu")}


def _engine(spec, dt, keep):
    import i2it
    e = i2it.Engine(dt, i2it.PIX2PIX, keep_stages=keep, text_heads=spec.heads, text_act=spec.act)
    e.load_state_dict(spec.sd)
    e.finalize(1.0, 1.0, 1.0, -1.0)
    return e


def _encode_keep0(spec, dt, tokens):
    e = _engine(spec, dt, 0)
    out = e.encode_text(tokens, spec.sd[TA.T + ".embeddings.token_embedding.weight"].shape[1])
    torch.cuda.synchronize()
    e.close()
    return out


def audit_text(tag, e, spec, dt, tokens, out):
    src = TA.TextEngineSource(e, dict(tokens=tokens.cuda(), out=out))
    with torch.no_grad():
        a = TA.TextAudit(src, spec, dt).run()
    print(f"\n[{tag}] {len(a.results)} checks, {len(src.stage_names())} stages, {len(a.keys_seen)} prepared weights\n" + a.report())
    a.assert_ok()
    assert len(src.stage_names()) == 1 + 8 * spec.layers and len(a.keys_seen) == 5 * spec.layers
    return a


def run_case(tag, spec, dt, tokens):
    t0 = time.time()
    hidden = spec.sd[TA.T + ".embeddings.token_embedding.weight"].shape[1]
    e = _engine(spec, dt, 2)
    out = e.encode_text(tokens, hidden)
    torch.cuda.synchronize()
    audit_text(tag, e, spec, dt, tokens, out)
    e.close()
    assert torch.equal(out, _encode_keep0(spec, dt, tokens)), f"{tag}: keep_stages = 2 changed the encoded text"
    print(f"[{tag}] wall {time.time() - t0:.1f} s")


@pytest.fixture(scope="module")
def sd_turbo_tower():
    return TA.clip_model(*SHAPES["sd_turbo"])


@pytest.mark.parametrize("dt", [hf, bf], ids=["fp16", "bf16"])
@pytest.mark.parametrize("shape", ["small", "small_quick", "sd_turbo"])
def test_tower_shapes(shape, dt, request):
    m = request.getfixturevalue("sd_turbo_tower") if shape == "sd_turbo" else TA.clip_model(*SHAPES[shape])
    run_case(f"{shape} {dt}", TA.TextSpec.from_model(m), dt, TA.eos_tokens(3))


def test_sd_turbo_bf16_batch16_pads_and_table_ends(sd_turbo_tower):
    """1232 rows: EOS-padded rows, rows padded with id 0 (SD-2's "!" pad), one full 77-token row, and ids 0 and 49407."""
    g = torch.Generator().manual_seed(5)
    full = torch.tensor([[49406] + torch.randint(1, 49000, (75,), generator=g).tolist() + [49407]])
    ends = TA.eos_tokens(1, seed=6)
    ends[0, 1], ends[0, 2] = 0, 49407
    tokens = torch.cat([TA.eos_tokens(8, seed=3), TA.eos_tokens(6, seed=4, pad=0), full, ends])
    assert tokens.shape == (16, 77) and int(tokens.min()) == 0 and int(tokens.max()) == 49407
    run_case("sd_turbo bf16 B=16", TA.TextSpec.from_model(sd_turbo_tower), bf, tokens)


def test_sd_turbo_fp16_large_offset_channels():
    """Trained CLIP towers carry a few residual channels with large offsets and a large position-0 row: the LayerNorm
    cancellation term and the fp16 range both see them here."""
    m = TA.clip_model(*SHAPES["sd_turbo"], seed=7)
    with torch.no_grad():
        emb = m.text_model.embeddings
        chans = torch.tensor([3, 100, 257, 511, 640, 777, 900, 1023])
        emb.token_embedding.weight[:, chans] += torch.tensor([20.0, -35.0, 50.0, 12.0, -60.0, 28.0, 44.0, -18.0])
        emb.position_embedding.weight[0] *= 40.0
    tokens = TA.eos_tokens(3, seed=8)
    with torch.no_grad():
        ref = m.double()(tokens)[0]
        m.float()
    assert torch.isfinite(ref).all() and ref.abs().max() < 6e4
    run_case("sd_turbo fp16 offsets", TA.TextSpec.from_model(m), hf, tokens)


def _public_path(tag, cfg, dt, enc, H, W):
    """Pix2Pix_Turbo(keep_stages=2) called as a user calls it: the text plan and the forward audited on the one handle, and
    together they cover every prepared weight."""
    from _host import HashTokenizer
    from pix2pix_turbo import Pix2Pix_Turbo
    t0 = time.time()
    prompt = "a photo of a bird on a branch"
    m = Pix2Pix_Turbo(cfg=cfg, perturb_norm=True, keep_stages=2, text_stack=(HashTokenizer(), enc))
    m.set_eval()
    m.to(dt)
    g = torch.Generator().manual_seed(1)
    x = ((torch.rand(1, 1, H, W, generator=g) < 0.08).float().expand(-1, 3, -1, -1) * 2 - 1).to(dt).cuda().contiguous()
    eps = torch.randn(1, 4, H // 8, W // 8, generator=g).to(dt).cuda()
    y = m(x, prompt, eps=eps)
    torch.cuda.synchronize()
    e, emb = m._engine, m._encode_text(prompt)              # the cached embedding the forward used (no second encode)
    assert m._text_on_engine
    tokens = m.tokenizer(prompt, max_length=77, padding="max_length", truncation=True, return_tensors="pt").input_ids
    tspec = TA.TextSpec.from_model(enc)
    ta = audit_text(f"{tag} text", e, tspec, dt, tokens, emb)
    spec = LA.Spec(m._sd, cfg, "pix2pix", adapter_scales=dict(m._adapter_scales))
    src = LA.EngineSource(e, dict(x=x, text=emb, eps=eps, noise=None, image=y))
    with torch.no_grad():
        ia = LA.Audit(src, spec, dt).run()
    print(f"\n[{tag} forward] {len(ia.results)} checks, {len(src.stage_names())} stages, {len(ia.keys_seen)} prepared weights\n"
          + ia.report())
    ia.assert_ok()
    keys = set(e.prepared_keys())
    assert set(ta.keys_seen) | set(ia.keys_seen) == keys and not set(ta.keys_seen) & set(ia.keys_seen)
    assert any(k.startswith("text_encoder.") for k in keys)
    assert torch.equal(emb, _encode_keep0(tspec, dt, tokens)), f"{tag}: keep_stages = 2 changed the encoded text"
    print(f"[{tag}] {len(keys)} prepared weights on the handle; wall {time.time() - t0:.1f} s")
    return m, x, eps, y, emb


def test_public_path_one_handle_tiny():
    import weights as Wt
    from _host import HashTokenizer
    from pix2pix_turbo import Pix2Pix_Turbo
    enc = TA.clip_model(128, 2, 2, 256)                        # TINY cross_dim 128
    m, x, eps, y, emb = _public_path("public tiny fp16", Wt.TINY, hf, enc, 64, 64)
    del m
    m0 = Pix2Pix_Turbo(cfg=Wt.TINY, perturb_norm=True, text_stack=(HashTokenizer(), enc))
    m0.set_eval()
    m0.to(hf)
    y0 = m0(x, "a photo of a bird on a branch", eps=eps)
    assert torch.equal(m0._encode_text("a photo of a bird on a branch"), emb) and torch.equal(y0, y)


def test_public_path_one_handle_sd_turbo_256(sd_turbo_tower):
    import weights as Wt
    _public_path("public sd_turbo 256 bf16", Wt.SD_TURBO, bf, sd_turbo_tower, 256, 256)


def test_bad_tokens_raise_before_any_launch():
    import i2it
    spec = TA.TextSpec.from_model(TA.clip_model(*SHAPES["small"]))
    e = _engine(spec, bf, 2)
    bad_id = TA.eos_tokens(2)
    bad_id[1, 4] = 49408
    for t in (TA.eos_tokens(2)[:, :20], torch.cat([TA.eos_tokens(2), TA.eos_tokens(2)[:, :1]], 1), bad_id):
        with pytest.raises(ValueError):
            e.encode_text(t, 128)
    with pytest.raises(ValueError):
        e.encode_text(TA.eos_tokens(2), 64)                    # output narrower than the tower
    with pytest.raises(RuntimeError, match="no encode_text has run yet"):
        e.text_stage_names()                                   # no text plan was built: nothing reached the engine
    out = e.encode_text(TA.eos_tokens(2), 128)
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all() and len(e.text_stage_names()) == 1 + 8 * spec.layers
