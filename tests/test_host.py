"""CPU tests of the host side: C-ABI library loads and exports every declared symbol (no compute calls), the mirrors of the
reference API keep its names / signatures / error behaviour, checkpoint formats round-trip, sharding logic (gloo, world 2)."""
import inspect
import os
import re
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _text_stack():
    class Tok:
        model_max_length = 77

        def __call__(self, text, **kw):
            from types import SimpleNamespace
            n = 1 if isinstance(text, str) else len(text)
            return SimpleNamespace(input_ids=torch.zeros(n, 77, dtype=torch.long))
    return Tok(), None


def test_library_exports_every_declared_symbol():
    import i2it
    hdr = open(os.path.join(ROOT, "include", "i2it.h")).read()
    declared = set(re.findall(r"\b(i2it_[a-z0-9_]+)\s*\(", hdr))
    assert declared == set(i2it.SYMBOLS), declared ^ set(i2it.SYMBOLS)
    lib = i2it.load_library()
    for s in declared:
        assert getattr(lib, s) is not None
    out = subprocess.run(["nm", "-D", "--defined-only", i2it.LIB_PATH], capture_output=True, text=True).stdout
    for s in declared:
        assert re.search(rf"\bT {s}\b", out), f"{s} not exported"


def test_default_config_matches_sd_turbo():
    import ctypes as C
    import i2it
    import weights as W
    lib = i2it.load_library()
    c = i2it.Config()
    assert lib.i2it_default_config(C.byref(c)) == 0
    assert tuple(c.unet_channels) == W.SD_TURBO["unet_channels"] and tuple(c.unet_heads) == W.SD_TURBO["unet_heads"]
    assert tuple(c.vae_channels) == W.SD_TURBO["vae_channels"] and c.cross_dim == 1024 and c.temb_dim == 1280
    assert abs(c.scaling_factor - 0.18215) < 1e-7


def test_no_gpu_fails_loudly():
    import i2it
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        i2it.Engine(torch.bfloat16)


def test_pix2pix_signature_matches_reference():
    from pix2pix_turbo import Pix2Pix_Turbo, TwinConv
    sig = inspect.signature(Pix2Pix_Turbo.__init__)
    names = list(sig.parameters)[1:6]
    assert names == ["pretrained_name", "pretrained_path", "ckpt_folder", "lora_rank_unet", "lora_rank_vae"]   # ref :30
    assert [sig.parameters[n].default for n in names] == [None, None, "checkpoints", 8, 4]
    f = inspect.signature(Pix2Pix_Turbo.forward)
    assert list(f.parameters)[1:7] == ["c_t", "prompt", "prompt_tokens", "deterministic", "r", "noise_map"]       # ref :186
    assert f.parameters["deterministic"].default is True and f.parameters["r"].default == 1.0
    for m in ("set_eval", "set_train", "save_model"):
        assert hasattr(Pix2Pix_Turbo, m)
    assert list(inspect.signature(TwinConv.__init__).parameters)[1:] == ["convin_pretrained", "convin_curr"]


def test_cyclegan_signature_matches_reference():
    from cyclegan_turbo import CycleGAN_Turbo, VAE_decode, VAE_encode
    sig = inspect.signature(CycleGAN_Turbo.__init__)
    assert list(sig.parameters)[1:6] == ["pretrained_name", "pretrained_path", "ckpt_folder", "lora_rank_unet", "lora_rank_vae"]
    f = inspect.signature(CycleGAN_Turbo.forward)
    assert list(f.parameters)[1:5] == ["x_t", "direction", "caption", "caption_emb"]                              # ref :241
    fw = inspect.signature(CycleGAN_Turbo.forward_with_networks)
    assert list(fw.parameters)[:8] == ["x", "direction", "vae_enc", "unet", "vae_dec", "sched", "timesteps", "text_emb"]
    assert hasattr(CycleGAN_Turbo, "get_traininable_params")
    for cls in (VAE_encode, VAE_decode):
        assert list(inspect.signature(cls.__init__).parameters)[1:3] == ["vae", "vae_b2a"]


def test_pix2pix_host_behaviour(tmp_path):
    import weights as W
    from pix2pix_turbo import Pix2Pix_Turbo
    m = Pix2Pix_Turbo(cfg=W.TINY, text_stack=_text_stack())
    assert m.timesteps.tolist() == [999] and m.vae.decoder.gamma == 1
    assert abs(float(m.sched.alphas_cumprod[999]) - 0.0046600951) < 1e-9
    m.set_eval()
    assert m.half() is m and m.compute_dtype == torch.float16
    m.unet.enable_xformers_memory_efficient_attention()                    # must exist (inference_unpaired.py:36)
    with pytest.raises(AssertionError, match="Either prompt or prompt_tokens"):   # reference :188
        m(torch.zeros(1, 3, 64, 64))
    with pytest.raises(AssertionError):
        m(torch.zeros(1, 3, 64, 64), prompt="a", prompt_tokens=torch.zeros(1, 77, dtype=torch.long))
    # checkpoint format of save_model (reference :221-229) round-trips through pretrained_path (reference :111-125)
    p = str(tmp_path / "m.pkl")
    m.save_model(p)
    sd = torch.load(p)
    assert set(sd) == {"unet_lora_target_modules", "vae_lora_target_modules", "rank_unet", "rank_vae", "state_dict_unet",
                       "state_dict_vae"}
    assert all(("lora" in k or "conv_in" in k) for k in sd["state_dict_unet"])
    assert all(("lora" in k or "skip" in k) for k in sd["state_dict_vae"])
    key = next(k for k in sd["state_dict_unet"] if "lora_B" in k)
    sd["state_dict_unet"][key] = sd["state_dict_unet"][key] + 1.0
    torch.save(sd, p)
    with pytest.warns(UserWarning):
        m2 = Pix2Pix_Turbo(pretrained_path=p, cfg=W.TINY, text_stack=_text_stack())
    assert torch.equal(m2.unet.state_dict()[key], sd["state_dict_unet"][key])


def test_cyclegan_host_behaviour():
    import weights as W
    from cyclegan_turbo import CycleGAN_Turbo
    m = CycleGAN_Turbo(cfg=W.TINY, text_stack=_text_stack())
    with pytest.raises(AssertionError):                                    # reference :243: direction must be known
        m(torch.zeros(1, 3, 64, 64))
    m.direction, m.caption = "a2b", None
    with pytest.raises(AssertionError):                                    # reference :246: caption must be known
        m(torch.zeros(1, 3, 64, 64))
    with pytest.raises(AssertionError):                                    # reference :202
        CycleGAN_Turbo.forward_with_networks(torch.zeros(1, 3, 64, 64), "sideways", m.vae_enc, m.unet, m.vae_dec, m.sched,
                                             m.timesteps, torch.zeros(1, 77, 128))
    assert m.eval() is m
    # every UNet LoRA layer belongs to exactly one of the three adapters (cyclegan_turbo.py:53-72)
    ads = {k.split(".lora_A.")[1].split(".")[0] for k in m._sd if k.startswith("unet.") and ".lora_A." in k}
    assert ads == {"default_encoder", "default_decoder", "default_others"}
    assert any(k.startswith("vae_b2a.") for k in m._sd)


def test_cyclegan_checkpoint_format(tmp_path):
    """The .pkl written by train_cyclegan_turbo.py:293-307 (read at cyclegan_turbo.py:162-190): three UNet adapter dicts with
    adapter-less peft keys, two VAE dicts whose keys carry the vae./vae_b2a. prefix, peft 'base_layer.' variants."""
    import weights as W
    from cyclegan_turbo import CycleGAN_Turbo
    m = CycleGAN_Turbo(cfg=W.TINY, text_stack=_text_stack(), synthetic_caption="c", synthetic_direction="a2b")
    enc_key = next(k for k in m._sd if k.startswith("unet.") and ".lora_B.default_encoder." in k)
    dec_key = next(k for k in m._sd if k.startswith("unet.") and ".lora_B.default_decoder." in k)
    oth_key = next(k for k in m._sd if k.startswith("unet.") and ".lora_B.default_others." in k)
    strip = lambda k, a: k[len("unet."):].replace(f".lora_B.{a}.", ".lora_B.")
    skip_key = next(k for k in m._sd if k.startswith("vae.") and "skip_conv_1" in k)
    conv_key = next(k for k in m._sd if k.startswith("vae_b2a.") and k.endswith("conv_in.weight"))
    ck = {"rank_unet": 8, "rank_vae": 4,
          "sd_encoder": {strip(enc_key, "default_encoder"): torch.full_like(m._sd[enc_key], 1.5)},
          "sd_decoder": {strip(dec_key, "default_decoder"): torch.full_like(m._sd[dec_key], 2.5)},
          "sd_other": {strip(oth_key, "default_others"): torch.full_like(m._sd[oth_key], 3.5)},
          "sd_vae_enc": {conv_key.replace("conv_in.weight", "conv_in.base_layer.weight"): torch.full_like(m._sd[conv_key], 4.5)},
          "sd_vae_dec": {skip_key: torch.full_like(m._sd[skip_key], 5.5)}}
    p = str(tmp_path / "cyc.pkl")
    torch.save(ck, p)
    with pytest.warns(UserWarning):                    # no SD-Turbo base offline: checkpoint tensors over a seeded base
        m2 = CycleGAN_Turbo(pretrained_path=p, cfg=W.TINY, text_stack=_text_stack())
    for k, v in ((enc_key, 1.5), (dec_key, 2.5), (oth_key, 3.5), (conv_key, 4.5), (skip_key, 5.5)):
        assert torch.all(m2._sd[k] == v), k
    with pytest.raises(ValueError):
        CycleGAN_Turbo(pretrained_name="no_such_model", cfg=W.TINY, text_stack=_text_stack())


def test_sd_turbo_snapshot_overlay(tmp_path, monkeypatch):
    """Real base weights come from a local snapshot ($I2IT_SD_TURBO_DIR/{unet,vae}/diffusion_pytorch_model.safetensors);
    pre-0.14 VAE attention key names (query/key/value/proj_attn) are mapped to to_q/to_k/to_v/to_out.0."""
    from safetensors.torch import save_file
    import _host
    (tmp_path / "unet").mkdir()
    (tmp_path / "vae").mkdir()
    save_file({"conv_in.weight": torch.full((2, 2), 7.0, dtype=torch.float16)},
              str(tmp_path / "unet" / "diffusion_pytorch_model.safetensors"))
    save_file({"encoder.mid_block.attentions.0.query.weight": torch.full((2, 2), 1.0),
               "encoder.mid_block.attentions.0.proj_attn.bias": torch.full((2,), 2.0),
               "decoder.conv_out.bias": torch.full((3,), 3.0)},
              str(tmp_path / "vae" / "diffusion_pytorch_model.safetensors"))
    sd = {}
    monkeypatch.delenv(_host.SD_TURBO_DIR_ENV, raising=False)
    assert _host.load_sd_turbo_base(sd, ["unet", "vae"]) is False and sd == {}
    monkeypatch.setenv(_host.SD_TURBO_DIR_ENV, str(tmp_path))
    assert _host.load_sd_turbo_base(sd, ["unet", "vae", "vae_b2a"]) is True
    assert sd["unet.conv_in.weight"].dtype == torch.float32 and float(sd["unet.conv_in.weight"][0, 0]) == 7.0
    for pre in ("vae.", "vae_b2a."):                   # both CycleGAN VAEs start from the same SD-Turbo VAE (cyclegan_turbo.py:80)
        assert float(sd[pre + "encoder.mid_block.attentions.0.to_q.weight"][0, 0]) == 1.0
        assert float(sd[pre + "encoder.mid_block.attentions.0.to_out.0.bias"][0]) == 2.0
        assert float(sd[pre + "decoder.conv_out.bias"][0]) == 3.0
    os.remove(str(tmp_path / "vae" / "diffusion_pytorch_model.safetensors"))
    assert _host.load_sd_turbo_base({}, ["unet", "vae"]) is False      # partial snapshot is reported, not silently accepted


def test_shard_ranges():
    from dist import shard_range
    for B in (1, 7, 8, 64, 128):
        for world in (1, 2, 3, 8):
            rs = [shard_range(B, r, world) for r in range(world)]
            assert rs[0][0] == 0 and rs[-1][1] == B
            assert all(rs[i][1] == rs[i + 1][0] for i in range(world - 1))
            assert max(h - l for l, h in rs) - min(h - l for l, h in rs) <= 1


def test_sharded_allgather_gloo_world2(tmp_path):
    # N>1 path on CPU: two gloo ranks shard a batch, run a per-sample "model", all-gather -> identical to unsharded
    script = tmp_path / "w.py"
    script.write_text(f"""
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, {os.path.join(ROOT, 'img2img-turbo_b200')!r})
from dist import sharded_forward
dist.init_process_group('gloo')
B = 5
x = torch.arange(B * 3 * 4 * 4, dtype=torch.float32).view(B, 3, 4, 4)
eps = torch.arange(B * 2, dtype=torch.float32).view(B, 2)
model = lambda xs, prompt, eps=None: xs * 2 + eps.view(-1, 1, 1, 1)[:, :, :1, :1]
y = sharded_forward(model, x, 'p', eps=eps[:, :1])
ref = x * 2 + eps[:, :1].view(-1, 1, 1, 1)
assert torch.equal(y, ref), (y - ref).abs().max()
x8 = torch.randn(8, 3, 2, 2, generator=torch.Generator().manual_seed(0))
y8 = sharded_forward(lambda xs: xs + 1, x8)
assert torch.equal(y8, x8 + 1)
dist.destroy_process_group()
print('rank', os.environ['RANK'], 'ok')
""")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
                        "127.0.0.1", "--master-port", "29533", str(script)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert r.stdout.count("ok") == 2


def test_save_model_uses_peft_key_names_the_reference_loader_expects(tmp_path):
    """ADVICE r1: the reference copies the checkpoint keys into vae.state_dict()/unet.state_dict() of peft-wrapped models and
    loads STRICTLY (pix2pix_turbo.py:66-78): base weights of LoRA-wrapped layers must be spelled `X.base_layer.weight`."""
    import weights as W
    from pix2pix_turbo import Pix2Pix_Turbo
    m = Pix2Pix_Turbo(cfg=W.TINY, text_stack=_text_stack(), twin=True)
    p = str(tmp_path / "m.pkl")
    m.save_model(p)
    ck = torch.load(p)
    vae = ck["state_dict_vae"]
    for i in range(1, 5):                                               # skip convs are LoRA targets (pix2pix_turbo.py:143-147)
        assert f"decoder.skip_conv_{i}.base_layer.weight" in vae and f"decoder.skip_conv_{i}.weight" not in vae
        assert f"decoder.skip_conv_{i}.lora_A.vae_skip.weight" in vae
    for k in vae:                                                       # every wrapped layer's base tensors carry the infix
        if k.endswith((".weight", ".bias")) and ".lora_" not in k:
            assert ".base_layer." in k, k
    unet = ck["state_dict_unet"]
    # TwinConv conv_in is not a LoRA target: plain names (reference filter `"conv_in" in k`)
    assert "conv_in.conv_in_pretrained.weight" in unet and "conv_in.conv_in_curr.bias" in unet
    assert all(("lora" in k) or ("conv_in" in k) for k in unet)
    # and our own loader reads that spelling back
    with pytest.warns(UserWarning):
        m2 = Pix2Pix_Turbo(pretrained_path=p, cfg=W.TINY, text_stack=_text_stack())
    assert m2._twin and torch.equal(m2._sd["vae.decoder.skip_conv_1.weight"], m._sd["vae.decoder.skip_conv_1.weight"])


def test_checkpoint_decides_which_layers_get_adapters(tmp_path):
    """ADVICE r1: adapters exist only where the checkpoint has them; no layer keeps a seeded random adapter."""
    import weights as W
    from pix2pix_turbo import Pix2Pix_Turbo
    m = Pix2Pix_Turbo(cfg=W.TINY, text_stack=_text_stack())
    p = str(tmp_path / "m.pkl")
    m.save_model(p)
    ck = torch.load(p)
    lora = [k for k in ck["state_dict_unet"] if "lora" in k]
    keep = set(lora[:6])
    ck["state_dict_unet"] = {k: v for k, v in ck["state_dict_unet"].items() if k in keep or "lora" not in k}
    ck["unet_lora_target_modules"] = ["to_q"]
    torch.save(ck, p)
    with pytest.warns(UserWarning):
        m2 = Pix2Pix_Turbo(pretrained_path=p, cfg=W.TINY, text_stack=_text_stack())
    got = {k for k in m2._sd if k.startswith("unet.") and ".lora_" in k}
    assert got == {"unet." + k for k in keep}
    assert m2.target_modules_unet == ["to_q"]


def test_named_cyclegan_model_does_not_run_on_random_weights(tmp_path, monkeypatch):
    """ADVICE r1: a named pretrained model whose checkpoint cannot be loaded raises (as Pix2Pix_Turbo does) unless the caller
    opts in; a partial download never poses as the checkpoint."""
    import weights as W
    import cyclegan_turbo as C
    import model as M

    def boom(url, outf):
        raise OSError("network unreachable")
    monkeypatch.setattr(C, "download_url", boom)
    with pytest.raises(RuntimeError, match="allow_synthetic_weights"):
        C.CycleGAN_Turbo(pretrained_name="day_to_night", cfg=W.TINY, text_stack=_text_stack(), ckpt_folder=str(tmp_path))
    with pytest.warns(UserWarning):
        m = C.CycleGAN_Turbo(pretrained_name="day_to_night", cfg=W.TINY, text_stack=_text_stack(), ckpt_folder=str(tmp_path),
                             allow_synthetic_weights=True)
    assert m.caption == "driving in the night" and m.direction == "a2b"
    # corrupt / truncated file on disk: torch.load fails -> raises too
    bad = tmp_path / "day2night.pkl"
    bad.write_bytes(b"not a pickle")
    monkeypatch.setattr(C, "download_url", M.download_url)               # "Skipping download": the file exists
    with pytest.raises(RuntimeError, match="allow_synthetic_weights"):
        C.CycleGAN_Turbo(pretrained_name="day_to_night", cfg=W.TINY, text_stack=_text_stack(), ckpt_folder=str(tmp_path))

    class Resp:
        def raise_for_status(self):
            pass

        def iter_content(self, n):
            yield b"abc"
            raise ConnectionError("dropped")
    import types
    monkeypatch.setitem(sys.modules, "requests", types.SimpleNamespace(get=lambda url, stream=True: Resp()))
    target = tmp_path / "x.pkl"
    with pytest.raises(ConnectionError):
        M.download_url("http://example.invalid/x.pkl", str(target))
    assert not target.exists()                                           # only a .part file is left behind


def test_fp32_model_warns_that_it_computes_in_bf16():
    import weights as W
    from pix2pix_turbo import Pix2Pix_Turbo
    m = Pix2Pix_Turbo(cfg=W.TINY, text_stack=_text_stack())
    with pytest.warns(UserWarning, match="bf16"):
        assert m.compute_dtype == torch.bfloat16
    m.half()
    assert m.compute_dtype == torch.float16


def test_tile_decode_magic_division_is_exact():
    """The GEMM kernels decode tile indices with host-made magic numbers (csrc/tapgemm.cuh: make_magic / fast_div: one 32-bit
    high multiply instead of an integer division).  Index arithmetic must be exact: every divisor the plans use (n-tiles, tile
    counts per dimension) against every dividend below the tile-space bound, through the library's own host function."""
    import random
    import i2it
    lib = i2it.load_library()
    rng = random.Random(0)
    # (max dividend, divisor): tile spaces of the path — 16384 m-tiles x 2 n-tiles (+ grid), token matrices of 32768 / 128 rows,
    # batch 128 sweeps, and adversarial divisors around powers of two
    cases = [(2 * 16384 + 2 + 148, d) for d in (1, 2, 3, 5, 7, 8, 9, 16, 31, 32, 33, 64, 74, 127, 128, 148, 160, 255, 256, 257, 4096)]
    cases += [(8 * 2 * 16384 + 150, d) for d in (2, 3, 6, 10, 100, 1000, 1023, 1025, 8191, 8193, 16384)]
    for maxd, d in cases:
        xs = {0, 1, d - 1, d, d + 1, maxd - 1, maxd // 2} | {rng.randrange(maxd) for _ in range(400)} | {k * d - 1 for k in range(1, 40)} | \
             {k * d for k in range(1, 40)}
        refused = d > 1 and maxd * d >= (1 << 32)          # the host raises for such a tile space instead of decoding wrongly
        for x in xs:
            if 0 <= x < maxd:
                assert lib.i2it_debug_fast_div(maxd, d, x) == (-1 if refused else x // d), (maxd, d, x)
    # exhaustive over a bound above any real launch's dividends (16384 m-tiles: tile index + grid)
    maxd = 2 * 16384 + 2 + 148
    for d in (2, 32, 128):
        assert all(lib.i2it_debug_fast_div(maxd, d, x) == x // d for x in range(maxd))
    # tile spaces too large for the 32-bit magic are refused (the host raises instead of decoding wrongly)
    assert lib.i2it_debug_fast_div(1 << 31, 3, 5) == -1
