"""-m gpu: the boundary around the fused path — scheduler-step rounding of the two wrappers, the prompt K/V cache, the uint8 HWC
boundary, the job-table weight preparation, checkpoints loaded through the engine.  Everything is called through the C ABI
(ctypes) or the reference-API mirrors; references are torch expressions on the same device / the CPU oracle."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def _inputs(kind, B, H, cfg, seed=1, W_=None):
    W_ = W_ or H
    g = torch.Generator().manual_seed(seed)
    if kind == "pix2pix":
        x = (torch.rand(B, 1, H, W_, generator=g) < 0.08).float().expand(-1, 3, -1, -1).contiguous()
    else:
        x = torch.rand(B, 3, H, W_, generator=g) * 2 - 1
    text = torch.randn(B, 77, cfg["cross_dim"], generator=g)
    eps = torch.randn(B, 4, H // 8, W_ // 8, generator=g)
    noise = torch.randn(B, 4, H // 8, W_ // 8, generator=g)
    return x, text, eps, noise


def _engine(kind, cfg, dt, sd, **kw):
    import i2it
    e = i2it.Engine(dt, i2it.CYCLEGAN if kind == "cyclegan" else i2it.PIX2PIX, cfg=cfg, **kw)
    e.load_state_dict(sd)
    if kind == "pix2pix":
        e.set_adapter_scale("default", 1.0)
        e.set_adapter_scale("vae_skip", 2.0)
    else:
        for a in ("default_encoder", "default_decoder", "default_others"):
            e.set_adapter_scale(a, 1.0)
        e.set_adapter_scale("vae_skip", 2.0)
    e.finalize(1.0, 1.0, 1.0, -1.0)
    return e


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("kind", ["cyclegan", "pix2pix"])
def test_ddpm_step_rounding_matches_torch_on_device(kind, dt):
    """x_denoised must equal, BIT FOR BIT, what the reference's scheduler call computes from the engine's own latent and model_pred:
    CycleGAN passes a 0-dim timestep (three activation-dtype roundings, src/cyclegan_turbo.py:205), Pix2Pix a 1-D timesteps tensor
    (fp32 promotion, one rounding, src/pix2pix_turbo.py:200-201).  The expressions below are diffusers' DDPMScheduler.step for
    t = 999 (prev alpha_bar = 1 -> prev_sample = pred_original_sample) evaluated by torch on the GPU with alphas_cumprod moved to
    the device exactly as make_1step_sched does (src/model.py:10)."""
    import weights as W
    from _host import OneStepDDPM
    cfg = W.TINY
    sd = W.make_state_dict(kind, cfg, seed=0, perturb_norm=True)
    e = _engine(kind, cfg, dt, sd, keep_stages=True)
    x, text, eps, _ = _inputs(kind, 2, 64, cfg)
    lat = torch.empty(2, 4, 8, 8, device="cuda", dtype=dt)
    e.forward(x.to(dt).cuda(), text.to(dt).cuda(), eps.to(dt).cuda(), out_latent=lat)
    torch.cuda.synchronize()
    sample = e.read_stage("latent")[:, :4].to(dt)            # stages are fp32 copies of 16-bit tensors: exact
    pred = e.read_stage("model_pred")[:, :4].to(dt)
    ac = OneStepDDPM().alphas_cumprod.cuda()
    timesteps = torch.tensor([999], device="cuda").long()
    t = timesteps[0] if kind == "cyclegan" else timesteps
    alpha_prod_t = ac[t]
    beta_prod_t = 1 - alpha_prod_t
    if kind == "cyclegan":
        ref = torch.stack([(sample[i] - beta_prod_t ** (0.5) * pred[i]) / alpha_prod_t ** (0.5) for i in range(2)])
        assert ref.dtype == dt
    else:
        ref = ((sample - beta_prod_t ** (0.5) * pred) / alpha_prod_t ** (0.5))
        assert ref.dtype == torch.float32
        ref = ref.to(dt)
    bad = (ref.view(torch.int16) != lat.view(torch.int16)).sum().item()
    assert bad == 0, f"{bad}/{ref.numel()} elements differ from torch's scheduler arithmetic; max diff {(ref.float() - lat.float()).abs().max().item()}"
    # and the decoder input is x_denoised / scaling_factor as torch divides a 16-bit tensor by a Python float
    dec_in = e.read_stage("dec_in")[:, :4].to(dt)
    assert torch.equal(dec_in, lat / cfg["scaling_factor"])


def test_text_cache_equals_inline_text():
    """i2it_set_text + text_emb=NULL is bit-identical to passing the embedding with every forward; a new prompt replaces it; the
    cache dies with i2it_finalize_weights."""
    import weights as W
    cfg, dt = W.TINY, torch.bfloat16
    sd = W.make_state_dict("pix2pix", cfg, seed=0, perturb_norm=True)
    e = _engine("pix2pix", cfg, dt, sd)
    x, text, eps, _ = _inputs("pix2pix", 2, 64, cfg)
    xd, ed = x.to(dt).cuda(), eps.to(dt).cuda()
    t1, t2 = text[:1].to(dt).cuda().contiguous(), (text[1:2] * 0.5).to(dt).cuda().contiguous()
    a = e.forward(xd, t1, ed).clone()
    n_inline = e.launch_count(2, 64, 64)
    e.set_text(t1)
    b = e.forward(xd, None, ed).clone()
    n_cached = e.launch_count(2, 64, 64)
    assert torch.equal(a, b)
    assert n_cached == n_inline - 33, (n_inline, n_cached)      # 16 x (to_k linear + V^T projection) + the text staging copy
    e.set_text(t2)
    c = e.forward(xd, None, ed).clone()
    assert torch.equal(c, e.forward(xd, t2, ed)) and not torch.equal(a, c)
    tb = torch.cat([t1, t2]).contiguous()                         # per-image prompts
    e.set_text(tb)
    d = e.forward(xd, None, ed).clone()
    assert torch.equal(d, e.forward(xd, tb, ed))
    e.finalize(0.5, 0.5, 1.0, -1.0)
    with pytest.raises(RuntimeError, match="i2it_set_text"):
        e._text_batch = 1
        e.forward(xd, None, ed)


def test_weight_prep_is_a_handful_of_launches():
    """Round 1 spent ~970 per-tensor launches per engine build; the job table folds every weight of a plan in one launch."""
    import weights as W
    cfg, dt = W.TINY, torch.bfloat16
    sd = W.make_state_dict("pix2pix", cfg, seed=0, perturb_norm=True)
    e = _engine("pix2pix", cfg, dt, sd)
    x, text, eps, _ = _inputs("pix2pix", 1, 64, cfg)
    e.forward(x.to(dt).cuda(), text[:1].to(dt).cuda(), eps.to(dt).cuda())
    torch.cuda.synchronize()
    assert 1 <= e.prep_launch_count() <= 5, e.prep_launch_count()
    e.forward(x.to(dt).cuda(), text[:1].to(dt).cuda(), eps.to(dt).cuda())
    assert e.prep_launch_count() <= 5                            # cached: a second forward prepares nothing


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_uint8_boundary_matches_host_pre_and_post_processing(dt):
    """The uint8 forward == torchvision-style host pre-processing -> i2it_forward -> ToPILImage()(out*0.5+0.5), bit for bit, for the
    three input transforms of the reference CLIs (src/inference_paired.py:50,56-57,72; src/inference_unpaired.py:45-47,53)."""
    import i2it
    import weights as W
    cfg = W.TINY
    sd = W.make_state_dict("pix2pix", cfg, seed=0, perturb_norm=True)
    e = _engine("pix2pix", cfg, dt, sd)
    g = torch.Generator().manual_seed(3)
    img = (torch.rand(2, 64, 128, 3, generator=g) * 255).to(torch.uint8)           # HWC uint8, H != W
    _, text, eps, _ = _inputs("pix2pix", 2, 64, cfg, W_=128)
    td, ed = text[:1].to(dt).cuda(), eps.to(dt).cuda()
    for mode in (i2it.IN_UNIT, i2it.IN_NORMALIZE, i2it.IN_SKETCH):
        t = img.permute(0, 3, 1, 2).to(torch.float32).div(255)                      # F.to_tensor
        if mode == i2it.IN_NORMALIZE:
            t = t.sub(0.5).div(0.5)                                                  # transforms.Normalize([0.5],[0.5])
        elif mode == i2it.IN_SKETCH:
            t = (t < 0.5).float()
        x = t.to(dt).cuda().contiguous()                                             # .half() / .to(dtype) of the CLI
        ref = e.forward(x, td, ed)
        pic = ref.cpu() * 0.5 + 0.5                                                  # output_image[0].cpu() * 0.5 + 0.5   (in dt)
        ref_u8 = pic.mul(255).byte().permute(0, 2, 3, 1).contiguous()                # ToPILImage: pic.mul(255).byte(), CHW -> HWC
        got = e.forward_u8(img.cuda(), mode, td, ed)
        torch.cuda.synchronize()
        assert got.dtype == torch.uint8 and got.shape == img.shape
        diff = (got.cpu().int() - ref_u8.int()).abs()
        assert diff.max().item() == 0, (mode, diff.max().item(), (diff > 0).float().mean().item())


def test_public_api_u8_and_checkpoint_through_engine(tmp_path):
    """save_model() -> pretrained_path -> engine: the loaded checkpoint (adapters only where the checkpoint has them, peft key
    spelling) reproduces the saving model's output bit for bit, and forward_u8 of the wrapper equals its own float path."""
    import oracle as O
    import weights as W
    from pix2pix_turbo import Pix2Pix_Turbo
    cfg = W.TINY
    m = Pix2Pix_Turbo(cfg=cfg, perturb_norm=True)
    m.set_eval(); m.half()
    x, _, eps, _ = _inputs("pix2pix", 2, 64, cfg)
    y = m(x.cuda().half(), "a bird", eps=eps)
    p = str(tmp_path / "ck.pkl")
    m.save_model(p)
    ck = torch.load(p)
    assert any(".base_layer." in k for k in ck["state_dict_vae"])                   # peft spelling of wrapped base weights
    with pytest.warns(UserWarning):
        m2 = Pix2Pix_Turbo(pretrained_path=p, cfg=cfg, perturb_norm=True)
    m2.set_eval(); m2.half()
    y2 = m2(x.cuda().half(), "a bird", eps=eps)
    assert torch.equal(y, y2)
    emb = m2._encode_text("a bird").float().cpu()
    ref = O.pix2pix_forward(m2._sd, x.half().float(), emb, eps.half().float(), cfg)
    assert (y2.float().cpu() - ref).abs().mean() < 5e-3
    # a checkpoint that covers only SOME layers: the others must run without any adapter (not with the seeded random one)
    keep = [k for k in ck["state_dict_unet"] if "lora" in k][:8]
    ck["state_dict_unet"] = {k: v for k, v in ck["state_dict_unet"].items() if k in keep or "lora" not in k}
    torch.save(ck, p)
    with pytest.warns(UserWarning):
        m3 = Pix2Pix_Turbo(pretrained_path=p, cfg=cfg, perturb_norm=True)
    m3.set_eval(); m3.half()
    y3 = m3(x.cuda().half(), "a bird", eps=eps)
    ref3 = O.pix2pix_forward(m3._sd, x.half().float(), emb, eps.half().float(), cfg)
    assert sum(1 for k in m3._sd if k.startswith("unet.") and ".lora_A." in k) == len(keep) // 2 == 4
    assert (y3.float().cpu() - ref3).abs().mean() < 5e-3 and not torch.equal(y3, y2)
    # wrapper-level uint8 boundary
    img = (x.permute(0, 2, 3, 1) * 255).to(torch.uint8).contiguous()
    u = m2.forward_u8(img, "a bird", eps=eps)
    yf = m2(img.permute(0, 3, 1, 2).float().div(255).half().cuda(), "a bird", eps=eps)
    ref_u8 = (yf.cpu() * 0.5 + 0.5).mul(255).byte().permute(0, 2, 3, 1)
    assert torch.equal(u.cpu(), ref_u8)


def test_two_rank_sharded_output_equals_single_rank(tmp_path):
    """N-rank sharded forward == 1-rank forward, bit for bit (needs 2 GPUs; skipped on a single-GPU host)."""
    import subprocess
    import sys
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", "29541", os.path.join(root, "tests", "gpu_two_rank.py")], capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.count("TWO_RANK_OK") == 2
