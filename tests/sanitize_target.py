"""compute-sanitizer target: one tiny forward of the hot path through the C ABI, eager launches (no CUDA graph), the GEMM kernel,
flash attention, GroupNorm / LayerNorm, the uint8 boundary and the prompt K/V cache.
    compute-sanitizer --tool memcheck  python tests/sanitize_target.py
    compute-sanitizer --tool racecheck python tests/sanitize_target.py"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "img2img-turbo_b200"))
import i2it  # noqa: E402
import weights as W  # noqa: E402

cfg, dt = W.TINY, torch.bfloat16
B, H = (2, 128) if len(sys.argv) < 2 else (int(sys.argv[1]), int(sys.argv[2]))
sd = W.make_state_dict("pix2pix", cfg, seed=0, perturb_norm=True)
e = i2it.Engine(dt, i2it.PIX2PIX, cfg=cfg, use_cuda_graph=False)
e.load_state_dict(sd)
e.set_adapter_scale("default", 1.0)
e.set_adapter_scale("vae_skip", 2.0)
e.finalize(1.0, 1.0, 1.0, -1.0)
g = torch.Generator().manual_seed(1)
x = (torch.rand(B, 1, H, H, generator=g) < 0.08).float().expand(-1, 3, -1, -1).contiguous().to(dt).cuda()
text = torch.randn(1, 77, cfg["cross_dim"], generator=g).to(dt).cuda()
eps = torch.randn(B, 4, H // 8, H // 8, generator=g).to(dt).cuda()
out = e.forward(x, text, eps)
e.set_text(text)
out2 = e.forward(x, None, eps)
img = (torch.rand(B, H, H, 3, generator=g) * 255).to(torch.uint8).cuda()
u8 = e.forward_u8(img, i2it.IN_UNIT, None, eps)
torch.cuda.synchronize()
assert torch.isfinite(out.float()).all() and torch.equal(out, out2)
print("sanitize target ok: launches", e.launch_count(B, H, H), "prep launches", e.prep_launch_count())
