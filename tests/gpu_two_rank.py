"""torchrun target (2 ranks, NCCL): the N-rank sharded forward (dist.sharded_forward: contiguous batch split + ONE all-gather of
the images) equals the single-rank forward of the whole batch bit for bit, through the public Pix2Pix_Turbo API.
Launched by tests/test_gpu_boundary.py::test_two_rank_sharded_output_equals_single_rank."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "img2img-turbo_b200"))

import weights as W  # noqa: E402
from dist import sharded_forward  # noqa: E402
from pix2pix_turbo import Pix2Pix_Turbo  # noqa: E402

rank, local = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
full = os.environ.get("I2IT_TWO_RANK_FULL", "0") == "1"
cfg, B, S = (W.SD_TURBO, 4, 512) if full else (W.TINY, 6, 64)
m = Pix2Pix_Turbo(cfg=None if full else cfg, perturb_norm=not full)
m.set_eval()
m.to(torch.bfloat16)
g = torch.Generator().manual_seed(7)
x = (torch.rand(B, 1, S, S, generator=g) < 0.08).float().expand(-1, 3, -1, -1).contiguous().cuda().bfloat16()
eps = torch.randn(B, 4, S // 8, S // 8, generator=g).cuda().bfloat16()
with torch.no_grad():
    whole = m(x, "a prompt", eps=eps)                       # single-rank output of the whole batch
    shard = sharded_forward(m, x, "a prompt", eps=eps)      # this rank's slice + NCCL all-gather
torch.cuda.synchronize()
assert shard.shape == whole.shape and torch.isfinite(whole.float()).all()
assert torch.equal(shard, whole), f"rank {rank}: sharded != single-rank, max diff {(shard.float() - whole.float()).abs().max().item()}"
# every rank holds the same gathered batch
chk = shard.float().sum().reshape(1)
both = [torch.zeros_like(chk) for _ in range(dist.get_world_size())]
dist.all_gather(both, chk)
assert all(torch.equal(b, both[0]) for b in both)
print(f"rank {rank}: TWO_RANK_OK world={dist.get_world_size()} B={B} S={S} cfg={'sd-turbo' if full else 'tiny'}", flush=True)
dist.destroy_process_group()
