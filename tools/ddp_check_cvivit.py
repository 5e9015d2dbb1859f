"""Two-or-more-GPU check of data-parallel C-ViViT training (torchrun, NCCL): ``CViViT.sync_gradients`` with the
all-reduce launched slice by slice on a side stream while phk_cvivit_backward still runs (phk_train_set_progress_events)
must give the same averaged gradients as one all-reduce of the whole bucket after the backward, and both must equal the
mean of the per-rank gradients.  Then it times the training step (loss = cvivit(shard); loss.backward()) both ways,
alternating them, at the configs[1] C-ViViT shape with a shard of 2 videos of 17 frames per rank, in bf16 mode; each
timing is the max over ranks.  Prints one line on rank 0 with the card's name and power limit.
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29518 \
        tools/ddp_check_cvivit.py [steps=5] [rounds=3]"""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import phenaki_pytorch_b200 as P  # noqa: E402
from phenaki_pytorch_b200 import _lib as L  # noqa: E402
from phenaki_pytorch_b200 import sharding  # noqa: E402

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 3
rank, local, world = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
dist.init_process_group("nccl", device_id=dev)
torch.manual_seed(0)  # same weights on every rank
cv = P.CViViT(dim=512, codebook_size=65536, image_size=256, patch_size=32, temporal_patch_size=2, spatial_depth=4,
              temporal_depth=4, use_vgg_and_gan=False).to(dev)
cv.precision = L.PREC_BF16
g = torch.Generator().manual_seed(100 + rank)  # different data per rank
video = torch.randn((2, 3, 17, 256, 256), generator=g).to(dev)
real_plan = sharding.overlap_plan


def step(sync, overlap):
    cv.sync_gradients = sync
    sharding.overlap_plan = real_plan if overlap else (lambda *a, **k: None)
    cv.zero_grad(set_to_none=True)
    cv(video).backward()


def grads(sync, overlap):
    step(sync, overlap)
    torch.cuda.synchronize()
    return {k: p.grad.detach().clone() for k, p in cv.named_parameters() if p.grad is not None}


local_g = grads(False, False)
mean_g = {}
for k, v in local_g.items():
    t = v.clone()
    dist.all_reduce(t)
    mean_g[k] = t / world
plain = grads(True, False)
over = grads(True, True)
used_overlap = bool(cv.__dict__.get("_overlap_cache"))
worst_a = worst_b = 0.0
top = max(float(v.abs().max()) for v in mean_g.values() if v.numel())
for k in mean_g:
    if mean_g[k].numel() == 0:
        continue
    # bf16 products and atomics: each step's gradients differ from the next by rounding, so the bar is relative to the
    # largest gradient (the per-rank gradients above were taken in their own step)
    worst_a = max(worst_a, (plain[k] - mean_g[k]).abs().max().item() / top)
    worst_b = max(worst_b, (over[k] - mean_g[k]).abs().max().item() / top)
ok = worst_a < 1e-5 and worst_b < 1e-5 and used_overlap


def window(overlap):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dist.barrier()
    e0.record()
    for _ in range(steps):
        step(True, overlap)
    e1.record()
    torch.cuda.synchronize()
    return sharding.max_over_ranks(e0.elapsed_time(e1) / steps, dev)


for overlap in (False, True):
    step(True, overlap)
times = {False: [], True: []}
for _ in range(rounds):
    for overlap in (False, True):
        times[overlap].append(window(overlap))
res = torch.tensor([float(ok)], device=dev)
dist.all_reduce(res, op=dist.ReduceOp.MIN)
if rank == 0:
    card = subprocess.run(["nvidia-smi", f"--id={local}", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    print(f"DDP_CHECK_CVIVIT world={world} card='{card}' overlap_used={used_overlap} worst_rel_err "
          f"whole-bucket={worst_a:.2e} sliced-overlapped={worst_b:.2e} step_ms whole-bucket={med[False]:.2f} "
          f"overlapped={med[True]:.2f} {'OK' if res.item() == 1.0 else 'FAILED'}")
dist.destroy_process_group()
sys.exit(0 if res.item() == 1.0 else 1)
