"""Times a training step through the differentiable MaskGit forward -- F.cross_entropy(maskgit(masked)[m], ids[m])
.backward(), i.e. the inference forward plus phk_maskgit_backward (which recomputes the forward with saved activations) --
against Phenaki.forward(...).backward() (phk_maskgit_train_step) on the same ids and text, alternating the two in one
process.  Shape: BASELINE.json configs[3] MaskGit (dim 512, depth 6, V 65536, ctx 768), b sequences of 576 tokens,
16 text tokens.  CUDA events around each window of steps, warm-up first; prints one JSON line with the card's name and
power limit.
usage: python tools/forward_backward_bench.py [batch=4] [steps=3] [rounds=3]"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import bench  # noqa: E402
import phenaki_pytorch_b200 as P  # noqa: E402
from phenaki_pytorch_b200 import _lib as L  # noqa: E402

b = int(sys.argv[1]) if len(sys.argv) > 1 else 4
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
rounds = int(sys.argv[3]) if len(sys.argv) > 3 else 3
dev = torch.device("cuda", 0)
torch.manual_seed(0)
mg = P.MaskGit(**bench.CFG3).to(dev).train()
cv = P.CViViT(dim=64, codebook_size=65536, image_size=32, patch_size=16, temporal_patch_size=2, spatial_depth=1,
              temporal_depth=1, dim_head=32, heads=2).to(dev)  # only the constructor needs one: the ids are given
ph = P.Phenaki(cvivit=cv, maskgit=mg, steps=18, text_embed_dim=768).to(dev).train()
ph.sync_gradients = False
n, shape, L_, V = 576, (9, 8, 8), 16, 65536
ids = torch.randint(0, V, (b, n), device=dev)
mask = torch.rand((b, n), device=dev) < 0.5
mask[:, 0] = True
ctx = torch.randn(b, L_, 768, device=dev)
inp = torch.where(mask, V, ids)


def through_forward():
    mg.zero_grad(set_to_none=True)
    logits = mg(inp, video_patch_shape=shape, context=ctx)
    F.cross_entropy(logits[mask], ids[mask]).backward()


def through_train_step():
    mg.zero_grad(set_to_none=True)
    ph(video_codebook_ids=ids.reshape(b, *shape), text_embeds=ctx).backward()


def window(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
result = dict(what="MaskGit training step: differentiable forward + cross entropy vs Phenaki.forward (train step)",
              batch=b, tokens=b * n, steps_per_window=steps, rounds=rounds, card=card)
for name, prec in (("f32", L.PREC_F32), ("bf16", L.PREC_BF16)):
    mg.precision = prec
    for fn in (through_forward, through_train_step):
        fn(), fn()
    torch.cuda.synchronize()
    fwd, step = [], []
    for _ in range(rounds):
        fwd.append(window(through_forward))
        step.append(window(through_train_step))
    result[name] = dict(forward_backward_ms=sorted(fwd)[len(fwd) // 2], train_step_ms=sorted(step)[len(step) // 2],
                        forward_backward_ms_all=fwd, train_step_ms_all=step)
result["peak_mem_gb"] = torch.cuda.max_memory_allocated() / 2 ** 30
print(json.dumps(result))
