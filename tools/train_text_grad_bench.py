"""Times Phenaki.forward(...).backward() (phk_maskgit_train_step) with and without text_embeds.requires_grad, alternating
the two in one process, in fp32 and bf16 mode.  Shape: BASELINE.json configs[3] MaskGit (dim 512, depth 6, V 65536,
ctx 768), b sequences of 576 tokens, 16 text tokens.  CUDA events around each window of steps, warm-up first; prints one
JSON line with the card's name and power limit.
usage: python tools/train_text_grad_bench.py [batch=4] [steps=5] [rounds=5]"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402
import phenaki_pytorch_b200 as P  # noqa: E402
from phenaki_pytorch_b200 import _lib as L  # noqa: E402

b = int(sys.argv[1]) if len(sys.argv) > 1 else 4
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
rounds = int(sys.argv[3]) if len(sys.argv) > 3 else 5
dev = torch.device("cuda", 0)
torch.manual_seed(0)
mg = P.MaskGit(**bench.CFG3).to(dev).train()
cv = P.CViViT(dim=64, codebook_size=65536, image_size=32, patch_size=16, temporal_patch_size=2, spatial_depth=1,
              temporal_depth=1, dim_head=32, heads=2).to(dev)  # only the constructor needs one: the ids are given
ph = P.Phenaki(cvivit=cv, maskgit=mg, steps=18, text_embed_dim=768).to(dev).train()
ph.sync_gradients = False
n, shape, L_, V = 576, (9, 8, 8), 16, 65536
ids = torch.randint(0, V, (b, *shape), device=dev)
ctx = torch.randn(b, L_, 768, device=dev)


def step(requires_grad):
    def run():
        mg.zero_grad(set_to_none=True)
        ph(video_codebook_ids=ids, text_embeds=ctx.detach().requires_grad_(requires_grad)).backward()
    return run


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
result = dict(what="Phenaki.forward(...).backward() without / with text_embeds.requires_grad", batch=b, tokens=b * n,
              steps_per_window=steps, rounds=rounds, card=card)
plain, with_grad = step(False), step(True)
for name, prec in (("f32", L.PREC_F32), ("bf16", L.PREC_BF16)):
    mg.precision = prec
    for fn in (plain, with_grad):
        fn(), fn()
    torch.cuda.synchronize()
    a, w = [], []
    for _ in range(rounds):
        a.append(window(plain))
        w.append(window(with_grad))
    result[name] = dict(no_text_grad_ms=sorted(a)[len(a) // 2], text_grad_ms=sorted(w)[len(w) // 2],
                        no_text_grad_ms_all=a, text_grad_ms_all=w)
print(json.dumps(result))
