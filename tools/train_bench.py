"""Times the training step (phk_maskgit_train_step through MaskGit.train_step) at BASELINE.json configs[2]/[3] sizes:
MaskGit(dim 512, depth 6, V 65536, ctx 768), b sequences of 576 tokens, L text tokens.  CUDA events, warm-up first.
usage: python tools/train_bench.py [batch=4] [steps=5] [f32|bf16] [dropout=0]       (prints one JSON line)
dropout: the attention and FF dropout probability of the step (attn_dropout = ff_dropout, training mode)."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402
import phenaki_pytorch_b200 as P  # noqa: E402

b = int(sys.argv[1]) if len(sys.argv) > 1 else 4
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
prec = sys.argv[3] if len(sys.argv) > 3 else "f32"
dropout = float(sys.argv[4]) if len(sys.argv) > 4 else 0.0
dev = torch.device("cuda", 0)
torch.manual_seed(0)
mg = P.MaskGit(**bench.CFG3, attn_dropout=dropout, ff_dropout=dropout).to(dev).train()
mg.precision = P._lib.PREC_BF16 if prec == "bf16" else P._lib.PREC_F32
n, L_, V = 576, 16, 65536
ids = torch.randint(0, V, (b, n), device=dev)
mask = torch.rand((b, n), device=dev) < 0.5
ctx = torch.randn(b, L_, 768, device=dev)
inp = torch.where(mask, V, ids)


def step():
    loss, gk, _ = mg.train_step(inp, (9, 8, 8), targets=ids, token_mask=mask, context=ctx)
    return loss, gk


for _ in range(2):
    loss, gk = step()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(steps):
    loss, gk = step()
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / steps
flops = 3 * 277.1e9 * b / 4  # forward (SURVEY 8d, 277.1 GFLOP at b=4) + ~2x for the backward
print(json.dumps(dict(what=f"maskgit_train_step {prec}", batch=b, dropout=dropout, tokens=b * n, ms_per_step=ms,
                      tokens_per_s=b * n / ms * 1e3, approx_tflops=flops / ms / 1e9, loss=float(loss),
                      grad_norm=float(gk.flat.norm()), peak_mem_gb=torch.cuda.max_memory_allocated() / 2 ** 30)))
