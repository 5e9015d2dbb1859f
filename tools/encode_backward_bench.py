"""Times the differentiable C-ViViT encoder -- encode(tokens), then (out * G).sum().backward(), i.e. the encoder stacks
plus phk_cvivit_encode_backward (which recomputes both stacks with saved activations) -- against the no-grad
encode(tokens) on the same tokens, alternating the two in one process.  Shape: BASELINE.json configs[1] C-ViViT encoder
(dim 512, 8 x 64 heads, depth 4 + 4, 8 x 8 patches of a 256^2 frame), T' = 9, B = 2 and 8.  fp32 and bf16 modes.  CUDA
events around each window, warm-up first, the median of `rounds` windows; prints one JSON line with the card's name and
power limit.
usage: python tools/encode_backward_bench.py [steps=5] [rounds=3]"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import phenaki_pytorch_b200 as P  # noqa: E402
from phenaki_pytorch_b200 import _lib as L  # noqa: E402

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 3
dev = torch.device("cuda", 0)
torch.manual_seed(0)
cv = P.CViViT(dim=512, codebook_size=65536, image_size=256, patch_size=32, temporal_patch_size=2, spatial_depth=4,
              temporal_depth=4, use_vgg_and_gan=False).to(dev)
TP = 9


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
result = dict(what="C-ViViT encode(tokens): no-grad encode vs encode + (out * G).sum().backward()", tp=TP,
              steps_per_window=steps, rounds=rounds, card=card)
for B in (2, 8):
    tokens = torch.randn((B, TP, 8, 8, 512), device=dev)
    leaf = tokens.clone().requires_grad_(True)
    G = torch.randn_like(tokens)

    def no_grad_encode():
        with torch.no_grad():
            cv.encode(tokens)

    def encode_backward():
        cv.zero_grad(set_to_none=True)
        leaf.grad = None
        (cv.encode(leaf) * G).sum().backward()

    for name, prec in (("f32", L.PREC_F32), ("bf16", L.PREC_BF16)):
        cv.precision = prec
        for fn in (no_grad_encode, encode_backward):
            fn(), fn()
        torch.cuda.synchronize()
        fwd, bwd = [], []
        for _ in range(rounds):
            fwd.append(window(no_grad_encode))
            bwd.append(window(encode_backward))
        result[f"B={B}/{name}"] = dict(encode_ms=sorted(fwd)[len(fwd) // 2], encode_backward_ms=sorted(bwd)[len(bwd) // 2],
                                       encode_ms_all=fwd, encode_backward_ms_all=bwd)
result["peak_mem_gb"] = torch.cuda.max_memory_allocated() / 2 ** 30
print(json.dumps(result))
