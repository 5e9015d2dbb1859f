"""Times the differentiable C-ViViT decode -- decode_from_codebook_indices(ids), then (video * G).sum().backward(), i.e.
the inference decode plus phk_cvivit_decode_backward (which recomputes the decode with saved activations) -- against the
no-grad decode on the same ids, alternating the two in one process.  Shape: BASELINE.json configs[4] C-ViViT decode
(dim 512, image 256, patch 32, temporal patch 2, depth 4 + 4), B = 2, T' = 9 and 10.  fp32 and bf16 modes.  CUDA events
around each window, warm-up first; prints one JSON line with the card's name and power limit.
usage: python tools/decode_backward_bench.py [steps=5] [rounds=3]"""
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
B = 2


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
result = dict(what="C-ViViT decode: no-grad decode vs decode + (video * G).sum().backward()", batch=B,
              steps_per_window=steps, rounds=rounds, card=card)
for tp in (9, 10):
    ids = torch.randint(0, 65536, (B, tp * 64), device=dev)
    frames = 1 + (tp - 1) * 2
    G = torch.randn((B, 3, frames, 256, 256), device=dev)

    def no_grad_decode():
        with torch.no_grad():
            cv.decode_from_codebook_indices(ids)

    def decode_backward():
        cv.zero_grad(set_to_none=True)
        (cv.decode_from_codebook_indices(ids) * G).sum().backward()

    for name, prec in (("f32", L.PREC_F32), ("bf16", L.PREC_BF16)):
        cv.precision = prec
        for fn in (no_grad_decode, decode_backward):
            fn(), fn()
        torch.cuda.synchronize()
        fwd, bwd = [], []
        for _ in range(rounds):
            fwd.append(window(no_grad_decode))
            bwd.append(window(decode_backward))
        result[f"T'={tp}/{name}"] = dict(decode_ms=sorted(fwd)[len(fwd) // 2], decode_backward_ms=sorted(bwd)[len(bwd) // 2],
                                         decode_ms_all=fwd, decode_backward_ms_all=bwd)
result["peak_mem_gb"] = torch.cuda.max_memory_allocated() / 2 ** 30
print(json.dumps(result))
