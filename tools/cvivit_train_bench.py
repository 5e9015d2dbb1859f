"""Times one C-ViViT tokenizer training step -- loss = cvivit(video); loss.backward(), i.e. the inference encode, decode
and loss plus phk_cvivit_backward (which recomputes the decoder and the encoder with saved activations) -- against the
no-grad cvivit(video, return_recons_only=True) on the same video, alternating the two in one process.  Shape:
BASELINE.json configs[1] C-ViViT (dim 512, image 256, patch 32, temporal patch 2, depth 4 + 4), F = 17, B = 2 and 8, in
fp32 and bf16 modes.  CUDA events around each window, warm-up first, medians of the windows; prints one JSON line with the
card's name and power limit and phk_cvivit_backward_workspace_bytes at B = 8.
usage: python tools/cvivit_train_bench.py [steps=5] [rounds=3]"""
import ctypes as C
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
F = 17


def window(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def median(v):
    return sorted(v)[len(v) // 2]


card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
result = dict(what="C-ViViT: no-grad return_recons_only vs loss = cvivit(video); loss.backward()", frames=F,
              steps_per_window=steps, rounds=rounds, card=card)
for B in (2, 8):
    video = torch.randn((B, 3, F, 256, 256), device=dev)

    def recon_only():
        with torch.no_grad():
            cv(video, return_recons_only=True)

    def train_step():
        cv.zero_grad(set_to_none=True)
        cv(video).backward()

    for name, prec in (("f32", L.PREC_F32), ("bf16", L.PREC_BF16)):
        cv.precision = prec
        for fn in (recon_only, train_step):
            fn(), fn()
        torch.cuda.synchronize()
        fwd, step = [], []
        for _ in range(rounds):
            fwd.append(window(recon_only))
            step.append(window(train_step))
        result[f"B={B}/{name}"] = dict(recon_only_ms=median(fwd), train_step_ms=median(step), recon_only_ms_all=fwd,
                                       train_step_ms_all=step)
        if B == 8:
            nbytes = L.lib().phk_cvivit_backward_workspace_bytes(C.byref(cv._table()), C.byref(cv._dec_table()), B, F, prec)
            result[f"B={B}/{name}"]["backward_workspace_gib"] = nbytes / 2 ** 30
result["peak_mem_gb"] = torch.cuda.max_memory_allocated() / 2 ** 30
print(json.dumps(result))
