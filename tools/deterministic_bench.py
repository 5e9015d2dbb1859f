"""Times the hand-written backwards with torch.use_deterministic_algorithms off and on, alternating the two in one
process, in fp32 and bf16 mode:
  Phenaki.forward(...).backward()  BASELINE.json configs[3] MaskGit (dim 512, depth 6, V 65536, ctx 768), 4 x 576 tokens,
                                   16 text tokens (phk_maskgit_train_step)
  cvivit(video).backward()         configs[1] C-ViViT (dim 512, depth 4 + 4, 256^2 images, 17 frames), B = 8
                                   (phk_cvivit_backward)
CUDA events around each window of steps, warm-up first; medians over the rounds; prints one JSON line with the card's
name and power limit.
usage: python tools/deterministic_bench.py [steps=3] [rounds=5]"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402
import phenaki_pytorch_b200 as P  # noqa: E402
from phenaki_pytorch_b200 import _lib as L  # noqa: E402

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 5
dev = torch.device("cuda", 0)
torch.manual_seed(0)


def window(fn, on):
    torch.use_deterministic_algorithms(on)
    try:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps
    finally:
        torch.use_deterministic_algorithms(False)


def median(v):
    return sorted(v)[len(v) // 2]


def compare(fn, set_precision):
    out = {}
    for name, prec in (("f32", L.PREC_F32), ("bf16", L.PREC_BF16)):
        set_precision(prec)
        for on in (False, True):  # warm-up of both (workspace sizes differ)
            window(fn, on)
        off, det = [], []
        for _ in range(rounds):
            off.append(window(fn, False))
            det.append(window(fn, True))
        out[name] = dict(off_ms=median(off), deterministic_ms=median(det), off_ms_all=off, deterministic_ms_all=det)
    return out


card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
result = dict(what="torch.use_deterministic_algorithms off vs on", steps_per_window=steps, rounds=rounds, card=card)

# ---- Phenaki.forward(...).backward() at configs[3]
mg = P.MaskGit(**bench.CFG3).to(dev).train()
cv = P.CViViT(dim=64, codebook_size=65536, image_size=32, patch_size=16, temporal_patch_size=2, spatial_depth=1,
              temporal_depth=1, dim_head=32, heads=2).to(dev)  # only the constructor needs one: the ids are given
ph = P.Phenaki(cvivit=cv, maskgit=mg, steps=18, text_embed_dim=768).to(dev).train()
ph.sync_gradients = False
b, V = 4, 65536
ids = torch.randint(0, V, (b, 9, 8, 8), device=dev)
ctx = torch.randn(b, 16, 768, device=dev)


def phenaki_step():
    mg.zero_grad(set_to_none=True)
    torch.manual_seed(1)
    ph(video_codebook_ids=ids, text_embeds=ctx).backward()


result["phenaki_cfg3"] = compare(phenaki_step, lambda p: setattr(mg, "precision", p))
del ph, mg, cv
torch.cuda.empty_cache()

# ---- cvivit(video).backward() at configs[1], B = 8
cvt = P.CViViT(dim=512, codebook_size=65536, image_size=256, patch_size=32, temporal_patch_size=2, spatial_depth=4,
               temporal_depth=4, use_vgg_and_gan=False).to(dev).train()
video = torch.randn((8, 3, 17, 256, 256), device=dev)


def cvivit_step():
    cvt.zero_grad(set_to_none=True)
    cvt(video).backward()


result["cvivit_cfg1_b8"] = compare(cvivit_step, lambda p: setattr(cvt, "precision", p))
print(json.dumps(result))
