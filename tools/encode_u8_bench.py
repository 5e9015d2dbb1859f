"""What uint8 frames buy a tokenisation job: the configs[1] C-ViViT (B = 8, F = 17, 256 x 256) encoding fp32 and uint8
videos, alternated in one process, in bf16 mode (the benchmarked mode) and the default split-bf16 mode:

  (a) device-resident  CViViT.encode_ids on videos already on the GPU (CUDA events around `--steps` calls);
  (b) host-to-host     CViViT.encode_host_iter over pinned batches (host clock around the stream, ending in a
                       synchronise), H2D copy + encode + D2H of the ids, the copy of batch i+1 overlapping batch i.

Three distinct batches per dtype are cycled so no call finds its video in L2.  Every figure is the median over
`--windows` windows (frames/s).  Also: the H2D time of one pinned batch per dtype (CUDA events, median of 10), whether
the uint8 ids equal the fp32 ids of the same frames at this size, and the card's name and power limit (read-only
nvidia-smi query).  Prints one JSON line.

    python tools/encode_u8_bench.py [--steps 200] [--host-steps 60] [--windows 5] [--warmup 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import phenaki_pytorch_b200 as P  # noqa: E402
from phenaki_pytorch_b200 import _lib as L  # noqa: E402

CFG2 = dict(dim=512, codebook_size=65536, image_size=256, patch_size=32, temporal_patch_size=2, spatial_depth=4,
            temporal_depth=4, dim_head=64, heads=8, use_vgg_and_gan=False)
VIDEO = (8, 3, 17, 256, 256)
MODES = {"bf16": L.PREC_BF16, "bf16x3": L.PREC_BF16X3}


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                      text=True, timeout=30)
        name, power = [s.strip() for s in out.splitlines()[0].split(",")]
        return dict(gpu=name, power_limit=power)
    except Exception as ex:  # the numbers stay valid; say what is missing
        return dict(gpu=torch.cuda.get_device_name(0), power_limit=f"unknown ({ex.__class__.__name__})")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--host-steps", type=int, default=60)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    assert args.windows >= 3
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    model = P.CViViT(**CFG2).to(dev).eval()
    B, F = VIDEO[0], VIDEO[2]
    host = {"u8": [torch.randint(0, 256, VIDEO, generator=torch.Generator().manual_seed(100 + i),
                                 dtype=torch.uint8).pin_memory() for i in range(3)]}
    host["f32"] = [(u.float() / 255).pin_memory() for u in host["u8"]]  # ToTensor's quotients, divided on the CPU
    vids = {k: [h.to(dev) for h in v] for k, v in host.items()}
    torch.cuda.synchronize()

    def device_window(dtype):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(args.steps):
            model.encode_ids(vids[dtype][i % 3])
        e1.record()
        e1.synchronize()
        return B * F * args.steps / (e0.elapsed_time(e1) / 1e3)

    def host_window(dtype):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in model.encode_host_iter((host[dtype][i % 3] for i in range(args.host_steps)), device=dev):
            pass
        torch.cuda.synchronize()
        return B * F * args.host_steps / (time.perf_counter() - t0)

    def h2d_ms(dtype):
        dst = torch.empty_like(vids[dtype][0])
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        times = []
        for i in range(10):
            e0.record()
            dst.copy_(host[dtype][i % 3], non_blocking=True)
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
        return statistics.median(times)

    result = dict(metric="configs[1] C-ViViT encode, fp32 vs uint8 videos", unit="frames/s", batch=list(VIDEO),
                  windows=args.windows, device_steps=args.steps, host_steps=args.host_steps, **card(),
                  h2d_ms={d: round(h2d_ms(d), 3) for d in ("f32", "u8")}, modes={})
    for mode, prec in MODES.items():
        model.precision = prec
        ids_match = all(torch.equal(model.encode_ids(vids["u8"][i]), model.encode_ids(vids["f32"][i])) for i in range(3))
        for dtype in ("f32", "u8"):  # the library captures a graph per buffer on its second call
            for v in vids[dtype]:
                for _ in range(3):
                    model.encode_ids(v)
            for _ in range(args.warmup):
                model.encode_ids(vids[dtype][0])
            host_window(dtype)
        samples = {(p, d): [] for p in ("a_device", "b_host") for d in ("f32", "u8")}
        for _ in range(args.windows):
            for dtype in ("f32", "u8"):
                samples[("a_device", dtype)].append(device_window(dtype))
                samples[("b_host", dtype)].append(host_window(dtype))
        out = {p: {d: round(statistics.median(samples[(p, d)]), 1) for d in ("f32", "u8")} for p in ("a_device", "b_host")}
        out["ids_match"] = ids_match
        result["modes"][mode] = out
    print(json.dumps(result))


if __name__ == "__main__":
    main()
