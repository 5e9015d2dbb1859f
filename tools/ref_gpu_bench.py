"""The same-box GPU bar (SURVEY 2a / 8d, BASELINE.md 4.4): the reference's own PyTorch path on the GPU -- the oracle
port (same ATen ops as the reference modules; /root/reference does not exist on the GPU box) on CUDA, eager fp32 (torch
defaults) and under torch.autocast(bfloat16) -- for configs[1] (C-ViViT encode) and configs[2] (18-step demasking loop).
bench.py imports `encode_leg` / `maskgit_leg`; standalone:  python tools/ref_gpu_bench.py
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

CFG2 = dict(dim=512, codebook_size=65536, image_size=256, patch_size=32, temporal_patch_size=2, spatial_depth=4,
            temporal_depth=4, dim_head=64, heads=8, use_vgg_and_gan=False)
CFG3 = dict(dim=512, num_tokens=65536, max_seq_len=1024, dim_context=768, depth=6)


def _time(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def encode_leg(dev, batch=8, frames=17, warmup=3, iters=10):
    from oracle import phenaki_oracle as O
    import phenaki_pytorch_b200 as P
    torch.manual_seed(0)
    sd = {k: v.detach().to(dev) for k, v in P.CViViT(**CFG2).state_dict().items()}
    video = torch.randn((batch, 3, frames, 256, 256), device=dev)
    out = {}
    with torch.no_grad():
        ms = _time(lambda: O.cvivit_codebook_ids(video, sd, (256, 256), (32, 32)), warmup, iters)
        out["eager_fp32"] = dict(ms_per_step=ms, value=batch * frames / ms * 1e3, unit="frames/s")
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ms = _time(lambda: O.cvivit_codebook_ids(video, sd, (256, 256), (32, 32)), warmup, iters)
        out["autocast_bf16"] = dict(ms_per_step=ms, value=batch * frames / ms * 1e3, unit="frames/s")
    out["what"] = (f"oracle port of the reference modules (same ATen ops) on {torch.cuda.get_device_name(dev)}, torch "
                   f"{torch.__version__} eager (cuBLAS / cuDNN kernels), ({batch},3,{frames},256,256), {iters} timed calls")
    return out


def maskgit_leg(dev, batch=4, steps=18, iters=2):
    from oracle import phenaki_oracle as O
    import phenaki_pytorch_b200 as P
    torch.manual_seed(1)
    sd = {k: v.detach().to(dev) for k, v in P.MaskGit(**CFG3).state_dict().items()}
    ctx = torch.randn((batch, 16, 768), device=dev)
    noise = lambda shape, tag: torch.rand(shape, device=dev)   # the reference's zeros_like(t).uniform_(0, 1)
    run = lambda: O.sample_token_ids(sd, num_tokens=576, patch_shape=(9, 8, 8), batch=batch, steps=steps,
                                     text_embeds=ctx, cond_scale=3.0, noise_fn=noise)
    out = {}
    tokens = batch * 576 * steps
    with torch.no_grad():
        ms = _time(run, 1, iters)
        out["eager_fp32"] = dict(ms_per_sample=ms, ms_per_decode_step=ms / steps, value=tokens / ms * 1e3, unit="tokens/s")
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ms = _time(run, 1, iters)
        out["autocast_bf16"] = dict(ms_per_sample=ms, ms_per_decode_step=ms / steps, value=tokens / ms * 1e3, unit="tokens/s")
    out["what"] = (f"oracle port of Phenaki.sample's demasking loop (2 MaskGit forwards per step, V-wide gumbel / softmax "
                   f"in ATen, one host sync per step as in the reference) on CUDA, b={batch}, N=576, {steps} steps, "
                   f"{iters} timed samples")
    return out


if __name__ == "__main__":
    d = torch.device("cuda", 0)
    print(json.dumps(dict(encode=encode_leg(d), maskgit=maskgit_leg(d)), indent=1))
