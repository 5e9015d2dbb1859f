"""GPU: uint8 videos through the C-ViViT encode.  A uint8 video u means the fp32 video u.float() / 255 (torchvision
ToTensor's convention, the quotient correctly rounded) and must give, bit for bit, what that fp32 video gives:

- phk_patchify_ln_u8 against phk_patchify_ln, fp32 and bf16 out, on the TMA path (configs[1] first and remaining frames)
  and on every fallback (bytes that do not fit a TMA box, a 1-byte-offset view, the generic kernel's two orders);
- the ids and the four encode taps of every C-ViViT golden case and of the configs[1] shape, in every precision mode;
- the host pipeline (pinned uint8 batches), CUDA-graph replay on a buffer an fp32 encode captured, and the consumers
  Phenaki.forward(videos=...) and Phenaki.sample(prime_frames=...);
- what stays refused: uint8 in the reconstruction loss, and any other dtype (before anything is launched).

The fp32 reference videos are divided on the CPU: on CUDA, u.float() / 255 multiplies by a rounded reciprocal and can be
one ulp off.  tests/test_encode_u8_emulated_cpu.py runs the kernel and model checks below on the CPU executor."""
import math

import pytest
import torch

import phenaki_pytorch_b200 as P
from phenaki_pytorch_b200 import _lib as L
from tests import cases as C
from tests import text_grad_cases as TG

pytestmark = pytest.mark.gpu

DEV = "cuda"
CFG2 = dict(dim=512, codebook_size=65536, image_size=256, patch_size=32, temporal_patch_size=2, spatial_depth=4,
            temporal_depth=4, dim_head=64, heads=8, use_vgg_and_gan=False)
CFG2_VIDEO = (8, 3, 17, 256, 256)
PRECISIONS = {"f32": L.PREC_F32, "bf16x3": L.PREC_BF16X3, "bf16": L.PREC_BF16}


def u8_video(shape, seed):
    return torch.randint(0, 256, shape, generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)


def as_float(u):
    """ToTensor's fp32 video of u, divided on the CPU."""
    return u.cpu().float() / 255


def at_offset(u, offset, dev):
    """u on `dev` at `offset` bytes past an allocation's (256-byte aligned) start."""
    buf = torch.empty(u.numel() + offset, dtype=torch.uint8, device=dev)
    view = buf[offset:].view(u.shape)
    view.copy_(u)
    return buf, view


# (B, C, F, H, W, f0, nt, pt, p1, p2), byte offset of the uint8 video
KERNEL_SHAPES = {
    "cfg2_first_frame": ((8, 3, 17, 256, 256, 0, 1, 1, 32, 32), 0),      # TMA
    "cfg2_rest_frames": ((8, 3, 17, 256, 256, 1, 8, 2, 32, 32), 0),      # TMA
    "p2_8": ((2, 3, 5, 32, 48, 1, 2, 2, 8, 8), 0),                       # fp32 TMA; bytes: register kernel
    "w_36": ((2, 3, 5, 24, 36, 1, 2, 2, 12, 12), 0),                     # W % 16 != 0: as above
    "offset_1": ((2, 3, 5, 64, 64, 1, 2, 2, 32, 32), 1),                 # fp32 TMA; bytes: generic kernel, grouped
    "offset_2_p2_8": ((2, 3, 5, 32, 48, 1, 2, 2, 8, 8), 2),              # as above
    "k_6400": ((1, 1, 3, 80, 80, 0, 1, 1, 80, 80), 0),                   # TMA beyond the register kernel's K
    "k_6400_offset_3": ((1, 1, 3, 80, 80, 0, 1, 1, 80, 80), 3),          # fp32 TMA; bytes: generic kernel, grouped
    "k_6912": ((1, 3, 3, 32, 72, 1, 1, 2, 32, 36), 0),                   # generic kernel, grouped mean only
    "p2_6": ((1, 1, 3, 12, 18, 0, 1, 1, 6, 6), 0),                       # generic kernel, element order
    "p2_6_offset_1": ((1, 1, 3, 12, 18, 0, 1, 1, 6, 6), 1),
}


def check_patchify(shape, offset, dev, seed=0):
    B, Cc, F, H, W, f0, nt, pt, p1, p2 = shape
    K = Cc * pt * p1 * p2
    u = u8_video((B, Cc, F, H, W), seed)
    g = (torch.randn(K, generator=torch.Generator().manual_seed(seed + 1)) * 0.5 + 1).to(dev)
    b = torch.randn(K, generator=torch.Generator().manual_seed(seed + 2)).to(dev)
    _buf, ud = at_offset(u, offset, dev)
    vf = as_float(u).to(dev)
    rows = B * nt * (H // p1) * (W // p2)
    lib = L.lib()
    for out_bf16, dtype in ((0, torch.float32), (1, torch.bfloat16)):
        want = torch.empty((rows, K), dtype=dtype, device=dev)
        got = torch.empty((rows, K), dtype=dtype, device=dev)
        L.check(lib.phk_patchify_ln(L.ptr(vf), B, Cc, F, H, W, f0, nt, pt, p1, p2, L.ptr(g), L.ptr(b), L.ptr(want),
                                    out_bf16, L.stream_ptr()), "phk_patchify_ln")
        L.check(lib.phk_patchify_ln_u8(L.ptr(ud), B, Cc, F, H, W, f0, nt, pt, p1, p2, L.ptr(g), L.ptr(b), L.ptr(got),
                                       out_bf16, L.stream_ptr()), "phk_patchify_ln_u8")
        assert bool(torch.isfinite(want.float()).all())
        assert torch.equal(got, want), f"out_bf16={out_bf16}: {int((got != want).sum())} elements differ"


def check_model(model, u, dev):
    """ids and the encode taps of the uint8 video u equal, bit for bit, those of its fp32 video; so does the public call
    (4-D u: an image)."""
    u5 = u if u.ndim == 5 else u.unsqueeze(2)
    got_taps, want_taps = {}, {}
    want = model.encode_ids(as_float(u5).to(dev), taps=want_taps)
    got = model.encode_ids(u5.to(dev), taps=got_taps)
    assert got.dtype == torch.int64 and torch.equal(got, want)
    assert got_taps.keys() == want_taps.keys() and {"patch", "spatial", "temporal"} <= set(want_taps)
    for k in want_taps:
        assert torch.equal(got_taps[k], want_taps[k]), f"tap {k} differs"
    ud = u.to(dev)
    for _ in range(3):  # eager, captured into a graph, replayed
        assert torch.equal(model(ud, return_only_codebook_ids=True), want)


def case_model(name, dev):
    case = C.CVIVIT_CASES[name]
    torch.manual_seed(case["seed"])
    return P.CViViT(**case["ctor"]).to(dev).eval(), u8_video(case["video"], case["video_seed"])


@pytest.mark.parametrize("name", list(KERNEL_SHAPES))
def test_patchify_ln_u8_equals_the_fp32_op(name):
    shape, offset = KERNEL_SHAPES[name]
    check_patchify(shape, offset, DEV)


_CFG2 = {}


def cfg2_model():
    if "m" not in _CFG2:
        torch.manual_seed(0)
        _CFG2["m"] = P.CViViT(**CFG2).to(DEV).eval()
    return _CFG2["m"]


@pytest.mark.parametrize("prec", list(PRECISIONS))
@pytest.mark.parametrize("name", [*C.CVIVIT_CASES, "configs1"])
def test_encode_ids_and_taps_of_uint8_equal_the_fp32_video(name, prec):
    if name == "configs1":
        model, u = cfg2_model(), u8_video(CFG2_VIDEO, 1)
    else:
        model, u = case_model(name, DEV)
    model.precision = PRECISIONS[prec]
    check_model(model, u, DEV)


@pytest.mark.parametrize("depth", [1, 2, 3])
def test_encode_host_iter_takes_pinned_uint8_batches(depth):
    model, _ = case_model("rect", DEV)
    shape = C.CVIVIT_CASES["rect"]["video"]
    batches = [u8_video(shape, 100 + i).pin_memory() for i in range(7)]
    want = [model(v.to(DEV), return_only_codebook_ids=True).cpu() for v in batches]
    got = list(model.encode_host_iter(iter(batches), depth=depth))
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(got, want)):
        assert not a.is_cuda and a.dtype == torch.int64 and torch.equal(a, b), f"batch {i}"
    assert torch.equal(model.encode_host(as_float(batches[3]).pin_memory()), want[3])
    with pytest.raises(AssertionError):
        list(model.encode_host_iter([batches[0], as_float(batches[1]).pin_memory()]))  # one dtype per stream
    with pytest.raises(AssertionError):
        list(model.encode_host_iter([as_float(batches[0]).pin_memory(), batches[1]]))


def test_graph_replay_keys_on_the_video_dtype():
    """One buffer seen as fp32 and as uint8 (same address): three fp32 encodes capture and replay a graph, then each
    uint8 encode of new bytes must equal the eager launches (taps keep a call eager)."""
    model, _ = case_model("rect", DEV)
    shape = C.CVIVIT_CASES["rect"]["video"]
    n = math.prod(shape)
    buf = torch.empty(4 * n, dtype=torch.uint8, device=DEV)
    f32, u8 = buf.view(torch.float32).view(shape), buf[:n].view(shape)
    assert f32.data_ptr() == u8.data_ptr()
    f32.copy_(C.seeded_randn(shape, 40))
    first = [model(f32, return_only_codebook_ids=True) for _ in range(3)]
    assert all(torch.equal(x, first[0]) for x in first)
    for i in range(3):
        u8.copy_(u8_video(shape, 50 + i))
        got = model(u8, return_only_codebook_ids=True)
        want = model.encode_ids(u8, taps={})
        assert torch.equal(got, want), f"uint8 call {i}"
        assert torch.equal(want, model.encode_ids(as_float(u8).to(DEV), taps={}))


def test_phenaki_forward_takes_uint8_videos():
    """Phenaki.forward(videos=u8) tokenises through the same encode: the loss and every gradient equal those of the fp32
    videos under the same seed and draws (deterministic mode: the backward's reductions repeat bit for bit)."""
    case = dict(C.FRAME_MASK_TRAIN_CASE, critic_kind="token")
    phenaki = TG.build(case, device=DEV)
    u = u8_video(case["video"], case["input_seed"])
    fmask = C.frame_mask_of(case["frames_valid"], case["video"][2]).to(DEV)
    ctx = C.train_inputs(case)[1].to(DEV)
    draws = TG.decisive_draws(case)

    def run(videos):
        phenaki.zero_grad(set_to_none=True)
        torch.manual_seed(3)
        loss = phenaki(videos, text_embeds=ctx, video_frame_mask=fmask, draw_fn=lambda shape, tag: draws[tag].to(DEV))
        loss.backward()
        return loss.detach(), TG.product_grads(phenaki)

    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        loss_u8, grads_u8 = run(u.to(DEV))
        loss_f, grads_f = run(as_float(u).to(DEV))
    finally:
        torch.use_deterministic_algorithms(was)
    assert torch.equal(loss_u8, loss_f)
    assert grads_u8.keys() == grads_f.keys() and any(g is not None for g in grads_f.values())
    for k, g in grads_f.items():
        assert (g is None) == (grads_u8[k] is None) and (g is None or torch.equal(grads_u8[k], g)), k


def test_phenaki_sample_primes_with_uint8_frames():
    case = C.SAMPLE_CASES["critic_primed"]
    torch.manual_seed(case["seed"])
    ph = P.Phenaki(cvivit=P.CViViT(**C.SAMPLE_CVIVIT).to(DEV), maskgit=P.MaskGit(**C.SAMPLE_MASKGIT).to(DEV),
                   critic=P.TokenCritic(**C.SAMPLE_CRITIC).to(DEV), steps=case["steps"],
                   text_embed_dim=C.SAMPLE_MASKGIT["dim_context"])
    ctx = C.synthetic_text_embeds(case["batch"], case["ctx_len"], C.SAMPLE_MASKGIT["dim_context"], case["ctx_valid"],
                                  case["seed"] + 1000).to(DEV)
    prime = u8_video((case["batch"], 3, case["prime_frames"], *C.SAMPLE_CVIVIT["image_size"]), case["seed"] + 2000)

    def sample(frames):
        tape = C.NoiseTape(case["noise_seed"])
        return ph.sample(num_frames=case["num_frames"], text_embeds=ctx, prime_frames=frames,
                         cond_scale=case["cond_scale"], return_token_ids=True,
                         noise_fn=lambda shape, tag: tape(shape, tag).to(DEV))

    assert torch.equal(sample(prime.to(DEV)), sample(as_float(prime).to(DEV)))


def test_other_dtypes_and_the_reconstruction_loss_are_refused():
    model, u = case_model("rect", DEV)
    ud = u.to(DEV)
    model(ud, return_only_codebook_ids=True)  # tables and the position bias exist: a refusal has nothing left to build
    with pytest.raises(L.PhkError, match="float32"):
        model(ud)
    with pytest.raises(L.PhkError, match="float32"):
        model(ud, return_recons=True)
    lib = L.lib()
    for dtype in (torch.float16, torch.int16):
        v = ud.to(dtype)
        torch.cuda.synchronize()
        n0 = lib.phk_launch_count()
        with pytest.raises(L.PhkError):
            model(v, return_only_codebook_ids=True)
        with pytest.raises(L.PhkError):
            model(v, return_recons_only=True)
        with pytest.raises(L.PhkError):
            list(model.encode_host_iter([v.cpu()]))
        assert lib.phk_launch_count() == n0
