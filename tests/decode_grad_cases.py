"""Check bodies of the differentiable C-ViViT decode tests, shared by the H100 file (tests/test_gpu_decode_backward.py) and
the CPU executor file (tests/test_decode_backward_emulated_cpu.py): every body takes (device, sync).

A case is a C-ViViT configuration of the decode goldens (tests/cases.py CVIVIT_CASES), or the configs[1]/[4] shape, with
seeded ids / tokens, and an entry point: ``decode(tokens)`` ("tokens") or ``decode_from_codebook_indices(ids)`` ("ids").
The product computes ``(video * G).sum().backward()`` for a seeded random G through phk_cvivit_decode_backward; the
reference is the float64 oracle (``oracle.cvivit_decode``) on the module's state dict under torch autograd."""
import functools

import torch
import torch.nn.functional as F

from oracle import phenaki_oracle as O
import phenaki_pytorch_b200 as P
from phenaki_pytorch_b200 import _lib as L
from tests import cases as CS
from tests import train_at_size_cases as T

# configs[1] / configs[4] C-ViViT: dim 512, 8 x 64 heads, depth 4 + 4, 256^2 images, patch 32, temporal patch 2
AT_SIZE = dict(dim=512, codebook_size=65536, image_size=256, patch_size=32, temporal_patch_size=2, spatial_depth=4,
               temporal_depth=4, use_vgg_and_gan=False)

# name -> (ctor, seed, batch, T')
CASES = {
    "cfg1": (CS.CVIVIT_CASES["cfg1"]["ctor"], 0, 1, 3),
    "rect": (CS.CVIVIT_CASES["rect"]["ctor"], 3, 2, 3),
    "image": (CS.CVIVIT_CASES["image"]["ctor"], 5, 3, 1),
    "cosine_vq": (CS.CVIVIT_CASES["cosine_vq"]["ctor"], 7, 2, 3),
    "at_size": (AT_SIZE, 11, 2, 9),
}
SMALL = ["cfg1", "rect", "image", "cosine_vq"]
ENTRIES = ["tokens", "ids"]

# Zero in exact arithmetic: the last bias of the position-bias MLP adds one constant per head to every spatial attention
# logit (no null keys there), and softmax is invariant to a constant shift.  Checked against an absolute bound only.
ANALYTICALLY_ZERO = ("spatial_rel_pos_bias.net.2.bias",)


def build_module(name):
    ctor, seed, _, _ = CASES[name]
    torch.manual_seed(seed)
    return P.CViViT(**ctor)


def _geometry(module):
    (ih, iw), (ph, pw) = module.image_size, module.patch_size
    return ih // ph, iw // pw


@functools.lru_cache(maxsize=None)
def inputs(name):
    """Seeded ids (b, T', h, w) and tokens (b, T', h, w, dim) of the case."""
    ctor, seed, b, tp = CASES[name]
    module = build_module(name)
    h, w = _geometry(module)
    g = torch.Generator().manual_seed(1000 + seed)
    ids = torch.randint(0, ctor["codebook_size"], (b, tp, h, w), generator=g)
    tokens = torch.randn((b, tp, h, w, ctor["dim"]), generator=g)
    return ids, tokens


def upstream_weights(name, entry, shape):
    g = torch.Generator().manual_seed(2000 + sorted(CASES).index(name) * 2 + ENTRIES.index(entry))
    return torch.randn(shape, generator=g, dtype=torch.float64)


@functools.lru_cache(maxsize=None)
def reference(name, entry):
    """{parameter name | "tokens": gradient} of (video * G).sum() by oracle autograd in float64 on the CPU; what the
    reference leaves without a gradient is absent."""
    module = build_module(name)
    ids, tokens = inputs(name)
    params = dict(module.named_parameters())
    sd = {}
    for k, v in module.state_dict().items():
        v = v.detach().to(torch.float64) if v.is_floating_point() else v.detach()
        sd[k] = v.requires_grad_(True) if k in params else v
    b, t, h, w = ids.shape
    tok = None
    if entry == "tokens":
        tok = tokens.to(torch.float64).requires_grad_(True)
        codes = tok
    elif "vq._codebook.embed" in sd:  # codes = vq.codebook[indices] (cvivit.py:441)
        codes = sd["vq._codebook.embed"][0][ids.reshape(b, -1)].reshape(b, t, h, w, -1)
    else:  # oracle.lfq_indices_to_codes in float64 (the oracle builds fp32 codes)
        bits = (ids.reshape(b, -1)[..., None].int() & sd["vq.mask"].int()) != 0
        codes = F.linear(torch.where(bits, 1.0, -1.0).to(torch.float64), sd["vq.project_out.weight"],
                         sd["vq.project_out.bias"]).reshape(b, t, h, w, -1)
    out = O.cvivit_decode(codes, sd, module.patch_size, module.temporal_patch_size, module.heads, module.channels)
    (out * upstream_weights(name, entry, out.shape)).sum().backward()
    grads = {k: sd[k].grad for k in params if sd[k].grad is not None}
    if t == 1:  # the reference runs to_pixels on an empty batch: zero gradients (the oracle returns before it)
        for k in ("to_pixels.0.weight", "to_pixels.0.bias"):
            grads[k] = torch.zeros_like(sd[k])
    if tok is not None:
        grads["tokens"] = tok.grad
    return grads


def product_out(name, entry, module, device, tokens_grad=True, ids=None, tokens=None):
    """The entry point on ``module`` (already on ``device``): (video, the tokens tensor or None)."""
    i0, t0 = inputs(name)
    dev = torch.device(device)
    if entry == "tokens":
        tok = (t0 if tokens is None else tokens).to(dev, copy=True).requires_grad_(tokens_grad)  # a fresh leaf per call
        return module.decode(tok), tok
    idx = (i0 if ids is None else ids).to(dev)
    return module.decode_from_codebook_indices(idx.reshape(idx.shape[0], -1)), None


def product_grads(name, entry, module, device, precision=L.PREC_F32):
    """{parameter name | "tokens": gradient on the CPU, or None} of (video * G).sum().backward() on the product."""
    module.precision = precision
    module.zero_grad(set_to_none=True)
    out, tok = product_out(name, entry, module, device)
    (out * upstream_weights(name, entry, out.shape).to(out.device, torch.float32)).sum().backward()
    grads = {k: None if p.grad is None else p.grad.detach().to("cpu", copy=True) for k, p in module.named_parameters()}
    if tok is not None:
        grads["tokens"] = None if tok.grad is None else tok.grad.detach().cpu()
    module.zero_grad(set_to_none=True)
    return grads


def _is_zero(k):
    return k in ANALYTICALLY_ZERO


def assert_same_none_set(name, grads, ref):
    got = {k for k, g in grads.items() if g is None}
    want = {k for k in grads if k not in ref}
    assert got == want, f"{name}: gradients left None {sorted(got)}, the reference leaves None {sorted(want)}"


# ---- check bodies ---------------------------------------------------------------------------------------------------

def check_fp32(device, sync, module, name, entry, precision=L.PREC_F32):
    """Every gradient tensor and d(tokens) within 1e-4 of its largest entry (max norm) and 2e-5 (relative Frobenius norm)
    of the fp64 reference; the None set equals the reference's.  Returns the worst max error / max|ref|."""
    ref = reference(name, entry)
    grads = product_grads(name, entry, module, device, precision)
    sync()
    assert_same_none_set(name, grads, ref)
    top = max(float(g.abs().max()) for g in ref.values() if g.numel())
    worst, failures = 0.0, []
    for k, got in grads.items():
        want = ref.get(k)
        if want is None or want.numel() == 0:
            continue
        assert got.shape == want.shape, k
        err = (got.double() - want).abs().max().item()
        if _is_zero(k):
            if err > 1e-6 * top:
                failures.append(f"{k}: |got - ref| {err:.3e} above 1e-6 x the largest gradient {top:.3e}")
            continue
        scale = want.abs().max().item()
        if scale == 0.0:  # (to_pixels with one latent frame)
            if err != 0.0:
                failures.append(f"{k}: {err:.3e} where the reference is exactly zero")
            continue
        fro = ((got.double() - want).norm() / want.norm()).item()
        worst = max(worst, err / scale)
        if err > 1e-4 * scale or fro > 2e-5:
            failures.append(f"{k}: max err / max|ref| {err / scale:.3e}, relative Frobenius error {fro:.3e}")
    assert not failures, f"{name}/{entry} (fp32):\n  " + "\n  ".join(failures)
    return worst


def check_bf16(device, sync, module, name, entry):
    """bf16 mode, at the bf16 bars of the training step: every tensor within 5 % of its largest entry at a cosine
    similarity of at least 0.995, and a worst error above 1e-5 (the tensor-core products were used)."""
    ref = reference(name, entry)
    grads = product_grads(name, entry, module, device, precision=L.PREC_BF16)
    sync()
    assert_same_none_set(name, grads, ref)
    top = max(float(g.abs().max()) for g in ref.values() if g.numel())
    worst, failures = 0.0, []
    for k, g in grads.items():
        r = ref.get(k)
        if g is None or r.numel() == 0:
            continue
        err = (g.double() - r).abs().max().item()
        if _is_zero(k):
            if err > 5e-2 * top:
                failures.append(f"{k}: |got - ref| {err:.3e} above 5e-2 x the largest gradient {top:.3e}")
            continue
        scale = r.abs().max().item()
        if scale == 0.0:
            continue
        cos = F.cosine_similarity(g.double().flatten(), r.flatten(), dim=0).item()
        worst = max(worst, err / scale)
        if err > 5e-2 * scale or cos < 0.995:
            failures.append(f"{k}: max err / max|ref| {err / scale:.3e}, cosine {cos:.5f}")
    assert not failures, f"{name}/{entry} (bf16):\n  " + "\n  ".join(failures)
    assert worst > 1e-5, f"{name}: bf16 mode gave fp32-exact gradients: the tensor-core products were not used"
    return worst


def check_forward_unchanged(device, sync, module, name, entry):
    """With grad enabled the decode returns bit-identical values and a graph; under no_grad, or when nothing requires
    grad, no graph is built; forward(return_recons_only=True) returns no graph."""
    module.precision = L.PREC_F32
    with torch.no_grad():
        plain, _ = product_out(name, entry, module, device)
    graphed, _ = product_out(name, entry, module, device)
    sync()
    assert plain.grad_fn is None and not plain.requires_grad
    assert graphed.grad_fn is not None
    assert torch.equal(plain, graphed.detach())
    for p in module.parameters():
        p.requires_grad_(False)
    try:
        frozen, _ = product_out(name, entry, module, device, tokens_grad=False)
        assert frozen.grad_fn is None and not frozen.requires_grad
    finally:
        for p in module.parameters():
            p.requires_grad_(True)
    ctor = CASES[name][0]
    ih, iw = module.image_size
    frames = 1 + (CASES[name][3] - 1) * module.temporal_patch_size
    video = torch.randn((1, module.channels, frames, ih, iw), generator=torch.Generator().manual_seed(5)).to(device)
    rec = module(video, return_recons_only=True)
    assert rec.grad_fn is None and not rec.requires_grad, ctor


def kernel_sequences(cases, device="cuda:0"):
    """{"name/entry/precision": (device ops of the no_grad decode, device ops of the decode with grad enabled)}: the
    kernel names of one call each in a torch.profiler trace, after a warm-up call of both (position-bias cache,
    workspace).  ``cases``: (name, entry, precision) triples."""
    from torch.profiler import ProfilerActivity, profile

    def device_ops(fn):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        ops = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        return [e.name for e in sorted(ops, key=lambda e: e.time_range.start)]

    out, modules = {}, {}
    for name, entry, precision in cases:
        module = modules.setdefault(name, build_module(name).to(device))
        module.precision = precision

        def plain():
            with torch.no_grad():
                product_out(name, entry, module, device)

        def graphed():
            product_out(name, entry, module, device)

        plain(), graphed()
        out[f"{name}/{entry}/{precision}"] = (device_ops(plain), device_ops(graphed))
    return out


def check_two_decodes_then_one_backward(device, sync, module, name, entry):
    """Two pending graphs of the same module, one backward through both, add up to the two backwards run apart (up to
    the order of atomic adds: 1e-6 of the largest gradient)."""
    module.precision = L.PREC_F32
    ids, tokens = inputs(name)
    second = dict(ids=torch.flip(ids, dims=(1,))) if entry == "ids" else dict(tokens=-tokens.flip(1))
    module.zero_grad(set_to_none=True)
    o1, _ = product_out(name, entry, module, device)
    o2, _ = product_out(name, entry, module, device, **second)
    (o1.square().sum() * 0.5 + o2.sum()).backward()
    together = {k: p.grad.detach().clone() for k, p in module.named_parameters() if p.grad is not None}
    module.zero_grad(set_to_none=True)
    o1, _ = product_out(name, entry, module, device)
    (o1.square().sum() * 0.5).backward()
    o2, _ = product_out(name, entry, module, device, **second)
    o2.sum().backward()
    apart = {k: p.grad.detach().clone() for k, p in module.named_parameters() if p.grad is not None}
    module.zero_grad(set_to_none=True)
    sync()
    assert together.keys() == apart.keys() and together
    top = max(float(g.abs().max()) for g in apart.values() if g.numel())
    for k, g in apart.items():
        if g.numel():
            diff = float((together[k] - g).abs().max())
            assert diff <= 1e-6 * top, f"{name} {k}: together vs apart differ by {diff:.3e} (largest {top:.3e})"


def check_deterministic(device, sync, module, name, entry):
    """The same backward twice: gradients differ only by the order of their atomic adds (1e-6 of the largest)."""
    a = product_grads(name, entry, module, device)
    b = product_grads(name, entry, module, device)
    sync()
    top = max(float(g.abs().max()) for g in a.values() if g is not None and g.numel())
    for k, g in a.items():
        assert (g is None) == (b[k] is None), k
        if g is not None and g.numel():
            diff = float((g - b[k]).abs().max())
            assert diff <= 1e-6 * top, f"{name} {k}: runs differ by {diff:.3e} (largest {top:.3e})"


def check_create_graph_refused(device, sync, module, name, entry):
    module.precision = L.PREC_F32
    out, _ = product_out(name, entry, module, device)
    params = [p for p in module.parameters() if p.requires_grad]
    try:
        torch.autograd.grad(out.sum(), params, create_graph=True, allow_unused=True)
    except RuntimeError as ex:
        assert "create_graph" in str(ex)
    else:
        raise AssertionError("create_graph=True was accepted")


def check_modified_weight_refused(device, sync, module, name, entry):
    module.precision = L.PREC_F32
    out, _ = product_out(name, entry, module, device)
    with torch.no_grad():
        module.to_pixels_first_frame[0].weight.mul_(1.5)
    try:
        out.sum().backward()
    except RuntimeError as ex:
        assert "modified" in str(ex)
    else:
        raise AssertionError("a weight modified between the decode and the backward was accepted")
    finally:
        module.zero_grad(set_to_none=True)
