"""Check bodies of the C-ViViT reconstruction-loss tests, shared by the H100 file (tests/test_gpu_recon_loss.py) and the
CPU executor file (tests/test_recon_loss_emulated_cpu.py): every body takes (device, sync).

A case is a C-ViViT configuration (tests/cases.py CVIVIT_CASES, or the configs[1]/[4] shape) with a seeded video and
optionally a frame mask.  The product computes ``loss = cvivit(video, mask=...); loss.backward()`` through
phk_cvivit_backward; the reference is ``cvivit_recon_loss`` below in float64 under torch autograd on the module's state
dict, with q taken from the product's ids (``codes_from_ids``), so that both differentiate the same function even where a
projection sits at zero.  Checks that assert the ids themselves say so."""
import functools

import torch
import torch.nn.functional as F

from oracle import phenaki_oracle as O
import phenaki_pytorch_b200 as P
from phenaki_pytorch_b200 import _lib as L
from tests import cases as CS
from tests.decode_grad_cases import AT_SIZE, ANALYTICALLY_ZERO

# name -> (ctor, module seed, video shape, frame mask rows or None)
CASES = {
    "cfg1": (CS.CVIVIT_CASES["cfg1"]["ctor"], 0, (1, 3, 5, 64, 64), None),
    "rect": (CS.CVIVIT_CASES["rect"]["ctor"], 3, (2, 3, 7, 32, 48), None),
    "rect_mask": (CS.CVIVIT_CASES["rect"]["ctor"], 3, (2, 3, 7, 32, 48), [[1, 1, 1, 1, 0, 0, 0], [1] * 7]),
    "image": (CS.CVIVIT_CASES["image"]["ctor"], 5, (3, 1, 32, 32), None),
    "at_size": (AT_SIZE, 11, (2, 3, 17, 256, 256), None),
}
SMALL = ["cfg1", "rect", "rect_mask", "image"]
ENCODER_PREFIXES = ("to_patch_emb", "enc_", "vq.project_in")


def cvivit_recon_loss(video, sd, image_size, patch_size, mask=None, training=True, codes_from_ids=None):
    """The reference's ``CViViT.forward(video, mask)`` with use_vgg_and_gan=False (cvivit.py:518-598) composed from the
    oracle, with upstream LFQ's training-mode straight-through estimator ``x + (q - x).detach()``: (loss, recon).
    ``codes_from_ids``: (b, t, h, w) ids whose +-1 codes replace sign(x) for q."""
    if video.ndim == 4:
        video = video.unsqueeze(2)
    b, c, f = video.shape[:3]
    dim, heads, pt, channels = O.cvivit_geometry(sd, image_size, patch_size)
    tokens = O.cvivit_encode_tokens(O.cvivit_patch_embed(video, sd, patch_size, pt), sd, heads)
    _, t, h, w, d = tokens.shape
    x = O.lfq_project(tokens.reshape(b, t * h * w, d), sd)
    if codes_from_ids is None:
        q = torch.where(x > 0, 1.0, -1.0).to(x.dtype)
    else:
        bits = (codes_from_ids.reshape(b, -1)[..., None].int() & sd["vq.mask"].int()) != 0
        q = torch.where(bits, 1.0, -1.0).to(x.dtype)
    if training:
        q = x + (q - x).detach()
    codes = F.linear(q, sd["vq.project_out.weight"], sd["vq.project_out.bias"]).reshape(b, t, h, w, d)
    recon = O.cvivit_decode(codes, sd, patch_size, pt, heads, channels)
    if mask is None:
        return F.mse_loss(video, recon), recon
    sq = F.mse_loss(video, recon, reduction="none")
    return sq[mask[:, None, :].expand(b, c, f)].mean(), recon


def build_module(name):
    ctor, seed, _, _ = CASES[name]
    torch.manual_seed(seed)
    return P.CViViT(**ctor)


@functools.lru_cache(maxsize=None)
def inputs(name):
    """Seeded video and frame mask (bool (b, f) or None) of the case."""
    _, seed, shape, mask = CASES[name]
    video = torch.randn(shape, generator=torch.Generator().manual_seed(3000 + seed))
    return video, None if mask is None else torch.tensor(mask, dtype=torch.bool)


def upstream_weights(name, shape):
    return torch.randn(shape, generator=torch.Generator().manual_seed(4000 + sorted(CASES).index(name)),
                       dtype=torch.float64)


def _objective(loss, recon, G):
    """a loss + (recon G).sum(), the return_recons objective (G None: the loss alone)."""
    return loss if G is None else 0.75 * loss + (recon * G).sum()


@functools.lru_cache(maxsize=None)
def reference(name, training, ids_key, with_recon):
    """(loss, {parameter name | "video": gradient}) by float64 oracle autograd on the CPU, q from the product ids
    registered under ``ids_key``; what the reference leaves without a gradient is absent."""
    module = build_module(name)
    ids = _IDS[ids_key]
    video, mask = inputs(name)
    params = dict(module.named_parameters())
    sd = {}
    for k, v in module.state_dict().items():
        v = v.detach().to(torch.float64) if v.is_floating_point() else v.detach()
        sd[k] = v.requires_grad_(True) if k in params else v
    vid = video.to(torch.float64).requires_grad_(True)
    loss, recon = cvivit_recon_loss(vid, sd, module.image_size, module.patch_size, mask, training, codes_from_ids=ids)
    if video.ndim == 4:
        recon = recon.squeeze(2)
    _objective(loss, recon, upstream_weights(name, recon.shape) if with_recon else None).backward()
    grads = {k: sd[k].grad for k in params if sd[k].grad is not None}
    if ids.shape[1] == 1:  # the reference runs to_patch_emb / to_pixels on empty batches: zero gradients
        for k in ("to_pixels.0.weight", "to_pixels.0.bias") + (tuple(k for k in params if k.startswith("to_patch_emb."))
                                                                 if training else ()):
            grads[k] = torch.zeros_like(sd[k])
    for k, p in params.items():  # self-attention null_kv (heads, 0, dim_head): autograd hands it an empty gradient
        if p.numel() == 0 and (training or not k.startswith(ENCODER_PREFIXES)):
            grads[k] = torch.zeros_like(sd[k])
    grads["video"] = vid.grad
    return float(loss), grads


_IDS = {}


def product_run(name, module, device, precision=L.PREC_F32, training=True, with_recon=False):
    """(loss, {parameter name | "video": gradient on the CPU, or None}, ids key) of the product's objective."""
    module.precision = precision
    module.train(training)
    module.zero_grad(set_to_none=True)
    video, mask = inputs(name)
    dev = torch.device(device)
    ids = module(video.to(dev), return_only_codebook_ids=True).cpu()
    key = (name, ids.numpy().tobytes())
    _IDS[key] = ids
    vid = video.to(dev, copy=True).requires_grad_(True)
    m = None if mask is None else mask.to(dev)
    if with_recon:
        loss, recon = module(vid, mask=m, return_recons=True)
        _objective(loss, recon, upstream_weights(name, recon.shape).to(dev, torch.float32)).backward()
    else:
        loss = module(vid, mask=m)
        loss.backward()
    grads = {k: None if p.grad is None else p.grad.detach().to("cpu", copy=True) for k, p in module.named_parameters()}
    grads["video"] = None if vid.grad is None else vid.grad.detach().cpu()
    module.zero_grad(set_to_none=True)
    return float(loss.detach()), grads, key


def assert_same_none_set(name, grads, ref):
    got = {k for k, g in grads.items() if g is None}
    want = {k for k in grads if k not in ref}
    assert got == want, f"{name}: gradients left None {sorted(got)}, the reference leaves None {sorted(want)}"


# ---- check bodies ---------------------------------------------------------------------------------------------------

def check_fp32(device, sync, module, name, precision=L.PREC_F32, training=True, with_recon=False):
    """The loss within 1e-6 relative; every gradient tensor and d video within 1e-4 of its largest entry (max norm) and
    2e-5 (relative Frobenius norm) of the fp64 reference (split-bf16 mode: 1e-5 and 1e-4, see below); the None set equals the reference's.  Returns the worst
    max error / max|ref|."""
    loss, grads, key = product_run(name, module, device, precision, training, with_recon)
    sync()
    ref_loss, ref = reference(name, training, key, with_recon)
    # split-bf16 mode: the loss and the recon that d recon is formed from are the split-bf16 inference forward's,
    # fp32-grade rather than fp32-exact; at the configs[1] shape that moves the gradients by ~3e-5 (relative Frobenius)
    loss_rtol, fro_bar = (1e-6, 2e-5) if precision == L.PREC_F32 else (1e-5, 1e-4)
    assert abs(loss - ref_loss) <= loss_rtol * abs(ref_loss), f"{name}: loss {loss!r}, reference {ref_loss!r}"
    assert_same_none_set(name, grads, ref)
    top = max(float(g.abs().max()) for g in ref.values() if g.numel())
    worst, failures = 0.0, []
    for k, got in grads.items():
        want = ref.get(k)
        if want is None or want.numel() == 0:
            continue
        assert got.shape == want.shape, k
        err = (got.double() - want).abs().max().item()
        if k in ANALYTICALLY_ZERO:
            if err > 1e-6 * top:
                failures.append(f"{k}: |got - ref| {err:.3e} above 1e-6 x the largest gradient {top:.3e}")
            continue
        scale = want.abs().max().item()
        if scale == 0.0:
            if err != 0.0:
                failures.append(f"{k}: {err:.3e} where the reference is exactly zero")
            continue
        fro = ((got.double() - want).norm() / want.norm()).item()
        worst = max(worst, err / scale)
        if err > 1e-4 * scale or fro > fro_bar:
            failures.append(f"{k}: max err / max|ref| {err / scale:.3e}, relative Frobenius error {fro:.3e}")
    assert not failures, f"{name} (fp32, training={training}):\n  " + "\n  ".join(failures)
    return worst


def check_bf16(device, sync, module, name):
    """bf16 mode at the training step's bf16 bars: every tensor within 5 % of its largest entry at a cosine similarity of
    at least 0.995, and a worst error above 1e-5 (the tensor-core products were used)."""
    _, grads, key = product_run(name, module, device, L.PREC_BF16)
    sync()
    _, ref = reference(name, True, key, False)
    assert_same_none_set(name, grads, ref)
    top = max(float(g.abs().max()) for g in ref.values() if g.numel())
    worst, failures = 0.0, []
    for k, g in grads.items():
        r = ref.get(k)
        if g is None or r.numel() == 0:
            continue
        err = (g.double() - r).abs().max().item()
        if k in ANALYTICALLY_ZERO:
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
    assert not failures, f"{name} (bf16):\n  " + "\n  ".join(failures)
    assert worst > 1e-5, f"{name}: bf16 mode gave fp32-exact gradients: the tensor-core products were not used"
    return worst


def check_forward_outputs(device, sync, module, name):
    """The loss forward's ids equal return_only_codebook_ids; recon is bit-identical to return_recons_only=True and
    carries a graph; the loss equals the masked MSE of that recon in float64 (1e-6 relative) and is bit-identical
    between two calls; return_recons_only still returns no graph."""
    module.precision = L.PREC_F32
    module.train(True)
    video, mask = inputs(name)
    dev = torch.device(device)
    v = video.to(dev)
    m = None if mask is None else mask.to(dev)
    ids = module(v, return_only_codebook_ids=True)
    v5 = v.unsqueeze(2) if v.ndim == 4 else v
    fwd_ids = module._recon_forward(v5, None if m is None else m.to(torch.uint8))[0]
    only = module(v, return_recons_only=True)
    loss, recon = module(v, mask=m, return_recons=True)
    loss2 = module(v, mask=m)
    sync()
    assert torch.equal(fwd_ids.cpu(), ids.cpu())
    assert only.grad_fn is None and not only.requires_grad
    assert recon.grad_fn is not None and loss.grad_fn is not None
    assert torch.equal(recon.detach().cpu(), only.cpu())
    assert torch.equal(loss.detach().cpu(), loss2.detach().cpu())
    r, x = recon.detach().cpu().double(), video.double()
    if r.ndim == 4:
        r, x = r.unsqueeze(2), x.unsqueeze(2)
    sq = (r - x).square()
    want = sq.mean() if mask is None else sq[mask[:, None, :].expand(*sq.shape[:3])].mean()
    assert abs(float(loss) - float(want)) <= 1e-6 * abs(float(want)), (float(loss), float(want))
    with torch.no_grad():
        plain = module(v, mask=m)
    assert plain.grad_fn is None and torch.equal(plain.cpu(), loss.detach().cpu())


def check_two_forwards_then_one_backward(device, sync, module, name):
    """Two pending graphs of the same module, one backward through both, add up to the two backwards run apart (up to
    the order of atomic adds: 1e-6 of the largest gradient)."""
    module.precision = L.PREC_F32
    module.train(True)
    video, _ = inputs(name)
    v1, v2 = video.to(device), (-video.flip(-1)).to(device)
    module.zero_grad(set_to_none=True)
    (module(v1) * 0.5 + module(v2)).backward()
    together = {k: p.grad.detach().clone() for k, p in module.named_parameters() if p.grad is not None}
    module.zero_grad(set_to_none=True)
    (module(v1) * 0.5).backward()
    module(v2).backward()
    apart = {k: p.grad.detach().clone() for k, p in module.named_parameters() if p.grad is not None}
    module.zero_grad(set_to_none=True)
    sync()
    assert together.keys() == apart.keys() and together
    top = max(float(g.abs().max()) for g in apart.values() if g.numel())
    for k, g in apart.items():
        if g.numel():
            diff = float((together[k] - g).abs().max())
            assert diff <= 1e-6 * top, f"{name} {k}: together vs apart differ by {diff:.3e} (largest {top:.3e})"


def check_deterministic(device, sync, module, name):
    """The same backward twice: gradients differ only by the order of their atomic adds (1e-6 of the largest); the
    losses are bit-identical."""
    la, a, _ = product_run(name, module, device)
    lb, b, _ = product_run(name, module, device)
    sync()
    assert la == lb
    top = max(float(g.abs().max()) for g in a.values() if g is not None and g.numel())
    for k, g in a.items():
        assert (g is None) == (b[k] is None), k
        if g is not None and g.numel():
            diff = float((g - b[k]).abs().max())
            assert diff <= 1e-6 * top, f"{name} {k}: runs differ by {diff:.3e} (largest {top:.3e})"


def check_cpu_rng_draw(device, sync, module, name):
    """The forward leaves the CPU generator where the reference's does: it draws torch.randn(b, f) once."""
    module.precision = L.PREC_F32
    video, mask = inputs(name)
    v = video.to(device)
    torch.manual_seed(123)
    module(v, mask=None if mask is None else mask.to(device))
    got = torch.randn(4)
    torch.manual_seed(123)
    f = 1 if video.ndim == 4 else video.shape[2]
    torch.randn(video.shape[0], f)
    assert torch.equal(got, torch.randn(4))


def _refused(fn, words):
    try:
        fn()
    except (RuntimeError, NotImplementedError) as ex:
        assert any(w in str(ex) for w in words), str(ex)
    else:
        raise AssertionError("accepted")


def check_refusals(device, sync, module, name):
    """create_graph=True, a weight modified between forward and backward, a cosine-sim tokenizer, a training-mode module
    with dropout, use_vgg_and_gan=True and return_discr_loss=True raise; the forward refusals launch nothing."""
    module.precision = L.PREC_F32
    module.train(True)
    video, _ = inputs(name)
    v = video.to(device)
    loss = module(v)
    params = [p for p in module.parameters() if p.requires_grad]
    _refused(lambda: torch.autograd.grad(loss, params, create_graph=True, allow_unused=True), ["create_graph"])
    loss = module(v)
    with torch.no_grad():
        module.enc_spatial_transformer.norm_out.gamma.mul_(1.5)
    _refused(loss.backward, ["modified"])
    module.zero_grad(set_to_none=True)
    before = L.lib().phk_launch_count()
    _refused(lambda: module(v, return_discr_loss=True), ["GAN"])
    ctor = dict(CASES[name][0])
    for extra, words in ((dict(lookup_free_quantization=False), ["lookup_free_quantization"]),
                         (dict(ff_dropout=0.1), ["dropout"]), (dict(attn_dropout=0.1), ["dropout"]),
                         (dict(use_vgg_and_gan=True), ["GAN"])):
        other = P.CViViT(**{**ctor, **extra}).to(device)
        _refused(lambda: other(v), words)
    assert L.lib().phk_launch_count() == before, "a refused forward launched kernels"
    dropout = P.CViViT(**{**ctor, "ff_dropout": 0.1}).to(device).eval()  # eval mode applies no dropout: accepted
    dropout(v).backward()
