"""Check bodies of the differentiable ``CViViT.encode(tokens)`` tests, shared by the H100 file
(tests/test_gpu_zz_encode_backward.py) and the CPU executor file (tests/test_encode_backward_emulated_cpu.py): every body
takes (device, sync).

A case is a C-ViViT configuration of tests/decode_grad_cases.py (the goldens' configurations and the configs[1] encoder
shape) with seeded patch tokens (b, T', h, w, dim).  The product computes ``(cvivit.encode(tokens) * G).sum().backward()``
for a seeded random G through phk_cvivit_encode_backward; the reference is the float64 oracle
(``oracle.cvivit_encode_tokens``) on the module's state dict under torch autograd."""
import ctypes as C
import functools

import torch
import torch.nn.functional as F

from oracle import phenaki_oracle as O
from phenaki_pytorch_b200 import _lib as L
from phenaki_pytorch_b200.modules import GradKeep
from tests import decode_grad_cases as DG

CASES = DG.CASES  # name -> (ctor, seed, batch, T'): cfg1, rect, image (T' = 1), cosine_vq, at_size (B = 2, T' = 9)
SMALL = DG.SMALL
build_module = DG.build_module
ANALYTICALLY_ZERO = DG.ANALYTICALLY_ZERO
PHK_E_WORKSPACE = -4


@functools.lru_cache(maxsize=None)
def inputs(name):
    """Seeded patch tokens (b, T', h, w, dim) of the case."""
    ctor, seed, b, tp = CASES[name]
    module = build_module(name)
    h, w = module.patch_height_width
    g = torch.Generator().manual_seed(3000 + seed)
    return torch.randn((b, tp, h, w, ctor["dim"]), generator=g)


def upstream_weights(name, shape, what="encode"):
    g = torch.Generator().manual_seed(4000 + sorted(CASES).index(name) * 2 + (what != "encode"))
    return torch.randn(shape, generator=g, dtype=torch.float64)


def _fp64_state(module):
    params = dict(module.named_parameters())
    sd = {}
    for k, v in module.state_dict().items():
        v = v.detach().to(torch.float64) if v.is_floating_point() else v.detach()
        sd[k] = v.requires_grad_(True) if k in params else v
    return params, sd


@functools.lru_cache(maxsize=None)
def reference(name, then_decode=False):
    """{parameter name | "tokens": gradient} of (encode(tokens) * G).sum(), or with ``then_decode`` of
    (decode(encode(tokens)) * G).sum(), by oracle autograd in float64 on the CPU; what the reference leaves without a
    gradient is absent."""
    module = build_module(name)
    params, sd = _fp64_state(module)
    tok = inputs(name).to(torch.float64).requires_grad_(True)
    out = O.cvivit_encode_tokens(tok, sd, module.heads)
    if then_decode:
        out = O.cvivit_decode(out, sd, module.patch_size, module.temporal_patch_size, module.heads, module.channels)
    (out * upstream_weights(name, out.shape, "decode" if then_decode else "encode")).sum().backward()
    grads = {k: sd[k].grad for k in params if sd[k].grad is not None}
    if then_decode and tok.shape[1] == 1:  # the reference runs to_pixels on an empty batch: zero gradients
        for k in ("to_pixels.0.weight", "to_pixels.0.bias"):
            grads[k] = torch.zeros_like(sd[k])
    grads["tokens"] = tok.grad
    return grads


def product_out(name, module, device, tokens_grad=True, tokens=None):
    """``module.encode`` on the case's tokens (a fresh leaf per call): (out, tokens)."""
    tok = (inputs(name) if tokens is None else tokens).to(torch.device(device), copy=True).requires_grad_(tokens_grad)
    return module.encode(tok), tok


def product_grads(name, module, device, precision=L.PREC_F32, then_decode=False):
    """{parameter name | "tokens": gradient on the CPU, or None} of the objective's backward on the product."""
    module.precision = precision
    module.zero_grad(set_to_none=True)
    out, tok = product_out(name, module, device)
    if then_decode:
        out = module.decode(out)
    G = upstream_weights(name, out.shape, "decode" if then_decode else "encode").to(out.device, torch.float32)
    (out * G).sum().backward()
    grads = {k: None if p.grad is None else p.grad.detach().to("cpu", copy=True) for k, p in module.named_parameters()}
    grads["tokens"] = None if tok.grad is None else tok.grad.detach().cpu()
    module.zero_grad(set_to_none=True)
    return grads


def assert_same_none_set(label, grads, ref):
    got = {k for k, g in grads.items() if g is None}
    want = {k for k in grads if k not in ref}
    assert got == want, f"{label}: gradients left None {sorted(got)}, the reference leaves None {sorted(want)}"


def _max_close(a, b, rel, label):
    """Same keys and None pattern; every tensor within rel x the largest entry of all of them."""
    assert a.keys() == b.keys(), label
    top = max(float(g.abs().max()) for g in b.values() if g is not None and g.numel())
    for k, g in a.items():
        assert (g is None) == (b[k] is None), f"{label} {k}"
        if g is not None and g.numel():
            diff = float((g - b[k]).abs().max())
            assert diff <= rel * top, f"{label} {k}: differ by {diff:.3e} (largest {top:.3e})"


# ---- check bodies ---------------------------------------------------------------------------------------------------

def check_fp32(device, sync, module, name, precision=L.PREC_F32, then_decode=False):
    """Every gradient tensor and d(tokens) within 1e-4 of its largest entry (max norm) and 2e-5 (relative Frobenius norm)
    of the fp64 reference; the analytically zero position-bias bias within 1e-6 of the largest gradient; the None set
    equals the reference's.  Returns the worst max error / max|ref|."""
    ref = reference(name, then_decode)
    grads = product_grads(name, module, device, precision, then_decode)
    sync()
    label = f"{name}{' then decode' if then_decode else ''}"
    assert_same_none_set(label, grads, ref)
    assert grads["tokens"] is not None
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
        if scale == 0.0:  # (to_pixels with one latent frame)
            if err != 0.0:
                failures.append(f"{k}: {err:.3e} where the reference is exactly zero")
            continue
        fro = ((got.double() - want).norm() / want.norm()).item()
        worst = max(worst, err / scale)
        if err > 1e-4 * scale or fro > 2e-5:
            failures.append(f"{k}: max err / max|ref| {err / scale:.3e}, relative Frobenius error {fro:.3e}")
    assert not failures, f"{label} (fp32):\n  " + "\n  ".join(failures)
    return worst


def check_encoder_grads_only(device, sync, module, name):
    """The gradients reach the encoder stacks, the position-bias MLP and the tokens; every other parameter stays None."""
    grads = product_grads(name, module, device)
    sync()
    reached = ("enc_spatial_transformer.", "enc_temporal_transformer.", "spatial_rel_pos_bias.net.")
    for k, g in grads.items():
        if k == "tokens":
            assert g is not None
        elif not k.startswith(reached):
            assert g is None, f"{k} got a gradient from encode"
    assert any(g is not None for k, g in grads.items() if k.startswith(reached[2]))


def check_split_bf16_equals_fp32(device, sync, module, name):
    """Split-bf16 mode differentiates in fp32 from the tokens: its gradients equal fp32 mode's up to the order of atomic
    adds (1e-6 of the largest entry)."""
    a = product_grads(name, module, device, L.PREC_F32)
    b = product_grads(name, module, device, L.PREC_BF16X3)
    sync()
    _max_close(b, a, 1e-6, f"{name} split-bf16 vs fp32")


def check_bf16(device, sync, module, name):
    """bf16 mode, at the training step's bf16 bars: every tensor within 5 % of its largest entry at a cosine similarity of
    at least 0.995, and a worst error above 1e-5 (the tensor-core products ran)."""
    ref = reference(name)
    grads = product_grads(name, module, device, precision=L.PREC_BF16)
    sync()
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
        cos = F.cosine_similarity(g.double().flatten(), r.flatten(), dim=0).item()
        worst = max(worst, err / scale)
        if err > 5e-2 * scale or cos < 0.995:
            failures.append(f"{k}: max err / max|ref| {err / scale:.3e}, cosine {cos:.5f}")
    assert not failures, f"{name} (bf16):\n  " + "\n  ".join(failures)
    assert worst > 1e-5, f"{name}: bf16 mode gave fp32-exact gradients: the tensor-core products were not used"
    return worst


def check_forward_unchanged(device, sync, module, name, precision=L.PREC_F32):
    """With grad enabled the encode returns bit-identical values and a graph; under no_grad, or when nothing requires
    grad, no graph is built."""
    module.precision = precision
    with torch.no_grad():
        plain, _ = product_out(name, module, device)
    graphed, _ = product_out(name, module, device)
    sync()
    assert plain.grad_fn is None and not plain.requires_grad
    assert graphed.grad_fn is not None
    assert plain.shape == graphed.shape == inputs(name).shape and plain.dtype == torch.float32
    assert torch.equal(plain, graphed.detach())
    for p in module.parameters():
        p.requires_grad_(False)
    try:
        frozen, _ = product_out(name, module, device, tokens_grad=False)
        assert frozen.grad_fn is None and not frozen.requires_grad
        assert torch.equal(plain, frozen)
    finally:
        for p in module.parameters():
            p.requires_grad_(True)


def kernel_sequences(cases, device="cuda:0"):
    """{"name/precision": (device ops of the no_grad encode, device ops of the encode with grad enabled)}: the kernel
    names of one call each in a torch.profiler trace, after a warm-up call of both.  ``cases``: (name, precision) pairs."""
    from torch.profiler import ProfilerActivity, profile

    def device_ops(fn):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        ops = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        return [e.name for e in sorted(ops, key=lambda e: e.time_range.start)]

    out, modules = {}, {}
    for name, precision in cases:
        module = modules.setdefault(name, build_module(name).to(device))
        module.precision = precision
        tok = inputs(name).to(device)
        leaf = tok.clone().requires_grad_(True)

        def plain():
            with torch.no_grad():
                module.encode(tok)

        def graphed():
            module.encode(leaf)

        plain(), graphed()
        out[f"{name}/{precision}"] = (device_ops(plain), device_ops(graphed))
    return out


def check_two_encodes_then_one_backward(device, sync, module, name):
    """Two pending graphs of the same module, one backward through both, add up to the two backwards run apart (up to
    the order of atomic adds: 1e-6 of the largest gradient)."""
    module.precision = L.PREC_F32
    second = dict(tokens=-inputs(name).flip(1))
    module.zero_grad(set_to_none=True)
    o1, t1 = product_out(name, module, device)
    o2, t2 = product_out(name, module, device, **second)
    (o1.square().sum() * 0.5 + o2.sum()).backward()
    together = {k: p.grad.detach().clone() for k, p in module.named_parameters() if p.grad is not None}
    together.update(t1=t1.grad.detach().clone(), t2=t2.grad.detach().clone())
    module.zero_grad(set_to_none=True)
    o1, t1 = product_out(name, module, device)
    (o1.square().sum() * 0.5).backward()
    o2, t2 = product_out(name, module, device, **second)
    o2.sum().backward()
    apart = {k: p.grad.detach().clone() for k, p in module.named_parameters() if p.grad is not None}
    apart.update(t1=t1.grad.detach().clone(), t2=t2.grad.detach().clone())
    module.zero_grad(set_to_none=True)
    sync()
    assert len(apart) > 2
    _max_close(together, apart, 1e-6, f"{name} together vs apart")


def check_deterministic(device, sync, module, name, precision=L.PREC_F32):
    """The same backward twice: gradients differ only by the order of their atomic adds (1e-6 of the largest)."""
    a = product_grads(name, module, device, precision)
    b = product_grads(name, module, device, precision)
    sync()
    _max_close(a, b, 1e-6, f"{name} run vs run")


def _launches():
    return L.lib().phk_launch_count()


def check_create_graph_refused(device, sync, module, name):
    module.precision = L.PREC_F32
    out, tok = product_out(name, module, device)
    params = [p for p in module.parameters() if p.requires_grad]
    sync()
    before = _launches()
    try:
        torch.autograd.grad(out.sum(), params + [tok], create_graph=True, allow_unused=True)
    except RuntimeError as ex:
        assert "create_graph" in str(ex)
    else:
        raise AssertionError("create_graph=True was accepted")
    assert _launches() == before, "a refused backward launched kernels"


def check_modified_weight_refused(device, sync, module, name):
    module.precision = L.PREC_F32
    out, _ = product_out(name, module, device)
    with torch.no_grad():
        module.enc_temporal_transformer.norm_out.gamma.mul_(1.5)
    sync()
    before = _launches()
    try:
        out.sum().backward()
    except RuntimeError as ex:
        assert "modified" in str(ex)
    else:
        raise AssertionError("a weight modified between the encode and the backward was accepted")
    finally:
        module.zero_grad(set_to_none=True)
    assert _launches() == before, "a refused backward launched kernels"


def check_bad_shapes_refused(device, sync, module, name):
    """Any other rank, h, w or dim fails an assertion before anything is launched."""
    module.precision = L.PREC_F32
    b, t, h, w, d = inputs(name).shape
    bad = [(b, t, h * w, d), (b, t, h + 1, w, d), (b, t, h, w + 1, d), (b, t, h, w, d + 4), (b, t, h, w, d, 1)]
    for shape in bad:
        x = torch.zeros(shape, device=torch.device(device), requires_grad=True)
        sync()
        before = _launches()
        try:
            module.encode(x)
        except AssertionError:
            pass
        else:
            raise AssertionError(f"tokens of shape {shape} were accepted")
        assert _launches() == before, f"tokens of shape {shape}: launched kernels before refusing"


def check_short_workspace_refused(device, sync, module, name):
    """Both entries, called through ctypes with one byte less than their *_workspace_bytes, return PHK_E_WORKSPACE and
    launch nothing."""
    lib = L.lib()
    dev = torch.device(device)
    module.precision = L.PREC_F32
    tok = inputs(name).to(dev)
    b, tp = tok.shape[:2]
    with torch.cuda.device(dev):
        table = module._table()
        bias = module._spatial_bias(table, dev)
        gk = GradKeep(module._encode_params())
        gtable = module._enc_grad_table(gk, False)
        out = torch.zeros_like(tok)
        need_f = lib.phk_cvivit_encode_tokens_workspace_bytes(C.byref(table), b, tp, L.PREC_F32)
        need_b = lib.phk_cvivit_encode_backward_workspace_bytes(C.byref(table), b, tp, L.PREC_F32)
        assert need_f > 0 and need_b > 0
        ws = torch.zeros(max(need_f, need_b), dtype=torch.uint8, device=dev)
        sync()
        before = _launches()
        rc = lib.phk_cvivit_encode_tokens(C.byref(table), L.ptr(tok), b, tp, L.ptr(out), L.ptr(ws), need_f - 1,
                                          L.PREC_F32, L.ptr(bias), L.stream_ptr())
        assert rc == PHK_E_WORKSPACE, rc
        rc = lib.phk_cvivit_encode_backward(C.byref(table), C.byref(gtable), L.ptr(tok), b, tp, L.ptr(tok), L.ptr(out),
                                            L.ptr(ws), need_b - 1, L.PREC_F32, L.stream_ptr())
        assert rc == PHK_E_WORKSPACE, rc
        sync()
        assert _launches() == before, "a refused call launched kernels"
        assert not out.any() and not gk.flat.any(), "a refused call wrote its outputs"
