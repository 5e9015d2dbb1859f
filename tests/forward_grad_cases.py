"""Check bodies of the differentiable-forward tests, shared by the H100 file (tests/test_gpu_forward_backward.py) and the
CPU executor file (tests/test_forward_backward_emulated_cpu.py): every body takes (lib, device, sync).

A case names a module and its inputs (a case of tests/train_at_size_cases.py, or a small one for the executor) and the
public forward it differentiates: MaskGit.forward (logits, ``return_embeds=True``, ``cond_drop_prob=1.0``, 4-D ids),
TokenCritic.forward, SelfCritic.forward, or their ``forward_with_cond_scale``.  The product computes
``(out * G).sum().backward()`` for a seeded random G through phk_maskgit_backward; the reference is the float64 oracle
(``oracle.maskgit_forward`` / ``critic_forward`` / ``with_cond_scale``) on the module's state dict under torch autograd,
with the text embeddings' gradient from the same graph (``"text_embeds"`` in the gradient dicts)."""
import functools

import torch
import torch.nn.functional as F

from oracle import phenaki_oracle as O
from phenaki_pytorch_b200 import _lib as L
from tests import train_at_size_cases as T

_SMALL = dict(dim=64, num_tokens=97, max_seq_len=64, heads=2, dim_head=64, depth=2, dim_context=40)
_SMALL_INPUTS = dict(batch=2, patch_shape=(2, 3, 4), ctx_len=5, ctx_valid=(5, 3), video_valid=(24, 19))
SMALL_MASKGIT = dict(kind="maskgit", seed=120, ctor=_SMALL, input_seed=121, **_SMALL_INPUTS)
SMALL_CRITIC = dict(kind="critic", seed=122, ctor=dict(_SMALL, has_cross_attn=True), input_seed=123, **_SMALL_INPUTS)
SMALL_CRITIC_NO_CROSS = dict(kind="critic", seed=124, input_seed=125, ctor=_SMALL, **_SMALL_INPUTS)
SMALL_SELF_CRITIC = dict(SMALL_MASKGIT, kind="self_critic", seed=126, input_seed=127)
# a TokenCritic at the ragged MaskGit's size without cross-attention (dim_context only shapes the unused text input)
RAGGED_CRITIC_NO_CROSS = dict(kind="critic", seed=128, input_seed=129, batch=3, patch_shape=(3, 7, 9), ctx_len=11,
                              ctx_valid=(11, 4, 7), video_valid=(189, 150, 123),
                              ctor=T.RAGGED_MASKGIT)

# call: "plain" | "cfg" (forward_with_cond_scale, cond_scale 3) ; options: return_embeds, cond_drop_prob, ids4d, precision
CASES = {
    "prod_logits": dict(base=T.CASES["prod_ce"], call="plain"),
    "prod_logits_cfg": dict(base=T.CASES["prod_ce"], call="cfg"),
    "ragged_logits": dict(base=T.CASES["ragged_ce"], call="plain"),
    "ragged_logits_cfg": dict(base=T.CASES["ragged_ce"], call="cfg"),
    "ragged_embeds": dict(base=T.CASES["ragged_ce"], call="plain", return_embeds=True),
    "ragged_embeds_cfg": dict(base=T.CASES["ragged_ce"], call="cfg", return_embeds=True),
    "ragged_cond_drop": dict(base=T.CASES["ragged_ce"], call="plain", cond_drop_prob=1.0),
    "ragged_ids4d": dict(base=T.CASES["ragged_ce"], call="plain", ids4d=True),
    "prod_critic": dict(base=T.CASES["prod_critic"], call="plain"),
    "prod_critic_cfg": dict(base=T.CASES["prod_critic"], call="cfg"),
    "ragged_critic_no_cross": dict(base=RAGGED_CRITIC_NO_CROSS, call="plain"),
    "ragged_critic_no_cross_cfg": dict(base=RAGGED_CRITIC_NO_CROSS, call="cfg"),
    "ragged_self_critic": dict(base=T.CASES["ragged_self_critic"], call="plain"),
    "ragged_self_critic_cfg": dict(base=T.CASES["ragged_self_critic"], call="cfg"),
    "ragged_logits_x3": dict(base=T.CASES["ragged_ce"], call="plain", precision=L.PREC_BF16X3),
}
BF16_CASES = ["prod_logits", "prod_logits_cfg", "ragged_logits", "ragged_logits_cfg"]

# small enough for the CPU executor of tests/cuda_emu; depth 2, so that d(text_embeds) sums over two layers
EMULATED_CASES = {
    "emu_logits": dict(base=SMALL_MASKGIT, call="plain"),
    "emu_logits_cfg": dict(base=SMALL_MASKGIT, call="cfg"),
    "emu_embeds": dict(base=SMALL_MASKGIT, call="plain", return_embeds=True),
    "emu_embeds_cfg": dict(base=SMALL_MASKGIT, call="cfg", return_embeds=True),
    "emu_cond_drop": dict(base=SMALL_MASKGIT, call="plain", cond_drop_prob=1.0),
    "emu_ids4d": dict(base=SMALL_MASKGIT, call="plain", ids4d=True),
    "emu_critic": dict(base=SMALL_CRITIC, call="plain"),
    "emu_critic_cfg": dict(base=SMALL_CRITIC, call="cfg"),
    "emu_critic_no_cross": dict(base=SMALL_CRITIC_NO_CROSS, call="plain"),
    "emu_critic_no_cross_cfg": dict(base=SMALL_CRITIC_NO_CROSS, call="cfg"),
    "emu_self_critic": dict(base=SMALL_SELF_CRITIC, call="plain"),
    "emu_self_critic_cfg": dict(base=SMALL_SELF_CRITIC, call="cfg"),
    "emu_logits_x3": dict(base=SMALL_MASKGIT, call="plain", precision=L.PREC_BF16X3),
}
ALL_CASES = {**CASES, **EMULATED_CASES}
COND_SCALE = 3.0


def _uses_context(base):
    return base["kind"] != "critic" or base["ctor"].get("has_cross_attn", False)


def network_input(base, x):
    """MaskGit reads the masked ids, the critics the sampled predictions at the masked positions."""
    if base["kind"] == "maskgit":
        return torch.where(x["token_mask"], base["ctor"]["num_tokens"], x["ids"])
    return torch.where(x["token_mask"], x["pred"], x["ids"])


def upstream_weights(name, shape):
    g = torch.Generator().manual_seed(1000 + sorted(ALL_CASES).index(name))
    return torch.randn(shape, generator=g, dtype=torch.float64)


@functools.lru_cache(maxsize=None)
def reference(name):
    """{"losses": {}, "grads": {parameter name | "text_embeds": gradient}} of (out * G).sum() by oracle autograd in
    float64 on the CPU; what the reference leaves without a gradient is absent."""
    case = ALL_CASES[name]
    base = case["base"]
    module = T.build_module(base)
    x = T.inputs(base)
    heads = base["ctor"].get("heads", 8)
    shape = base["patch_shape"]
    params = dict(module.named_parameters())
    sd = {}
    for k, v in module.state_dict().items():
        v = v.detach().to(torch.float64) if v.is_floating_point() else v.detach()
        sd[k] = v.requires_grad_(True) if k in params else v
    ctx = x["context"].to(torch.float64).requires_grad_(True) if _uses_context(base) else None
    ids = network_input(base, x)
    if case.get("ids4d"):
        ids = ids.reshape(ids.shape[0], *shape)
    kw = dict(video_patch_shape=shape, heads=heads, context=ctx, text_mask=x["text_mask"] if ctx is not None else None,
              video_mask=x["video_mask"])
    if base["kind"] == "maskgit":
        def fn(cond_drop):
            return O.maskgit_forward(ids, sd, cond_drop=cond_drop, return_embeds=case.get("return_embeds", False), **kw)
    elif base["kind"] == "critic":
        def fn(cond_drop):
            return O.critic_forward(ids, sd, cond_drop=cond_drop, **kw)
    else:
        msd = {k[len("maskgit."):]: v for k, v in sd.items() if k.startswith("maskgit.")}

        def fn(cond_drop):
            emb = O.maskgit_forward(ids, msd, cond_drop=cond_drop, return_embeds=True, **kw)
            return F.linear(emb, sd["to_pred.0.weight"], sd["to_pred.0.bias"]).squeeze(-1)
    if case["call"] == "cfg":
        out = O.with_cond_scale(fn, COND_SCALE)
    else:
        out = fn(case.get("cond_drop_prob", 0.0) >= 1.0)
    (out * upstream_weights(name, out.shape)).sum().backward()
    grads = {k: sd[k].grad for k in params if sd[k].grad is not None}
    if ctx is not None and ctx.grad is not None:
        grads["text_embeds"] = ctx.grad
    return {"losses": {}, "grads": grads}


def set_precision(module, precision):
    (module.maskgit if hasattr(module, "maskgit") else module).precision = precision


def product_out(name, module, device, context_grad=True, ids=None):
    """The case's public forward on ``module`` (already on ``device``): (output, the text embeddings tensor or None)."""
    case = ALL_CASES[name]
    base = case["base"]
    x = T.inputs(base)
    dev = torch.device(device)
    shape = base["patch_shape"]
    ids = network_input(base, x) if ids is None else ids
    ids = ids.to(dev)
    ctx = None
    kw = dict(video_mask=None if x["video_mask"] is None else x["video_mask"].to(dev))
    if _uses_context(base):
        ctx = x["context"].to(dev).requires_grad_(context_grad)
        kw.update(context=ctx, text_mask=x["text_mask"].to(dev))
    if case.get("ids4d"):
        ids = ids.reshape(ids.shape[0], *shape)
    else:
        kw["video_patch_shape"] = shape
    if base["kind"] == "maskgit":
        kw["return_embeds"] = case.get("return_embeds", False)
    if case["call"] == "cfg":
        return module.forward_with_cond_scale(ids, cond_scale=COND_SCALE, **kw), ctx
    if base["kind"] == "critic" or case.get("cond_drop_prob"):
        kw["cond_drop_prob"] = case.get("cond_drop_prob", 0.0)
    return module(ids, **kw), ctx


def product_grads(name, module, device, precision=None):
    """{parameter name | "text_embeds": gradient on the CPU, or None} of (out * G).sum().backward() on the product."""
    set_precision(module, ALL_CASES[name].get("precision", L.PREC_F32) if precision is None else precision)
    module.zero_grad(set_to_none=True)
    out, ctx = product_out(name, module, device)
    (out * upstream_weights(name, out.shape).to(out.device, torch.float32)).sum().backward()
    grads = {k: None if p.grad is None else p.grad.detach().to("cpu", copy=True) for k, p in module.named_parameters()}
    if ctx is not None:
        grads["text_embeds"] = None if ctx.grad is None else ctx.grad.detach().cpu()
    module.zero_grad(set_to_none=True)
    return grads


# ---- check bodies ---------------------------------------------------------------------------------------------------

def check_fp32(lib, device, sync, module, name):
    """Every gradient tensor and d(text_embeds) within 1e-4 of its largest entry (max norm) and 2e-5 (relative
    Frobenius norm) of the fp64 reference; the None set equals the reference's."""
    ref = reference(name)
    grads = product_grads(name, module, device)
    sync()
    assert_same_none_set(name, grads, ref)
    # exactly zero in the reference (cond_drop_prob=1.0: every text key is masked out, so the text path of the
    # cross-attention gets no gradient): held to the bar of the analytically zero tensors
    top = T.largest_gradient(ref)
    zero = {k for k, g in ref["grads"].items() if g.numel() and not bool(g.any())}
    for k in zero:
        err = float(grads[k].abs().max())
        assert err <= 1e-6 * top, f"{name} {k}: {err:.3e} where the reference is exactly zero (largest {top:.3e})"
    rest = {k: g for k, g in grads.items() if k not in zero}
    return T.check_fp32(name, {}, rest, {"losses": {}, "grads": {k: g for k, g in ref["grads"].items() if k not in zero}})


def assert_same_none_set(name, grads, ref):
    got = {k for k, g in grads.items() if g is None}
    want = {k for k in grads if k not in ref["grads"]}
    assert got == want, f"{name}: gradients left None {sorted(got)}, the reference leaves None {sorted(want)}"


def check_bf16(lib, device, sync, module, name):
    """bf16 mode, at the bf16 bars of the training step: every tensor within 5 % of its largest entry at a cosine
    similarity of at least 0.995, and a worst error above 1e-5 (the tensor-core products were used)."""
    ref = reference(name)
    grads = product_grads(name, module, device, precision=L.PREC_BF16)
    sync()
    assert_same_none_set(name, grads, ref)
    top = T.largest_gradient(ref)
    worst, failures = 0.0, []
    for k, g in grads.items():
        r = ref["grads"].get(k)
        if g is None or r.numel() == 0:
            continue
        err = (g.double() - r).abs().max().item()
        if T.is_analytically_zero(k):
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


def check_matches_train_step(lib, device, sync, module, base_name):
    """F.cross_entropy(maskgit(masked)[mask], ids[mask]).backward() and maskgit.train_step on the same draws give the
    same gradients to fp32 rounding: per tensor within 1e-5 of its largest entry plus 1e-6 of the largest gradient."""
    base = T.CASES[base_name] if isinstance(base_name, str) else base_name
    x = T.inputs(base)
    dev = torch.device(device)
    shape = base["patch_shape"]
    ids, tm = x["ids"].to(dev), x["token_mask"].to(dev)
    masked = torch.where(tm, base["ctor"]["num_tokens"], ids)
    kw = dict(context=x["context"].to(dev), text_mask=x["text_mask"].to(dev),
              video_mask=None if x["video_mask"] is None else x["video_mask"].to(dev))
    module.precision = L.PREC_F32
    module.zero_grad(set_to_none=True)
    logits = module(masked, video_patch_shape=shape, **kw)
    F.cross_entropy(logits[tm], ids[tm]).backward()
    via_forward = {k: p.grad for k, p in module.named_parameters()}
    _, gk, _ = module.train_step(masked, shape, targets=ids, token_mask=tm, **kw)
    via_step = {k: gk.grad_of(p) for k, p in module.named_parameters()}
    sync()
    top = max(float(g.abs().max()) for g in via_step.values() if g is not None and g.numel())
    worst = 0.0
    for k, want in via_step.items():
        got = via_forward[k]
        assert (got is None) == (want is None), k
        if want is None or want.numel() == 0:
            continue
        err = float((got - want).abs().max())
        bound = 1e-5 * float(want.abs().max()) + 1e-6 * top
        worst = max(worst, err / bound)
        assert err <= bound, f"{k}: forward + cross entropy vs train_step differ by {err:.3e} (bound {bound:.3e})"
    gk.busy = False
    module.zero_grad(set_to_none=True)
    return worst


def check_forward_unchanged(lib, device, sync, module, name):
    """With grad enabled the forward returns bit-identical values and a graph; under no_grad no graph is built."""
    set_precision(module, L.PREC_F32)
    with torch.no_grad():
        plain, _ = product_out(name, module, device)
    graphed, _ = product_out(name, module, device)
    sync()
    assert plain.grad_fn is None and not plain.requires_grad
    assert graphed.grad_fn is not None
    assert torch.equal(plain, graphed.detach())


def check_two_forwards_then_one_backward(lib, device, sync, module, name):
    """Two pending graphs of the same module, one backward through both, add up to the two backwards run apart (up to
    the order of atomic adds: 1e-6 of the largest gradient)."""
    case = ALL_CASES[name]
    base = case["base"]
    set_precision(module, L.PREC_F32)
    x = T.inputs(base)
    ids1 = network_input(base, x)
    ids2 = torch.flip(ids1, dims=(1,))
    g1 = upstream_weights(name, (1,))  # only the seed matters: one scalar per graph
    module.zero_grad(set_to_none=True)
    o1, c1 = product_out(name, module, device, ids=ids1)
    o2, c2 = product_out(name, module, device, ids=ids2)
    (o1.square().sum() * float(g1) + o2.sum()).backward()
    together = {k: p.grad.detach().clone() for k, p in module.named_parameters() if p.grad is not None}
    module.zero_grad(set_to_none=True)
    for ids, w in ((ids1, float(g1)), (ids2, None)):
        o, _ = product_out(name, module, device, ids=ids)
        (o.square().sum() * w if w is not None else o.sum()).backward()
    apart = {k: p.grad.detach().clone() for k, p in module.named_parameters() if p.grad is not None}
    module.zero_grad(set_to_none=True)
    sync()
    assert together.keys() == apart.keys()
    top = max(float(g.abs().max()) for g in apart.values() if g.numel())
    for k, g in apart.items():
        if g.numel():
            diff = float((together[k] - g).abs().max())
            assert diff <= 1e-6 * top, f"{name} {k}: together vs apart differ by {diff:.3e} (largest {top:.3e})"


def check_deterministic(lib, device, sync, module, name):
    """The same backward twice: gradients differ only by the order of their atomic adds (1e-6 of the largest)."""
    a = product_grads(name, module, device)
    b = product_grads(name, module, device)
    sync()
    top = max(float(g.abs().max()) for g in a.values() if g is not None and g.numel())
    for k, g in a.items():
        assert (g is None) == (b[k] is None), k
        if g is not None and g.numel():
            diff = float((g - b[k]).abs().max())
            assert diff <= 1e-6 * top, f"{name} {k}: runs differ by {diff:.3e} (largest {top:.3e})"


def check_create_graph_refused(lib, device, sync, module, name):
    set_precision(module, L.PREC_F32)
    out, _ = product_out(name, module, device)
    params = [p for p in module.parameters() if p.requires_grad]
    try:
        torch.autograd.grad(out.sum(), params, create_graph=True)
    except RuntimeError as ex:
        assert "create_graph" in str(ex)
    else:
        raise AssertionError("create_graph=True was accepted")


def check_unsupported_configuration_raises(lib, device, sync):
    """A configuration the forward runs but the backward does not support (dim > 1024: the PEG backward keeps a
    channel row per thread block) raises PhkError from backward(); it does not fault."""
    import phenaki_pytorch_b200 as P
    torch.manual_seed(0)
    m = P.MaskGit(dim=1040, num_tokens=17, max_seq_len=8, heads=1, dim_head=64, depth=1, dim_context=8).to(device)
    m.precision = L.PREC_F32
    ids = torch.randint(0, 17, (1, 4)).to(device)
    ctx = torch.randn(1, 3, 8).to(device)
    out = m(ids, video_patch_shape=(1, 2, 2), context=ctx)
    try:
        out.sum().backward()
    except L.PhkError as ex:
        assert "code -3" in str(ex), ex  # PHK_E_UNSUPPORTED
    else:
        raise AssertionError("the unsupported backward did not raise")
    sync()
