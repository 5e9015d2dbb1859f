"""Training-step cases at the sizes the step is used at, and their float64 autograd reference.

phk_maskgit_train_step chooses its code path by shape: the batched-product attention backward (n * nkt >= 64 * 64), the
split-K wgrad (a weight of <= 16384 elements reduced over >= 1024 rows, in 256-row slices that meet through atomics),
the bf16 mma.sync products over several K chunks and tiles, dim_head 64, and the row kernels at V = 65536 and D = 512.
The cases below land on both sides of those thresholds: the ``prod_*`` cases at the MaskGit production shape (dim 512,
8 x 64 heads, V 65536, 576 tokens, 16 text tokens), the ``ragged_*`` cases at sizes that leave partial tiles and a
partial last split-K slice.

For each case this module builds the product module under a fixed seed, draws the inputs from seeded generators and
computes the loss and every parameter gradient with the oracle under torch autograd in float64 (the oracle restates
the reference; tests/test_oracle_golden.py pins it).  The references are cached per process: each costs seconds.
"""
import functools
import math

import torch

import phenaki_pytorch_b200 as P
from oracle import phenaki_oracle as O

PROD_MASKGIT = dict(dim=512, num_tokens=65536, max_seq_len=1024, dim_context=768, depth=2)  # heads 8 x dim_head 64
PROD_CRITIC = dict(dim=512, num_tokens=65536, max_seq_len=1024, dim_context=768, depth=2, has_cross_attn=True)
RAGGED_MASKGIT = dict(dim=192, num_tokens=4099, max_seq_len=200, heads=3, dim_head=64, depth=1, dim_context=72)

CASES = {
    # self- and cross-attention backward as batched products (576 x 576, 576 x (2 + 16)), position-bias MLP split-K
    # over U = 17 * 15 * 15 = 3825 deltas, dim_head 64, CE over V = 65536, D = 512 row kernels, masked text tail
    "prod_ce": dict(kind="maskgit", seed=80, ctor=PROD_MASKGIT, batch=2, patch_shape=(9, 8, 8), ctx_len=16,
                    ctx_valid=(16, 11), video_valid=None, input_seed=81),
    # TokenCritic: the BCE head's [1, 512] wgrad split over R = 1152 = 4 * 256 + 128 rows
    "prod_critic": dict(kind="critic", seed=82, ctor=PROD_CRITIC, batch=2, patch_shape=(9, 8, 8), ctx_len=16,
                        ctx_valid=(16, 13), video_valid=None, input_seed=83),
    # n = 189 = 2 * 64 + 61 (partial tiles), U = 5 * 13 * 17 = 1105 (a partial last 256-row slice), masked text tails
    # and a padding tail in the video mask
    "ragged_ce": dict(kind="maskgit", seed=84, ctor=RAGGED_MASKGIT, batch=3, patch_shape=(3, 7, 9), ctx_len=11,
                      ctx_valid=(11, 4, 7), video_valid=(189, 150, 123), input_seed=85),
    # SelfCritic on that MaskGit: its [1, 192] head wgrad split over R = 6 * 189 = 1134 rows (a partial last slice);
    # Phenaki trains it as two steps (CE, then BCE through the same body) whose MaskGit gradients add up
    "ragged_self_critic": dict(kind="self_critic", seed=86, ctor=RAGGED_MASKGIT, batch=6, patch_shape=(3, 7, 9),
                               ctx_len=11, ctx_valid=(11, 4, 7, 11, 1, 9), video_valid=None, input_seed=87),
}

# Small enough for the CPU executor of tests/cuda_emu and still past thresholds of the step
EMULATED_CASES = {
    # ragged_ce at b = 1, dim 64: n * n = 189 * 189 >= 4096, U = 1105.  Two 64-wide heads, so that the batched products'
    # walk over the heads of the token-major dO is exercised (with one head its head offset is always zero)
    "emu_ragged_ce": dict(kind="maskgit", seed=88, batch=1, patch_shape=(3, 7, 9), ctx_len=11, ctx_valid=(7,),
                          video_valid=(160,), input_seed=89,
                          ctor=dict(dim=64, num_tokens=300, max_seq_len=200, heads=2, dim_head=64, depth=1,
                                    dim_context=40)),
    # TokenCritic with b * n = 16 * 65 = 1040 rows: the head wgrad split into 256-row slices, the last one of 16 rows
    "emu_critic_split_head": dict(kind="critic", seed=90, batch=16, patch_shape=(1, 5, 13), ctx_len=6,
                                  ctx_valid=(6, 2, 5, 6, 1, 3, 6, 4, 6, 6, 2, 5, 6, 3, 6, 1), video_valid=None,
                                  input_seed=91,
                                  ctor=dict(dim=64, num_tokens=300, max_seq_len=72, heads=1, dim_head=64, depth=1,
                                            dim_context=40, has_cross_attn=True)),
}

ALL_CASES = {**CASES, **EMULATED_CASES}

# Gradients that are zero in exact arithmetic: the last bias of the position-bias MLP adds one constant per head to every
# self-attention logit of that head (no null keys there), and softmax is invariant to a constant shift.  What either side
# computes for them is rounding noise, so they are checked against an absolute bound only.
ANALYTICALLY_ZERO = ("continuous_pos_bias.net.2.bias",)


def is_analytically_zero(name):
    return any(name == z or name.endswith("." + z) for z in ANALYTICALLY_ZERO)


def build_module(case):
    """The product module (MaskGit, TokenCritic or SelfCritic) of the case, on the CPU, under its seed."""
    torch.manual_seed(case["seed"])
    if case["kind"] == "critic":
        return P.TokenCritic(**case["ctor"])
    maskgit = P.MaskGit(**case["ctor"])
    return P.SelfCritic(maskgit) if case["kind"] == "self_critic" else maskgit


def inputs(case):
    """Seeded inputs: target ids, a token mask of about 50 % (inside the video mask, at least one token per sequence),
    synthetic text embeddings whose tail rows are padding (zero) where ``ctx_valid`` says so, and, for the critics, the
    sampled predictions (about a third of them equal to the target)."""
    b = case["batch"]
    n = math.prod(case["patch_shape"])
    V = case["ctor"]["num_tokens"]
    g = torch.Generator().manual_seed(case["input_seed"])
    ids = torch.randint(0, V, (b, n), generator=g)
    vmask = None
    if case["video_valid"] is not None:
        vmask = torch.arange(n)[None, :] < torch.tensor(case["video_valid"])[:, None]
    token_mask = torch.rand((b, n), generator=g) < 0.5
    token_mask[:, 0] = True
    if vmask is not None:
        token_mask &= vmask
    ctx = torch.randn((b, case["ctx_len"], case["ctor"]["dim_context"]), generator=g)
    for i, v in enumerate(case["ctx_valid"]):
        ctx[i, v:] = 0.0
    pred = torch.where(torch.rand((b, n), generator=g) < 1 / 3, ids, torch.randint(0, V, (b, n), generator=g))
    return dict(ids=ids, token_mask=token_mask, context=ctx, text_mask=torch.any(ctx != 0, dim=-1), video_mask=vmask,
                pred=pred, n=n)


def reference(name, dtype=torch.float64):
    """{"losses": {name: 0-d tensor}, "grads": {parameter name: gradient}} of the case by oracle autograd in ``dtype``
    on the CPU; a parameter the reference leaves without a gradient is absent from "grads"."""
    return _reference(name, dtype)


@functools.lru_cache(maxsize=None)
def _reference(name, dtype):
    case = ALL_CASES[name]
    module = build_module(case)
    x = inputs(case)
    heads = case["ctor"].get("heads", 8)
    shape = case["patch_shape"]
    params = dict(module.named_parameters())
    sd = {}
    for k, v in module.state_dict().items():
        v = v.detach().to(dtype) if v.is_floating_point() else v.detach()
        sd[k] = v.requires_grad_(True) if k in params else v
    ctx = x["context"].to(dtype)
    kw = dict(video_patch_shape=shape, heads=heads, context=ctx, text_mask=x["text_mask"], video_mask=x["video_mask"])
    losses = {}
    if case["kind"] == "maskgit":
        losses["loss"] = O.maskgit_train_loss(x["ids"], sd, x["token_mask"], **kw)
        total = losses["loss"]
    elif case["kind"] == "critic":
        losses["loss"] = O.critic_train_loss(x["ids"], x["pred"], x["token_mask"], sd, **kw)
        total = losses["loss"]
    else:  # SelfCritic: the state dict is {"maskgit.*", "to_pred.0.*"}; Phenaki.forward's loss is ce + 1.0 * bce
        msd = {k[len("maskgit."):]: v for k, v in sd.items() if k.startswith("maskgit.")}
        losses["ce"] = O.maskgit_train_loss(x["ids"], msd, x["token_mask"], **kw)
        losses["bce"] = O.self_critic_train_loss(x["ids"], x["pred"], x["token_mask"], msd, sd["to_pred.0.weight"],
                                                 sd["to_pred.0.bias"], **kw)
        total = losses["ce"] + losses["bce"]
    total.backward()
    grads = {k: sd[k].grad for k in params if sd[k].grad is not None}
    return {"losses": {k: v.detach() for k, v in losses.items()}, "grads": grads}


def product_step(name, module, device, precision=None):
    """One training step of the product (phk_maskgit_train_step through train_step) on ``module`` (already on
    ``device``): ({loss name: float tensor on the CPU}, {parameter name: gradient on the CPU, or None when the step
    gives it none}).  The SelfCritic case runs Phenaki's two steps and adds their MaskGit gradients."""
    from phenaki_pytorch_b200 import _lib as L
    case = ALL_CASES[name]
    x = inputs(case)
    dev = torch.device(device)
    ids, tm = x["ids"].to(dev), x["token_mask"].to(dev)
    kw = dict(context=x["context"].to(dev), text_mask=x["text_mask"].to(dev),
              video_mask=None if x["video_mask"] is None else x["video_mask"].to(dev))
    shape = case["patch_shape"]
    labels = (ids != x["pred"].to(dev)).float()
    critic_in = torch.where(tm, x["pred"].to(dev), ids)
    mask_id = case["ctor"]["num_tokens"]
    maskgit = module.maskgit if case["kind"] == "self_critic" else module
    maskgit.precision = L.PREC_F32 if precision is None else precision

    def grads_of(gk, named):
        out = {}
        for k, p in named:
            g = gk.grad_of(p)
            out[k] = None if g is None else g.detach().to("cpu", copy=True)
        return out

    if case["kind"] == "maskgit":
        loss, gk, _ = module.train_step(torch.where(tm, mask_id, ids), shape, targets=ids, token_mask=tm, **kw)
        return {"loss": loss.detach().cpu()}, grads_of(gk, module.named_parameters())
    if case["kind"] == "critic":
        loss, gk, _ = module.train_step(critic_in, shape, labels=labels, **kw)
        return {"loss": loss.detach().cpu()}, grads_of(gk, module.named_parameters())
    ce, gk, _ = maskgit.train_step(torch.where(tm, mask_id, ids), shape, targets=ids, token_mask=tm, **kw)
    first = grads_of(gk, (("maskgit." + k, p) for k, p in maskgit.named_parameters()))
    bce, cgk, _ = module.train_step(critic_in, shape, labels=labels, **kw)
    grads = grads_of(cgk, module.named_parameters())
    for k, g in first.items():
        if g is not None:
            grads[k] = g if grads[k] is None else grads[k] + g
    return {"ce": ce.detach().cpu(), "bce": bce.detach().cpu()}, grads


def largest_gradient(ref):
    return max(float(g.abs().max()) for g in ref["grads"].values() if g.numel())


def check_fp32(name, losses, grads, ref, *, max_ratio=1e-4, fro_ratio=2e-5, zero_ratio=1e-6):
    """fp32 parity against the fp64 reference: every loss within 1e-5 relative; per gradient tensor
    max|got - ref| <= max_ratio * max|ref| and ||got - ref|| / ||ref|| <= fro_ratio; the ANALYTICALLY_ZERO tensors
    within zero_ratio * (the step's largest gradient entry); no gradient where the reference has none.
    Returns the worst max|got - ref| / max|ref| over the other tensors."""
    for k, want in ref["losses"].items():
        got = float(losses[k])
        assert abs(got - float(want)) <= 1e-5 * abs(float(want)), f"{name} {k}: {got!r} vs fp64 {float(want)!r}"
    top = largest_gradient(ref)
    worst, failures = 0.0, []
    for k, got in grads.items():
        want = ref["grads"].get(k)
        if want is None:
            if got is not None:
                failures.append(f"{k}: the reference leaves this gradient unset")
            continue
        if got is None:
            failures.append(f"{k}: no gradient")
            continue
        assert got.shape == want.shape, k
        if want.numel() == 0:
            continue
        err = (got.double() - want).abs().max().item()
        if is_analytically_zero(k):
            if err > zero_ratio * top or float(want.abs().max()) > zero_ratio * top:
                failures.append(f"{k}: |got - ref| {err:.3e} above {zero_ratio:g} x the largest gradient {top:.3e}")
            continue
        scale = want.abs().max().item()
        fro = ((got.double() - want).norm() / want.norm()).item()
        worst = max(worst, err / scale)
        if err > max_ratio * scale or fro > fro_ratio:
            failures.append(f"{k}: max err / max|ref| {err / scale:.3e}, relative Frobenius error {fro:.3e}")
    assert not failures, f"{name} (fp32):\n  " + "\n  ".join(failures)
    return worst
