"""Training-step cases with attention and FF dropout, and their float64 reference with the masks rebuilt from the counter
contract (tests/dropout_ref.py).

The product step draws its masks from counters it reserves through ``phenaki._rng_take``; ``record_rng`` wraps that
function so a test learns the (seed, first counter) of every step and can rebuild exactly the masks the step used.  The
cases are those of tests/train_at_size_cases.py with dropout added to the constructor, plus ``tiny``: small enough that
one wrong mask element moves the loss far beyond the fp32 bar.
"""
import contextlib
import math

import torch

from phenaki_pytorch_b200 import _lib as L
from phenaki_pytorch_b200 import phenaki as PH
from tests import dropout_ref as DR
from tests import train_at_size_cases as T

ATTN_P, FF_P = 0.1, 0.25

TINY = dict(kind="maskgit", seed=92, batch=2, patch_shape=(2, 2, 3), ctx_len=3, ctx_valid=(3, 2), video_valid=None,
            input_seed=93, ctor=dict(dim=32, num_tokens=23, max_seq_len=16, heads=2, dim_head=16, depth=2,
                                     dim_context=12))
CASES = {"tiny": TINY, **T.ALL_CASES}


def case(name, attn_p=ATTN_P, ff_p=FF_P):
    c = dict(CASES[name])
    c["ctor"] = dict(c["ctor"], attn_dropout=attn_p, ff_dropout=ff_p)
    return c


@contextlib.contextmanager
def record_rng():
    """Yields a list that receives (seed, first counter, count) of every counter reservation of the product."""
    calls, real = [], PH._rng_take

    def take(dev, seed, count):
        first = real(dev, seed, count)
        calls.append((int(seed), int(first), int(count)))
        return first

    PH._rng_take = take
    try:
        yield calls
    finally:
        PH._rng_take = real


def product_step(c, module, device, precision=None):
    """T.product_step for a case dict: ({loss name: tensor}, {parameter name: gradient or None}); the SelfCritic case
    runs the CE step and then the BCE step through the same body, and adds their MaskGit gradients."""
    x = T.inputs(c)
    dev = torch.device(device)
    ids, tm = x["ids"].to(dev), x["token_mask"].to(dev)
    kw = dict(context=x["context"].to(dev), text_mask=x["text_mask"].to(dev),
              video_mask=None if x["video_mask"] is None else x["video_mask"].to(dev))
    shape = c["patch_shape"]
    labels = (ids != x["pred"].to(dev)).float()
    critic_in = torch.where(tm, x["pred"].to(dev), ids)
    mask_id = c["ctor"]["num_tokens"]
    maskgit = module.maskgit if c["kind"] == "self_critic" else module
    maskgit.precision = L.PREC_F32 if precision is None else precision

    def grads_of(gk, named):
        return {k: (None if gk.grad_of(p) is None else gk.grad_of(p).detach().to("cpu", copy=True)) for k, p in named}

    if c["kind"] == "maskgit":
        loss, gk, _ = module.train_step(torch.where(tm, mask_id, ids), shape, targets=ids, token_mask=tm, **kw)
        return {"loss": loss.detach().cpu()}, grads_of(gk, module.named_parameters())
    if c["kind"] == "critic":
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


def masks_of(c, module, seed, offset, dtype=torch.float64, attn_p=None, ff_p=None):
    """The multipliers of one step of the case's network (the MaskGit body for the SelfCritic) at (seed, offset)."""
    net = module.maskgit if c["kind"] == "self_critic" else module
    tf = net.transformer
    n = math.prod(c["patch_shape"])
    return DR.step_masks(net, c["batch"], n, c["ctx_len"], seed, offset,
                         tf.attn_dropout if attn_p is None else attn_p, tf.ff_dropout if ff_p is None else ff_p, dtype)


def reference(c, step_masks, dtype=torch.float64):
    """{"losses", "grads"} of the case by autograd over tests/dropout_ref.py in ``dtype`` on the CPU; ``step_masks``: the
    masks of each product step (one; two for the SelfCritic: CE then BCE)."""
    module = T.build_module(c)
    x = T.inputs(c)
    heads = c["ctor"].get("heads", 8)
    params = dict(module.named_parameters())
    sd = {}
    for k, v in module.state_dict().items():
        v = v.detach().to(dtype) if v.is_floating_point() else v.detach()
        sd[k] = v.requires_grad_(True) if k in params else v
    kw = dict(video_patch_shape=c["patch_shape"], heads=heads, context=x["context"].to(dtype),
              text_mask=x["text_mask"], video_mask=x["video_mask"])
    losses = {}
    if c["kind"] == "maskgit":
        losses["loss"] = DR.maskgit_train_loss(x["ids"], sd, x["token_mask"], masks=step_masks[0], **kw)
        total = losses["loss"]
    elif c["kind"] == "critic":
        losses["loss"] = DR.critic_train_loss(x["ids"], x["pred"], x["token_mask"], sd, masks=step_masks[0], **kw)
        total = losses["loss"]
    else:
        msd = {k[len("maskgit."):]: v for k, v in sd.items() if k.startswith("maskgit.")}
        losses["ce"] = DR.maskgit_train_loss(x["ids"], msd, x["token_mask"], masks=step_masks[0], **kw)
        losses["bce"] = DR.self_critic_train_loss(x["ids"], x["pred"], x["token_mask"], msd, sd["to_pred.0.weight"],
                                                  sd["to_pred.0.bias"], masks=step_masks[1], **kw)
        total = losses["ce"] + losses["bce"]
    total.backward()
    grads = {k: sd[k].grad for k in params if sd[k].grad is not None}
    return {"losses": {k: v.detach() for k, v in losses.items()}, "grads": grads}


def run_and_reference(name, module, device, precision=None, **ps):
    """One product step of case ``name`` on ``module`` and the fp64 reference fed the masks rebuilt from the counters
    that step reserved: (losses, grads, ref, rng calls)."""
    c = case(name, **ps)
    with record_rng() as calls:
        losses, grads = product_step(c, module, device, precision)
    masks = [masks_of(c, module, seed, first) for seed, first, _ in calls]
    return losses, grads, reference(c, masks), calls
