"""Cases of ``Phenaki.forward(video_codebook_ids=ids, text_embeds=e).backward()`` with ``e.requires_grad``, and their
float64 autograd reference.

The reference composes the training loss of phenaki_pytorch.py:596-687 from the oracle's pieces (tests/dropout_ref.py,
which takes dropout masks, on top of oracle/phenaki_oracle.py): the cosine-schedule token mask from the injected draws,
MaskGit's cross entropy, the gumbel-sampled predictions, the critic's BCE times ``critic_loss_weight``; the text
embeddings are a float64 leaf of that graph, so autograd gives ``e.grad`` next to every parameter gradient.
tests/test_train_text_grad_golden_cpu.py pins this composition against the unmodified reference
(tests/golden/train_text_grad.pt).

The product is run with injected draws (``draw_fn``).  ``decisive_draws`` makes the gumbel draw pick one token per row
by a margin of about 16 logits, so the sampled predictions -- and with them the critic's input -- are the same for the
product in either precision mode and for the reference.
"""
import math

import torch
import torch.nn.functional as F

import phenaki_pytorch_b200 as P
from oracle import phenaki_oracle as O
from tests import cases as C
from tests import dropout_ref as DR
from tests import train_at_size_cases as T

# configs[3] of BASELINE.json: MaskGit dim 512, depth 6, V 65536, 4 videos of 9 x 8 x 8 = 576 tokens, 16 text tokens
# of width 768; a one-layer cross-attention TokenCritic of the same width
AT_SIZE = dict(seed=100, steps=18, batch=4, patch_shape=(9, 8, 8), ctx_len=16, ctx_valid=(16, 11, 16, 5),
               input_seed=101, maskgit=dict(dim=512, num_tokens=65536, max_seq_len=1024, dim_context=768, depth=6),
               critic=dict(dim=512, num_tokens=65536, max_seq_len=1024, dim_context=768, depth=1, has_cross_attn=True))

# small cases: TRAIN_CASES' networks, text and video shapes (padded text rows included), optionally with dropout
SMALL = {
    "generator": dict(C.TRAIN_CASES["generator"], critic_kind=None),
    "token_critic": dict(C.TRAIN_CASES["with_critic"], critic_kind="token"),
    "self_critic": dict(C.TRAIN_CASES["self_critic"], critic_kind="self"),
}
AT_SIZE_CASE = dict(AT_SIZE, critic_kind="token")


def build(case, *, dropout=0.0, device="cpu"):
    """Phenaki (training mode) of the case under its seed; ``dropout``: attn_dropout = ff_dropout of both networks."""
    torch.manual_seed(case["seed"])
    cvivit = P.CViViT(**C.SAMPLE_CVIVIT)
    maskgit = P.MaskGit(**case["maskgit"], attn_dropout=dropout, ff_dropout=dropout)
    critic = None
    if case["critic_kind"] == "token":
        critic = P.TokenCritic(**case["critic"], attn_dropout=dropout, ff_dropout=dropout)
    return P.Phenaki(cvivit=cvivit, maskgit=maskgit, critic=critic, steps=case["steps"],
                     self_token_critic=case["critic_kind"] == "self",
                     text_embed_dim=case["maskgit"]["dim_context"]).to(device).train()


# the existing golden of the same reference run (same weights, inputs and draws): its parameter gradients do not depend on
# whether the text embeddings require grad, so tests/golden/train_text_grad.pt holds only the loss and e.grad
GOLDEN_SOURCE = {"token_critic": "with_critic", "self_critic": "self_critic"}


def reference_draws(case):
    """The draws of the reference's Phenaki.forward seeded with the case's noise_seed, in its order: rand_step (b,), the
    uniform behind the random subset (b, n) and, with a critic, the gumbel uniform (b, n, V)."""
    b, n, V = case["batch"], math.prod(case["patch_shape"]), case["maskgit"]["num_tokens"]
    g = torch.Generator().manual_seed(case["noise_seed"])
    draws = {"rand_step": torch.randint(0, case["steps"], (b,), generator=g), "perm": torch.rand((b, n), generator=g)}
    if case["critic_kind"] is not None:
        draws["gumbel"] = torch.zeros((b, n, V)).uniform_(0, 1, generator=g)
    return draws


def golden_case(load, name):
    """The unmodified reference's run of case ``name`` with ``e.requires_grad``: its inputs and draws, the loss and e.grad
    (tests/golden/train_text_grad.pt), every parameter gradient (tests/golden/train_<case>.pt, named as ``product_grads``
    names them) and, for the SelfCritic, the reference's ``to_pred`` weights."""
    tg, tr = load("train_text_grad")[name], load("train_" + GOLDEN_SOURCE[name])
    ids, ctx = C.train_inputs(SMALL[name])
    to_pred = None
    if "to_pred_weight" in tr:
        to_pred = {"0.weight": tr["to_pred_weight"], "0.bias": tr["to_pred_bias"]}
    return dict(ids=ids, text_embeds=ctx, draws=reference_draws(SMALL[name]), loss=tg["loss"],
                grads=golden_parameter_grads(tr), text_embeds_grad=tg["text_embeds_grad"],
                maskgit_digest=tr["maskgit_digest"], to_pred=to_pred)


def golden_parameter_grads(tr):
    """{name: gradient} of a tests/golden/train_<case>.pt, named as ``product_grads`` names them."""
    grads = {f"maskgit.{k}": v for k, v in tr["maskgit_grads"].items()}
    grads.update({f"critic.{k}": v for k, v in (tr["critic_grads"] or {}).items()})
    grads.update({f"critic.to_pred.0.{k}": v for k, v in tr.get("to_pred_grads", {}).items()})
    return grads


def decisive_draws(case, seed=5):
    """rand_step (b,), perm (b, n) and a gumbel uniform (b, n, V) that is 0.5 everywhere except one token per row at the
    largest float32 below 1; that token is the target id for about a third of the rows."""
    b, n, V = case["batch"], math.prod(case["patch_shape"]), case["maskgit"]["num_tokens"]
    g = torch.Generator().manual_seed(seed)
    rand_step = torch.randint(0, case["steps"], (b,), generator=g)
    perm = torch.rand((b, n), generator=g)
    ids, _ = C.train_inputs(case)
    pick = torch.randint(0, V, (b, n), generator=g)
    pick = torch.where(torch.rand((b, n), generator=g) < 1 / 3, ids.reshape(b, n), pick)
    gumbel = torch.full((b, n, V), 0.5)
    gumbel.scatter_(2, pick[..., None], float(torch.tensor(1.0).nextafter(torch.tensor(0.0))))
    return {"rand_step": rand_step, "perm": perm, "gumbel": gumbel}


def product(phenaki, ids, ctx, draws, *, requires_grad=True, **kw):
    """loss.backward() of Phenaki.forward with the draws injected: (loss, {name: gradient or None}, e.grad or None).
    Names: "maskgit.<parameter>", "critic.<parameter>" (a SelfCritic's are "to_pred.*" only: its body is the MaskGit)."""
    dev = next(phenaki.maskgit.parameters()).device
    for p in phenaki.parameters():
        p.grad = None
    e = ctx.detach().to(dev, copy=True).requires_grad_(requires_grad)
    loss = phenaki(video_codebook_ids=ids.to(dev), text_embeds=e, draw_fn=lambda shape, tag: draws[tag].to(dev), **kw)
    loss.backward()
    return loss.detach().cpu(), product_grads(phenaki), (None if e.grad is None else e.grad.detach().cpu())


def product_grads(phenaki):
    grads = {f"maskgit.{k}": (None if p.grad is None else p.grad.detach().cpu()) for k, p in phenaki.maskgit.named_parameters()}
    if isinstance(phenaki.critic, P.TokenCritic):
        grads.update({f"critic.{k}": (None if p.grad is None else p.grad.detach().cpu())
                      for k, p in phenaki.critic.named_parameters()})
    elif phenaki.critic is not None:
        grads.update({f"critic.to_pred.0.{k}": (None if p.grad is None else p.grad.detach().cpu())
                      for k, p in phenaki.critic.to_pred[0].named_parameters()})
    return grads


def _leaves(module, dtype, device):
    params = dict(module.named_parameters())
    sd = {}
    for k, v in module.state_dict().items():
        v = v.detach().to(device)
        v = v.to(dtype) if v.is_floating_point() else v
        sd[k] = v.requires_grad_(True) if k in params else v
    return sd, params


def reference(phenaki, ids, ctx, draws, *, video_mask=None, masks=(None, None), only_train_generator=False,
              only_train_critic=False, dtype=torch.float64, device="cpu"):
    """{"losses": {"loss": 0-d}, "grads": {name: gradient}} by autograd over the oracle in ``dtype`` on ``device``;
    "text_embeds" is d loss / d e.  ``masks``: the dropout multipliers of the MaskGit step and of the critic step (None:
    no dropout).  A parameter without a gradient in the reference is absent."""
    mg = phenaki.maskgit
    msd, mparams = _leaves(mg, dtype, device)
    b, n = ids.shape[0], ids[0].numel()
    shape = tuple(int(v) for v in ids.shape[1:])
    flat = ids.reshape(b, n).to(device)
    e = ctx.detach().to(device=device, dtype=dtype, copy=True).requires_grad_(True)
    text_mask = torch.any(e != 0, dim=-1)
    vmask = torch.ones((b, n), dtype=torch.bool, device=device) if video_mask is None else video_mask.to(device)
    token_mask = O.train_token_mask(draws["rand_step"].to(device), draws["perm"].to(device), phenaki.steps, vmask)
    masked = torch.where(token_mask, mg.mask_id, flat)
    kw = dict(video_patch_shape=shape, heads=mg.transformer.heads, context=e, text_mask=text_mask, video_mask=vmask)
    with torch.set_grad_enabled(not only_train_critic):
        emb = DR._maskgit_embeds(masked, msd, masks=None if only_train_critic else masks[0], **kw)
        logits = F.linear(emb, msd["to_logits.weight"], msd["to_logits.bias"])
    loss = 0.0 if only_train_critic else F.cross_entropy(logits[token_mask], flat[token_mask])
    critic = phenaki.critic
    csd = cparams = None
    if critic is not None and not only_train_generator:
        gumbel = draws["gumbel"].to(device, dtype)
        pred = O.gumbel_sample(logits.detach(), phenaki.critic_train_sample_temperature, gumbel)
        weight = 1.0 if only_train_critic else phenaki.critic_loss_weight
        if isinstance(critic, P.TokenCritic):
            csd, cparams = _leaves(critic, dtype, device)
            ckw = dict(kw, heads=critic.transformer.heads)
            if not critic.has_cross_attn:
                ckw.update(context=None, text_mask=None)
            bce = DR.critic_train_loss(flat, pred, token_mask, csd, masks=masks[1], **ckw)
        else:
            csd, cparams = _leaves(critic.to_pred, dtype, device)
            bce = DR.self_critic_train_loss(flat, pred, token_mask, msd, csd["0.weight"], csd["0.bias"], masks=masks[1],
                                            **kw)
        loss = loss + bce * weight
    loss.backward()
    grads = {f"maskgit.{k}": msd[k].grad for k in mparams if msd[k].grad is not None}
    if cparams is not None:
        pre = "critic." if isinstance(critic, P.TokenCritic) else "critic.to_pred."
        grads.update({pre + k: csd[k].grad for k in cparams if csd[k].grad is not None})
    if e.grad is not None:
        grads["text_embeds"] = e.grad
    return {"losses": {"loss": loss.detach()}, "grads": {k: v.detach().cpu() for k, v in grads.items()}}


def dropout_masks(phenaki, calls, b, n, ctx_len, *, only_train_critic=False):
    """The multipliers the product's steps drew, rebuilt from the (seed, first counter, count) reservations that
    ``tests.train_dropout_cases.record_rng`` saw: (MaskGit step's or None, critic step's or None).  The sampling noise's
    reservation between the two steps is skipped by its count."""
    mg, critic = phenaki.maskgit, phenaki.critic
    nets = [] if only_train_critic else [(0, mg, ctx_len)]
    if critic is not None:
        body = critic if isinstance(critic, P.TokenCritic) else mg
        nets.append((1, body, ctx_len if critic.has_cross_attn else 0))
    out = [None, None]
    pending = list(calls)
    for slot, net, L_ctx in nets:
        tf = net.transformer
        count = DR.layout(net, b, n, L_ctx)[1]
        while pending and pending[0][2] != count:
            pending.pop(0)
        assert pending, "no counter reservation of the dropout step"
        seed, first, _ = pending.pop(0)
        out[slot] = DR.step_masks(net, b, n, L_ctx, seed, first, tf.attn_dropout, tf.ff_dropout, torch.float64)
    return tuple(out)


def masks_to(masks, device):
    if masks is None:
        return None
    return [{k: (None if v is None else v.to(device)) for k, v in layer.items()} for layer in masks]


def padded_rows_are_zero(grad, ctx):
    """Every all-zero (padding) text row has an exactly zero gradient."""
    pad = ~torch.any(ctx != 0, dim=-1)
    return bool(pad.any()) and float(grad[pad].abs().max()) == 0.0


def check(name, loss, grads, e_grad, ref, *, bf16=False):
    """The product's loss, parameter gradients and e.grad against ``reference``: fp32 mode at the parity bars of
    tests/train_at_size_cases.py::check_fp32, bf16 mode within 5 % of each tensor's largest entry (the loss within 2 %).
    Returns the worst max|got - ref| / max|ref|."""
    grads = dict(grads, text_embeds=e_grad)
    if not bf16:
        return T.check_fp32(name, {"loss": loss}, grads, ref)
    want_loss = float(ref["losses"]["loss"])
    assert abs(float(loss) - want_loss) <= 2e-2 * abs(want_loss), f"{name}: bf16 loss {float(loss)!r} vs {want_loss!r}"
    top = T.largest_gradient(ref)
    worst, failures = 0.0, []
    for k, got in grads.items():
        want = ref["grads"].get(k)
        if (got is None) != (want is None):
            failures.append(f"{k}: gradient {'missing' if got is None else 'where the reference has none'}")
            continue
        if got is None or not want.numel():
            continue
        err = float((got.double() - want).abs().max())
        if T.is_analytically_zero(k):
            if err > 5e-2 * top:
                failures.append(f"{k}: |got - ref| {err:.3e} above 5e-2 x the largest gradient {top:.3e}")
            continue
        scale = float(want.abs().max())
        worst = max(worst, err / scale)
        if err > 5e-2 * scale:
            failures.append(f"{k}: max err / max|ref| {err / scale:.3e}")
    assert not failures, f"{name} (bf16):\n  " + "\n  ".join(failures)
    return worst


def run_and_reference(case, phenaki, draws, *, ref_device="cpu", **kw):
    """One product ``Phenaki.forward(...).backward()`` of the case's inputs with ``e.requires_grad`` and the float64
    reference on the same draws, fed the dropout masks the product's steps drew: (loss, grads, e.grad, reference).
    ``kw``: only_train_generator / only_train_critic."""
    from tests import train_dropout_cases as TD
    ids, ctx = C.train_inputs(case)
    with TD.record_rng() as calls:
        loss, grads, e_grad = product(phenaki, ids, ctx, draws, **kw)
    masks = (None, None)
    tf = phenaki.maskgit.transformer
    if phenaki.training and (tf.attn_dropout > 0 or tf.ff_dropout > 0):
        masks = dropout_masks(phenaki, calls, ids.shape[0], ids[0].numel(), ctx.shape[1],
                              only_train_critic=kw.get("only_train_critic", False))
        masks = tuple(masks_to(m, ref_device) for m in masks)
    return loss, grads, e_grad, reference(phenaki, ids, ctx, draws, masks=masks, device=ref_device, **kw)
