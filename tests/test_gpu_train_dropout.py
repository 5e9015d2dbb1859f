"""GPU: the training step with attention and FF dropout (include/phk.h, phk_dropout_t).

fp32 mode is held to the parity bars of tests/test_gpu_train_at_size.py against the float64 autograd reference fed the
masks rebuilt in numpy from the counters the step reserved (tests/train_dropout_cases.py); bf16 mode to its closeness
bars.  Dropout off -- probabilities 0, or the module in eval mode -- is the plain step: same launches, same loss, no
counters.  With dropout on the step reserves exactly its counters from the device generator, so successive steps draw
new masks and ``torch.manual_seed`` repeats them.  ``Phenaki.forward`` + ``backward()`` trains with dropout end to end."""
import ctypes
import math

import pytest
import torch

import phenaki_pytorch_b200 as P
from phenaki_pytorch_b200 import _lib as L
from tests import cases as C
from tests import dropout_ref as DR
from tests import train_at_size_cases as T
from tests import train_dropout_cases as TD

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _gen():
    return torch.cuda.default_generators[0]


def _module(name, attn_p=TD.ATTN_P, ff_p=TD.FF_P):
    return T.build_module(TD.case(name, attn_p, ff_p)).to(DEV).train()


def _within_atomics(g1, g2, top):
    for k, a in g1.items():
        b = g2[k]
        assert (a is None) == (b is None), k
        if a is not None and a.numel():
            diff = float((a - b).abs().max())
            assert diff <= 1e-6 * top, f"{k}: differ by {diff:.3e}, the largest gradient is {top:.3e}"


@pytest.mark.parametrize("name", ["tiny", "ragged_ce", "prod_ce", "prod_critic", "ragged_self_critic"])
def test_fp32_dropout_step_matches_fp64_autograd_with_the_rebuilt_masks(name):
    module = _module(name)
    losses, grads, ref, calls = TD.run_and_reference(name, module, DEV)
    assert len(calls) == (2 if name == "ragged_self_critic" else 1)
    worst = T.check_fp32(name, losses, grads, ref)
    print(f"\nDROPOUT {name} fp32: worst max err / max|ref| {worst:.3e}")


def test_bf16_dropout_step_is_close_to_fp64_autograd():
    name = "prod_ce"
    module = _module(name)
    losses, grads, ref, _ = TD.run_and_reference(name, module, DEV, precision=L.PREC_BF16)
    got, want = float(losses["loss"]), float(ref["losses"]["loss"])
    assert abs(got - want) <= 2e-2 * abs(want), f"bf16 loss {got!r} vs fp64 {want!r}"
    top = T.largest_gradient(ref)
    failures, worst = [], 0.0
    for k, g in grads.items():
        r = ref["grads"].get(k)
        if (g is None) != (r is None):
            failures.append(f"{k}: gradient {'missing' if g is None else 'where the reference has none'}")
            continue
        if g is None or r.numel() == 0:
            continue
        err = (g.double() - r).abs().max().item()
        if T.is_analytically_zero(k):
            if err > 5e-2 * top:
                failures.append(f"{k}: |got - ref| {err:.3e} above 5e-2 x the largest gradient {top:.3e}")
            continue
        scale = r.abs().max().item()
        cos = torch.nn.functional.cosine_similarity(g.double().flatten(), r.flatten(), dim=0).item()
        worst = max(worst, err / scale)
        if err > 5e-2 * scale or cos < 0.995:
            failures.append(f"{k}: max err / max|ref| {err / scale:.3e}, cosine {cos:.5f}")
    assert not failures, "prod_ce (bf16):\n  " + "\n  ".join(failures)
    assert worst > 1e-5, "bf16 mode gave fp32-exact gradients: the tensor-core products were not used"
    print(f"\nDROPOUT prod_ce bf16: worst max err / max|ref| {worst:.3e}")


@pytest.mark.parametrize("name", ["ragged_ce", "prod_critic"])
def test_dropout_off_is_the_plain_step(name):
    """Probabilities 0 in training mode, and probabilities > 0 in eval mode: the launches of the module built without
    dropout, its loss bit for bit, its gradients up to the order of atomics, and no counters drawn."""
    lib = L.lib()
    c0 = TD.case(name, 0.0, 0.0)

    def run(module, c):
        torch.cuda.synchronize()
        before, offset = lib.phk_launch_count(), _gen().get_offset()
        losses, grads = TD.product_step(c, module, DEV)
        torch.cuda.synchronize()
        return lib.phk_launch_count() - before, _gen().get_offset() - offset, losses, grads

    plain = run(_module(name, 0.0, 0.0), c0)
    top = max(float(g.abs().max()) for g in plain[3].values() if g is not None and g.numel())
    for module, c in ((_module(name, 0.0, 0.0), c0), (_module(name).eval(), TD.case(name))):
        launches, advanced, losses, grads = run(module, c)
        assert launches == plain[0] and advanced == 0
        for k in plain[2]:
            assert torch.equal(losses[k], plain[2][k]), k
        _within_atomics(grads, plain[3], top)
    on = run(_module(name), TD.case(name))
    assert on[0] != plain[0] and on[1] > 0  # the comparison can see the dropout path


def test_rng_accounting_and_repeatability():
    name = "ragged_ce"
    c = TD.case(name)
    module = _module(name)
    n = math.prod(c["patch_shape"])
    counters = DR.layout(module, c["batch"], n, c["ctx_len"])[1]
    assert counters == L.lib().phk_maskgit_train_dropout_counters(ctypes.byref(module._table()), c["batch"], n,
                                                                  c["ctx_len"])
    torch.manual_seed(1234)
    o0 = _gen().get_offset()
    l1, g1 = TD.product_step(c, module, DEV)
    o1 = _gen().get_offset()
    assert o1 - o0 == (counters + 3) // 4 * 4
    l2, _ = TD.product_step(c, module, DEV)
    assert _gen().get_offset() - o1 == (counters + 3) // 4 * 4
    assert not torch.equal(l1["loss"], l2["loss"]), "two successive steps drew the same masks"
    torch.manual_seed(1234)
    l3, g3 = TD.product_step(c, module, DEV)
    assert torch.equal(l1["loss"], l3["loss"])
    _within_atomics(g1, g3, max(float(g.abs().max()) for g in g1.values() if g is not None and g.numel()))


@pytest.mark.parametrize("critic", ["token", "self"])
def test_phenaki_forward_backward_trains_with_dropout(critic):
    case = C.TRAIN_CASES["with_critic" if critic == "token" else "self_critic"]
    ids, ctx = C.train_inputs(case)

    def forward_backward(p):
        torch.manual_seed(case["seed"])
        cvivit = P.CViViT(**C.SAMPLE_CVIVIT)
        maskgit = P.MaskGit(**case["maskgit"], attn_dropout=p, ff_dropout=p)
        tcritic = P.TokenCritic(**case["critic"], attn_dropout=p, ff_dropout=p) if critic == "token" else None
        phenaki = P.Phenaki(cvivit=cvivit, maskgit=maskgit, critic=tcritic, steps=case["steps"],
                            self_token_critic=critic == "self",
                            text_embed_dim=case["maskgit"]["dim_context"]).to(DEV).train()
        o0 = _gen().get_offset()
        loss = phenaki(video_codebook_ids=ids.to(DEV), text_embeds=ctx.to(DEV))
        loss.backward()
        torch.cuda.synchronize()
        return phenaki, loss, _gen().get_offset() - o0

    _, _, plain_advance = forward_backward(0.0)
    phenaki, loss, advance = forward_backward(0.25)
    assert torch.isfinite(loss).item()
    b, n = ids.shape[0], ids[0].numel()
    # on top of the draws of the step without dropout: the MaskGit step's counters and the critic step's (both critics
    # here have cross-attention; the SelfCritic's BCE step draws fresh masks through the MaskGit body)
    critic_net = phenaki.critic if critic == "token" else phenaki.maskgit
    extra = sum((DR.layout(net, b, n, case["ctx_len"])[1] + 3) // 4 * 4 for net in (phenaki.maskgit, critic_net))
    assert advance - plain_advance == extra
    for owner in (phenaki.maskgit, phenaki.critic):
        for k, p in owner.named_parameters():
            if p.numel() and ".1.context_norm." not in k:  # the self-attention's context_norm is unused (no gradient)
                assert p.grad is not None and torch.isfinite(p.grad).all(), k
