"""CPU: the float64 composition of the training loss in tests/text_grad_cases.py -- the reference the GPU and emulated
tests hold ``Phenaki.forward(text_embeds=e).backward()`` to -- against the unmodified reference's autograd: loss,
every parameter gradient and ``e.grad`` (tests/golden/train_text_grad.pt for the loss and ``e.grad``, the parameter
gradients of the same run from train_with_critic.pt / train_self_critic.pt), with a cross-attention TokenCritic and
with a SelfCritic.  Both cases have padded (all-zero) text rows, whose gradient is exactly zero on both sides."""
import pytest
import torch

from tests import cases as C
from tests import text_grad_cases as TG
from tests import train_at_size_cases as T


def _reference_of(name, g):
    case = TG.SMALL[name]
    phenaki = TG.build(case)
    assert C.state_digest(phenaki.maskgit.state_dict()) == g["maskgit_digest"]
    if g["to_pred"] is not None:
        phenaki.critic.to_pred.load_state_dict(g["to_pred"])
    return TG.reference(phenaki, g["ids"], g["text_embeds"], g["draws"])


@pytest.mark.parametrize("name", ["token_critic", "self_critic"])
def test_fp64_composition_matches_the_reference_autograd(golden, name):
    g = TG.golden_case(golden, name)
    ref = _reference_of(name, g)
    want_loss = float(g["loss"])
    assert abs(float(ref["losses"]["loss"]) - want_loss) <= 1e-5 * abs(want_loss)
    want = dict(g["grads"], text_embeds=g["text_embeds_grad"])
    assert set(ref["grads"]) == set(want), set(ref["grads"]) ^ set(want)
    top = max(float(v.abs().max()) for v in want.values() if v.numel())
    for k, w in want.items():
        got = ref["grads"][k]
        assert got.shape == w.shape, k
        if not w.numel():
            continue
        err = float((got - w.double()).abs().max())
        if T.is_analytically_zero(k):
            assert err <= 1e-6 * top, k
            continue
        assert err <= 1e-4 * float(w.abs().max()), f"{k}: max err {err:.3e}, max|ref| {float(w.abs().max()):.3e}"


@pytest.mark.parametrize("name", ["token_critic", "self_critic"])
def test_padded_text_rows_get_exactly_zero_gradient(golden, name):
    g = TG.golden_case(golden, name)
    ctx = g["text_embeds"]
    assert TG.padded_rows_are_zero(g["text_embeds_grad"], ctx)
    assert TG.padded_rows_are_zero(_reference_of(name, g)["grads"]["text_embeds"], ctx)
    # and the valid rows do get one
    valid = torch.any(ctx != 0, dim=-1)
    assert float(g["text_embeds_grad"][valid].abs().min(dim=-1).values.max()) > 0
