"""CPU: ``Phenaki.forward(text_embeds=e).backward()`` in fp32 mode on the CPU executor of tests/cuda_emu (csrc/train.cu
compiled by g++), against the float64 reference of tests/text_grad_cases.py: ``e.grad`` and every parameter gradient at
the fp32 parity bars, for MaskGit alone, with a cross-attention TokenCritic and with a SelfCritic, for
``only_train_generator`` / ``only_train_critic``, and with attention and FF dropout.  Padded text rows get exactly zero
gradient; asking for ``e.grad`` changes neither the loss nor any parameter gradient."""
import pytest
import torch

from tests import cases as C
from tests import emu_runtime
from tests import text_grad_cases as TG


@pytest.fixture(scope="module")
def emu():
    return emu_runtime.build_emu()


@pytest.fixture
def on_cpu(emu, monkeypatch):
    emu_runtime.route_product_to_emulator(emu, monkeypatch)


@pytest.mark.parametrize("name,dropout,mode", [
    ("generator", 0.0, None), ("token_critic", 0.0, None), ("self_critic", 0.0, None),
    ("token_critic", 0.0, "only_train_generator"), ("token_critic", 0.0, "only_train_critic"),
    ("token_critic", 0.2, None), ("self_critic", 0.2, None)])
def test_emulated_text_grad_matches_fp64_autograd(on_cpu, name, dropout, mode):
    case = TG.SMALL[name]
    phenaki = TG.build(case, dropout=dropout)
    kw = {mode: True} if mode else {}
    loss, grads, e_grad, ref = TG.run_and_reference(case, phenaki, TG.decisive_draws(case), **kw)
    TG.check(name, loss, grads, e_grad, ref)
    assert TG.padded_rows_are_zero(e_grad, C.train_inputs(case)[1])


@pytest.mark.parametrize("name", ["token_critic", "self_critic"])
def test_emulated_text_grad_matches_the_reference_golden(on_cpu, golden, name):
    g = TG.golden_case(golden, name)
    phenaki = TG.build(TG.SMALL[name])
    if g["to_pred"] is not None:
        phenaki.critic.to_pred.load_state_dict(g["to_pred"])
    loss, grads, e_grad = TG.product(phenaki, g["ids"], g["text_embeds"], g["draws"])
    torch.testing.assert_close(loss, g["loss"], rtol=1e-4, atol=1e-5)
    want = g["text_embeds_grad"]
    torch.testing.assert_close(e_grad, want, rtol=2e-3, atol=2e-4 * float(want.abs().max()))
    assert TG.padded_rows_are_zero(e_grad, g["text_embeds"])


def test_emulated_parameter_gradients_do_not_depend_on_the_text_grad(on_cpu):
    case = TG.SMALL["token_critic"]
    phenaki = TG.build(case)
    ids, ctx = C.train_inputs(case)
    draws = TG.decisive_draws(case)
    l0, g0, e0 = TG.product(phenaki, ids, ctx, draws, requires_grad=False)
    l1, g1, e1 = TG.product(phenaki, ids, ctx, draws)
    assert e0 is None and e1 is not None
    assert torch.equal(l0, l1)
    for k, g in g0.items():
        assert (g is None) == (g1[k] is None), k
        assert g is None or torch.equal(g, g1[k]), k
