"""GPU: the training step (phk_maskgit_train_step) at the sizes it is used at, against the float64 autograd reference of
tests/train_at_size_cases.py.  The cases put the step past every shape threshold of csrc/train.cu: the batched-product
attention backward of the self- and cross-attention, the split-K wgrad of the position-bias MLP and of the BCE heads
(with partial last slices), dim_head 64, the CE row kernel at V = 65536, the PEG / LayerNorm backward at D = 512.

fp32 mode is held to parity: each loss within 1e-5 relative, each gradient tensor within 1e-4 of its largest entry
(max norm) and 2e-5 (relative Frobenius norm).  The gradients that are zero in exact arithmetic
(``ANALYTICALLY_ZERO``) are held to 1e-6 of the step's largest gradient entry instead.

bf16 mode runs the nn.Linear products on the wgmma GEMM and the attention-backward contractions (dP, dS.kh, dS^T.qh,
P^T.dO, with K up to 576) on the mma.sync kernel, with bf16 operands and fp32 accumulation.  Rounding the operands to
bf16 makes those products differ from the fp32 ones by design, so bf16 mode is compared for closeness, not parity:
loss within 2 %, every gradient tensor within 5 % of its largest entry at a cosine similarity of at least 0.995, and a
worst error above 1e-5 to show that the tensor-core path was taken.

Running the same step twice gives the same loss, and gradients that differ only by the order of their atomic adds."""
import pytest
import torch

from phenaki_pytorch_b200 import _lib as L
from tests import train_at_size_cases as T

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


@pytest.fixture(scope="module")
def modules():
    """One product module per case on the GPU, shared by this file's tests (each call sets its own precision)."""
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = T.build_module(T.CASES[name]).to(DEV).train()
        return cache[name]

    yield get
    cache.clear()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name", list(T.CASES))
def test_fp32_training_step_at_size_matches_fp64_autograd(modules, name):
    ref = T.reference(name)
    losses, grads = T.product_step(name, modules(name), DEV)
    worst = T.check_fp32(name, losses, grads, ref)
    loss_err = max(abs(float(losses[k]) / float(v) - 1) for k, v in ref["losses"].items())
    print(f"\nAT_SIZE {name} fp32: worst max err / max|ref| {worst:.3e}, loss relative error {loss_err:.3e}")


@pytest.mark.parametrize("name", ["prod_ce", "ragged_ce"])
def test_bf16_training_step_at_size_is_close_to_fp64_autograd(modules, name):
    ref = T.reference(name)
    losses, grads = T.product_step(name, modules(name), DEV, precision=L.PREC_BF16)
    got, want = float(losses["loss"]), float(ref["losses"]["loss"])
    assert abs(got - want) <= 2e-2 * abs(want), f"{name} bf16 loss {got!r} vs fp64 {want!r}"
    top = T.largest_gradient(ref)
    worst, failures = 0.0, []
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
    assert not failures, f"{name} (bf16):\n  " + "\n  ".join(failures)
    assert worst > 1e-5, f"{name}: bf16 mode gave fp32-exact gradients: the tensor-core products were not used"
    print(f"\nAT_SIZE {name} bf16: worst max err / max|ref| {worst:.3e}")


@pytest.mark.parametrize("name", list(T.CASES))
def test_same_step_twice_gives_the_same_loss_and_gradients_up_to_the_order_of_atomics(modules, name):
    """Bit equality is not expected of the gradients: several kernels reduce through atomicAdd, whose order varies.
    The rounding of such a sum depends on its summands, not on its total.  The summands of some sums cancel: q_scale and
    k_scale sum one term per (sequence, head, query) row, folded in by one atomic per CTA.  Run to run, such a sum
    moves by more than 1e-6 of its own largest entry (1.5e-6 was seen at prod_ce).  So the bound is 1e-6 of the
    step's largest gradient entry, for every tensor."""
    ref = T.reference(name)
    top = T.largest_gradient(ref)
    l1, g1 = T.product_step(name, modules(name), DEV)
    l2, g2 = T.product_step(name, modules(name), DEV)
    for k in l1:
        assert torch.equal(l1[k], l2[k]), f"{name} {k}: {float(l1[k])!r} then {float(l2[k])!r}"
    worst = 0.0
    for k, a in g1.items():
        b = g2[k]
        assert (a is None) == (b is None), k
        if a is None or a.numel() == 0:
            continue
        diff = (a - b).abs().max().item()
        worst = max(worst, diff / top)
        assert diff <= 1e-6 * top, f"{name} {k}: runs differ by {diff:.3e}, the largest gradient is {top:.3e}"
    print(f"\nAT_SIZE {name} twice: largest difference / largest gradient {worst:.3e}")
