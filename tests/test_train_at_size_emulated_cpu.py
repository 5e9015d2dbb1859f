"""CPU: the fp32 training step (csrc/train.cu, compiled by g++ for the CPU executor of tests/cuda_emu) at sizes past the
step's shape thresholds, against the float64 autograd reference of tests/train_at_size_cases.py -- the batched-product
attention backward (189 x 189 scores), the split-K wgrad of the position-bias MLP (1105 coordinate deltas) and of a
TokenCritic head (1040 rows), each with a partial last tile or slice.  In order and under a shuffled block / thread
schedule.  The bf16 mma.sync products are not compiled into the executor; tests/test_gpu_train_at_size.py covers them.

Also: the float64 oracle itself agrees with the float32 oracle at the ``ragged_ce`` shape."""
import pytest
import torch

from tests import emu_runtime
from tests import train_at_size_cases as T


@pytest.fixture(scope="module")
def emu():
    return emu_runtime.build_emu()


@pytest.fixture
def on_cpu(emu, monkeypatch):
    emu_runtime.route_product_to_emulator(emu, monkeypatch)


@pytest.fixture(params=[0, 1], ids=["in-order", "shuffled"])
def schedule(emu, request):
    emu.phk_emu_set_shuffle(request.param)
    yield request.param
    emu.phk_emu_set_shuffle(0)


@pytest.mark.parametrize("name", list(T.EMULATED_CASES))
def test_emulated_step_past_the_shape_thresholds_matches_fp64_autograd(on_cpu, schedule, name):
    module = T.build_module(T.ALL_CASES[name])
    losses, grads = T.product_step(name, module, "cpu")
    T.check_fp32(name, losses, grads, T.reference(name))


def test_fp64_oracle_gradients_match_the_fp32_oracle():
    """The oracle is dtype-generic: in float64 and float32 it computes the same loss and gradients up to fp32 rounding
    (1e-5 of each tensor's largest entry; the analytically zero tensors against the step's largest gradient)."""
    r64, r32 = T.reference("ragged_ce"), T.reference("ragged_ce", torch.float32)
    assert all(g.dtype == torch.float64 for g in r64["grads"].values())
    assert all(g.dtype == torch.float32 for g in r32["grads"].values())
    torch.testing.assert_close(r32["losses"]["loss"].double(), r64["losses"]["loss"], rtol=1e-6, atol=0)
    assert r32["grads"].keys() == r64["grads"].keys()
    top = T.largest_gradient(r64)
    for k, want in r64["grads"].items():
        if want.numel() == 0:  # the self-attention's (heads, 0, dim_head) null key / value
            continue
        scale = top if T.is_analytically_zero(k) else float(want.abs().max())
        err = float((r32["grads"][k].double() - want).abs().max())
        assert err <= 1e-5 * scale, f"{k}: {err:.3e} vs max|ref| {scale:.3e}"
