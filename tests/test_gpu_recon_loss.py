"""GPU: the C-ViViT reconstruction loss -- ``loss = cvivit(video, mask=...); loss.backward()`` through
phk_cvivit_backward -- against the float64 autograd reference of tests/recon_loss_cases.py.

fp32 mode (and a split-bf16-mode module, whose backward runs fp32 products) is held to the decode backward's bars: the
loss within 1e-6 relative, every gradient tensor and d video within 1e-4 of its largest entry (max norm) and 2e-5
(relative Frobenius norm), the analytically zero position-bias bias within 1e-6 of the largest gradient, and the set of
gradients left None equal to the reference's.  bf16 mode is held to the training step's bf16 closeness bars."""
import pytest
import torch

from phenaki_pytorch_b200 import _lib as L
from tests import recon_loss_cases as RL

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _sync():
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def modules():
    """One product module per case on the GPU, shared by this file's tests (each call sets its own precision)."""
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = RL.build_module(name).to(DEV)
        return cache[name]

    yield get
    cache.clear()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name", RL.SMALL + ["at_size"])
def test_fp32_recon_loss_gradients_match_fp64_autograd(modules, name):
    worst = RL.check_fp32(DEV, _sync, modules(name), name)
    print(f"\nRECON_GRAD {name} fp32: worst max err / max|ref| {worst:.3e}")


@pytest.mark.parametrize("name", ["rect_mask", "image", "at_size"])
def test_eval_mode_sends_nothing_to_the_encoder(modules, name):
    RL.check_fp32(DEV, _sync, modules(name), name, training=False)


@pytest.mark.parametrize("name", ["rect", "image"])
def test_return_recons_objective(modules, name):
    RL.check_fp32(DEV, _sync, modules(name), name, with_recon=True)


@pytest.mark.parametrize("name", ["rect_mask", "at_size"])
def test_split_bf16_mode_differentiates_in_fp32(modules, name):
    worst = RL.check_fp32(DEV, _sync, modules(name), name, precision=L.PREC_BF16X3)
    print(f"\nRECON_GRAD {name} split-bf16: worst max err / max|ref| {worst:.3e}")


@pytest.mark.parametrize("name", ["cfg1", "at_size"])
def test_bf16_recon_loss_gradients_are_close_to_fp64_autograd(modules, name):
    worst = RL.check_bf16(DEV, _sync, modules(name), name)
    print(f"\nRECON_GRAD {name} bf16: worst max err / max|ref| {worst:.3e}")


@pytest.mark.parametrize("name", ["rect_mask", "image", "at_size"])
def test_forward_outputs_match_the_inference_path(modules, name):
    RL.check_forward_outputs(DEV, _sync, modules(name), name)


def test_two_forwards_then_one_backward_accumulate(modules):
    RL.check_two_forwards_then_one_backward(DEV, _sync, modules("rect"), "rect")


@pytest.mark.parametrize("name", ["cfg1", "at_size"])
def test_recon_loss_backward_is_deterministic_up_to_the_order_of_atomics(modules, name):
    RL.check_deterministic(DEV, _sync, modules(name), name)


@pytest.mark.parametrize("name", ["rect_mask", "image"])
def test_cpu_rng_draw_matches_the_reference(modules, name):
    RL.check_cpu_rng_draw(DEV, _sync, modules(name), name)


def test_refused_cases():
    RL.check_refusals(DEV, _sync, RL.build_module("rect").to(DEV), "rect")
