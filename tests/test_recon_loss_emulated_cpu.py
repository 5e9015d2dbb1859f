"""CPU: the C-ViViT reconstruction loss and its backward (phk_cvivit_recon_loss / phk_cvivit_backward through
``_ReconLossFn``) with the whole product path executed by the CPU executor of tests/cuda_emu, for the small fp32 cases
of tests/recon_loss_cases.py: the check bodies and bars of tests/test_gpu_recon_loss.py, in order and under a shuffled
block / thread schedule.  bf16 mode (wgmma) is covered on the GPU only."""
import pytest

from tests import emu_runtime
from tests import recon_loss_cases as RL

DEV = "cpu"


def _sync():
    pass


@pytest.fixture(scope="module")
def emu():
    return emu_runtime.build_emu()


@pytest.fixture
def on_cpu(emu, monkeypatch):
    emu_runtime.route_product_to_emulator(emu, monkeypatch)
    return emu


@pytest.fixture(params=[0, 1], ids=["in-order", "shuffled"])
def schedule(emu, request):
    emu.phk_emu_set_shuffle(request.param)
    yield request.param
    emu.phk_emu_set_shuffle(0)


@pytest.mark.parametrize("name", RL.SMALL)
def test_emulated_recon_loss_gradients_match_fp64_autograd(on_cpu, schedule, name):
    RL.check_fp32(DEV, _sync, RL.build_module(name), name)


@pytest.mark.parametrize("name", ["rect_mask", "image"])
def test_emulated_eval_mode_sends_nothing_to_the_encoder(on_cpu, name):
    RL.check_fp32(DEV, _sync, RL.build_module(name), name, training=False)


def test_emulated_return_recons_objective(on_cpu):
    RL.check_fp32(DEV, _sync, RL.build_module("rect"), "rect", with_recon=True)


@pytest.mark.parametrize("name", ["rect_mask", "image"])
def test_emulated_forward_outputs(on_cpu, name):
    RL.check_forward_outputs(DEV, _sync, RL.build_module(name), name)


def test_emulated_two_forwards_then_one_backward(on_cpu):
    RL.check_two_forwards_then_one_backward(DEV, _sync, RL.build_module("rect"), "rect")
