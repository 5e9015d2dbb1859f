"""CPU: the differentiable MaskGit / TokenCritic / SelfCritic forwards (phk_maskgit_backward through
``_ForwardBackwardFn``) with the whole product path executed by the CPU executor of tests/cuda_emu, for the small fp32
cases of tests/forward_grad_cases.py: the check bodies and bars of tests/test_gpu_forward_backward.py, in order and under a
shuffled block / thread schedule.  bf16 mode (wgmma) and the profiler trace are covered on the GPU only."""
import pytest
import torch

from tests import emu_runtime
from tests import forward_grad_cases as FG
from tests import train_at_size_cases as T

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


def _module(name):
    return T.build_module(FG.ALL_CASES[name]["base"])


@pytest.mark.parametrize("name", list(FG.EMULATED_CASES))
def test_emulated_forward_gradients_match_fp64_autograd(on_cpu, schedule, name):
    FG.check_fp32(on_cpu, DEV, _sync, _module(name), name)


def test_emulated_cross_entropy_through_the_forward_matches_the_train_step(on_cpu):
    FG.check_matches_train_step(on_cpu, DEV, _sync, _module("emu_logits"), FG.SMALL_MASKGIT)


@pytest.mark.parametrize("name", ["emu_logits", "emu_critic_cfg", "emu_self_critic"])
def test_emulated_forward_values_are_unchanged_and_no_grad_builds_no_graph(on_cpu, name):
    FG.check_forward_unchanged(on_cpu, DEV, _sync, _module(name), name)


@pytest.mark.parametrize("name", ["emu_logits_cfg", "emu_self_critic"])
def test_emulated_two_forwards_then_one_backward(on_cpu, name):
    FG.check_two_forwards_then_one_backward(on_cpu, DEV, _sync, _module(name), name)


def test_emulated_create_graph_is_refused(on_cpu):
    FG.check_create_graph_refused(on_cpu, DEV, _sync, _module("emu_logits"), "emu_logits")


def test_emulated_unsupported_configuration_raises(on_cpu):
    FG.check_unsupported_configuration_raises(on_cpu, DEV, _sync)
