"""CPU: the differentiable C-ViViT decode (phk_cvivit_decode_backward through ``_DecodeFn``) with the whole product path
executed by the CPU executor of tests/cuda_emu, for the small fp32 cases of tests/decode_grad_cases.py: the check bodies
and bars of tests/test_gpu_decode_backward.py, in order and under a shuffled block / thread schedule.  bf16 mode (wgmma)
and the profiler trace are covered on the GPU only."""
import pytest

from tests import decode_grad_cases as DG
from tests import emu_runtime

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


@pytest.mark.parametrize("entry", DG.ENTRIES)
@pytest.mark.parametrize("name", DG.SMALL)
def test_emulated_decode_gradients_match_fp64_autograd(on_cpu, schedule, name, entry):
    DG.check_fp32(DEV, _sync, DG.build_module(name), name, entry)


@pytest.mark.parametrize("name,entry", [("rect", "ids"), ("image", "tokens")])
def test_emulated_decode_values_are_unchanged_and_no_grad_builds_no_graph(on_cpu, name, entry):
    DG.check_forward_unchanged(DEV, _sync, DG.build_module(name), name, entry)


@pytest.mark.parametrize("name,entry", [("rect", "tokens"), ("cosine_vq", "ids")])
def test_emulated_two_decodes_then_one_backward(on_cpu, name, entry):
    DG.check_two_decodes_then_one_backward(DEV, _sync, DG.build_module(name), name, entry)


def test_emulated_create_graph_is_refused(on_cpu):
    DG.check_create_graph_refused(DEV, _sync, DG.build_module("image"), "image", "ids")


def test_emulated_modified_weight_is_refused(on_cpu):
    DG.check_modified_weight_refused(DEV, _sync, DG.build_module("image"), "image", "tokens")
