"""CPU: the differentiable ``CViViT.encode(tokens)`` (phk_cvivit_encode_tokens and phk_cvivit_encode_backward through
``_EncodeFn``) with the whole product path executed by the CPU executor of tests/cuda_emu, for three small fp32 cases of
tests/encode_grad_cases.py: the check bodies and bars of tests/test_gpu_zz_encode_backward.py.  bf16 mode (wgmma), the
golden comparisons and the profiler trace are covered on the GPU only."""
import pytest

from tests import emu_runtime
from tests import encode_grad_cases as EG

DEV = "cpu"
CASES = ["cfg1", "image", "cosine_vq"]


def _sync():
    pass


@pytest.fixture(scope="module")
def emu():
    return emu_runtime.build_emu()


@pytest.fixture
def on_cpu(emu, monkeypatch):
    emu_runtime.route_product_to_emulator(emu, monkeypatch)
    return emu


@pytest.mark.parametrize("name", CASES)
def test_emulated_encode_gradients_match_fp64_autograd(on_cpu, name):
    EG.check_fp32(DEV, _sync, EG.build_module(name), name)


@pytest.mark.parametrize("name", CASES)
def test_emulated_encode_values_are_unchanged_and_no_grad_builds_no_graph(on_cpu, name):
    EG.check_forward_unchanged(DEV, _sync, EG.build_module(name), name)


@pytest.mark.parametrize("name", CASES)
def test_emulated_encode_then_decode_gradients_match_fp64_autograd(on_cpu, name):
    EG.check_fp32(DEV, _sync, EG.build_module(name), name, then_decode=True)


@pytest.mark.parametrize("name", CASES)
def test_emulated_two_encodes_then_one_backward_accumulate(on_cpu, name):
    EG.check_two_encodes_then_one_backward(DEV, _sync, EG.build_module(name), name)


@pytest.mark.parametrize("name", CASES)
def test_emulated_encode_backward_is_deterministic(on_cpu, name):
    EG.check_deterministic(DEV, _sync, EG.build_module(name), name)
