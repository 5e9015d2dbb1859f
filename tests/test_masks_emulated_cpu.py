"""CPU: tests/test_gpu_masks_and_self_critic.py a second time with the whole fp32 product path (classes, ctypes tables,
csrc drivers, every kernel incl. the training step's backward kernels) executed by tests/cuda_emu -- the same bodies and
bars as on the H100."""
import pytest
import torch

from tests import emu_runtime
from tests import test_gpu_masks_and_self_critic as M

for _n in [n for n in dir(M) if n.startswith("test_")]:
    globals()[_n] = getattr(M, _n)


@pytest.fixture(scope="module")
def _emu_lib():
    return emu_runtime.build_emu()


@pytest.fixture(autouse=True)
def _product_on_the_cpu(_emu_lib, monkeypatch):
    emu_runtime.route_product_to_emulator(_emu_lib, monkeypatch)
    monkeypatch.setattr(M, "DEV", "cpu")
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
