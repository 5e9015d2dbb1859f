"""CPU: the uint8-video checks of tests/test_gpu_encode_u8.py whose kernels are plain CUDA, EXECUTED ON THE CPU by
tests/cuda_emu: phk_patchify_ln_u8 against phk_patchify_ln on shapes that take the register kernel and each order of the
generic kernel, and the encode driver's ids and taps for the cfg1, rect and image cases in fp32 mode -- bit for bit
against the fp32 video divided on the CPU.  The TMA kernels are not part of the emulated build (the GPU file covers
them), so the shapes here are those where no fp32 call would take TMA beyond what the register kernel also serves."""
import numpy as np
import pytest
import torch

from phenaki_pytorch_b200 import _lib as L
from tests import emu_runtime
from tests import test_gpu_encode_u8 as G

EMULATED_SHAPES = ["p2_8", "w_36", "offset_1", "offset_2_p2_8", "k_6912", "p2_6", "p2_6_offset_1"]


@pytest.fixture(scope="module")
def _emu_lib():
    return emu_runtime.build_emu()


def test_uint8_quotients_are_the_correctly_rounded_ones():
    """The CPU division the fp32 reference videos use is IEEE division (numpy's float32 quotient)."""
    u = torch.arange(256, dtype=torch.uint8)
    assert torch.equal(G.as_float(u), torch.from_numpy(np.arange(256, dtype=np.float32) / np.float32(255)))


@pytest.mark.parametrize("name", EMULATED_SHAPES)
def test_patchify_ln_u8_equals_the_fp32_op(_emu_lib, monkeypatch, name):
    monkeypatch.setattr(L, "lib", lambda: _emu_lib)
    monkeypatch.setattr(L, "stream_ptr", lambda: None)
    shape, offset = G.KERNEL_SHAPES[name]
    G.check_patchify(shape, offset, "cpu")


@pytest.mark.parametrize("name", ["cfg1", "rect", "image"])
def test_encode_ids_and_taps_of_uint8_equal_the_fp32_video(_emu_lib, monkeypatch, name):
    emu_runtime.route_product_to_emulator(_emu_lib, monkeypatch)
    model, u = G.case_model(name, "cpu")
    model.precision = L.PREC_F32
    G.check_model(model, u, "cpu")


def test_other_dtypes_are_refused_before_any_launch(_emu_lib, monkeypatch):
    emu_runtime.route_product_to_emulator(_emu_lib, monkeypatch)
    model, u = G.case_model("image", "cpu")
    model.precision = L.PREC_F32
    model(u, return_only_codebook_ids=True)
    n0 = _emu_lib.phk_launch_count()
    for dtype in (torch.float16, torch.int16, torch.float64):
        with pytest.raises(L.PhkError, match="float32 or torch.uint8"):
            model(u.to(dtype), return_only_codebook_ids=True)
    assert _emu_lib.phk_launch_count() == n0
