"""CPU: the fp32 training step with attention and FF dropout (csrc/train.cu, compiled by g++ for the CPU executor of
tests/cuda_emu) against the float64 autograd reference fed the masks rebuilt in numpy from the counter contract
(tests/dropout_ref.py).  ``tiny`` is small enough that one wrong mask element moves the loss far past the 1e-5 bar;
``emu_ragged_ce`` puts the dropout through the batched-product attention backward, partial tiles, masked text and video
tails and null-key columns.

Also: the library's counter count is the layout the contract describes; the step without dropout draws nothing."""
import ctypes
import os
import subprocess
import tempfile

import pytest
import torch

from phenaki_pytorch_b200 import _lib as L
from tests import dropout_ref as DR
from tests import emu_runtime
from tests import train_at_size_cases as T
from tests import train_dropout_cases as TD


@pytest.fixture(scope="module")
def emu():
    return emu_runtime.build_emu()


@pytest.fixture
def on_cpu(emu, monkeypatch):
    emu_runtime.route_product_to_emulator(emu, monkeypatch)


@pytest.mark.parametrize("name", ["tiny", "emu_ragged_ce"])
def test_emulated_dropout_step_matches_fp64_autograd_with_the_rebuilt_masks(on_cpu, name):
    torch.manual_seed(0)
    module = T.build_module(TD.case(name)).train()
    losses, grads, ref, calls = TD.run_and_reference(name, module, "cpu")
    assert len(calls) == 1
    T.check_fp32(name, losses, grads, ref)


@pytest.mark.parametrize("site", ["self", "cross", "ff"])
def test_one_wrong_mask_element_fails_the_parity_check(on_cpu, site):
    """The comparison above has the power to see a single mask element: flipping one element of one site of the
    reference's masks (the last layer's, whose gradients see it most directly) breaks the fp32 bars."""
    c = TD.case("tiny")
    module = T.build_module(c).train()
    with TD.record_rng() as calls:
        losses, grads = TD.product_step(c, module, "cpu")
    masks = TD.masks_of(c, module, calls[0][0], calls[0][1])
    m = masks[-1][site].view(-1)
    p = TD.FF_P if site == "ff" else TD.ATTN_P
    m[0] = 0.0 if m[0] != 0 else 1.0 / (1.0 - p)
    with pytest.raises(AssertionError):
        T.check_fp32("tiny", losses, grads, TD.reference(c, [masks]))


@pytest.mark.parametrize("attn_p,ff_p", [(1.0, 1.0), (1.0, 0.0), (0.0, 0.5)])
def test_emulated_extreme_and_single_site_probabilities(on_cpu, attn_p, ff_p):
    """p = 1 drops everything and gives zeros, not NaN; one probability at 0 leaves that site alone."""
    module = T.build_module(TD.case("tiny", attn_p, ff_p)).train()
    losses, grads, ref, calls = TD.run_and_reference("tiny", module, "cpu", attn_p=attn_p, ff_p=ff_p)
    assert all(torch.isfinite(v).all() for v in losses.values())
    assert all(g is None or torch.isfinite(g).all() for g in grads.values())
    # with everything dropped, the parameters before the dropped product get exactly zero gradients
    zero = {k for k, g in ref["grads"].items() if g.numel() and float(g.abs().max()) == 0.0}
    assert (attn_p == 1.0) == bool(zero)
    for k in zero:
        assert float(grads[k].abs().max()) == 0.0, k
    rest = {"losses": ref["losses"], "grads": {k: g for k, g in ref["grads"].items() if k not in zero}}
    T.check_fp32("tiny", losses, {k: g for k, g in grads.items() if k not in zero}, rest)


@pytest.mark.parametrize("name", ["tiny", "emu_ragged_ce", "emu_critic_split_head"])
def test_library_counter_count_is_the_contract_layout(on_cpu, emu, name):
    c = TD.case(name)
    module = T.build_module(c)
    table = module._table()
    n = 1
    for v in c["patch_shape"]:
        n *= v
    for L_ctx in (0, c["ctx_len"]):
        want = DR.layout(module, c["batch"], n, L_ctx)[1]
        assert emu.phk_maskgit_train_dropout_counters(ctypes.byref(table), c["batch"], n, L_ctx) == want


def test_emulated_eval_mode_and_zero_probabilities_draw_nothing(on_cpu):
    """Dropout off (eval mode, or both probabilities 0) is the plain step: no counters reserved, same loss as a module
    built without dropout."""
    plain = T.build_module(TD.case("tiny", 0.0, 0.0)).train()
    with TD.record_rng() as calls:
        base, _ = TD.product_step(TD.case("tiny", 0.0, 0.0), plain, "cpu")
        off = T.build_module(TD.case("tiny")).eval()
        got, _ = TD.product_step(TD.case("tiny"), off, "cpu")
    assert calls == []
    assert torch.equal(got["loss"], base["loss"])


def test_out_of_range_probability_is_rejected_before_the_call(on_cpu):
    module = T.build_module(TD.case("tiny")).train()
    module.transformer.ff_dropout = 1.5
    with TD.record_rng() as calls, pytest.raises(ValueError):
        TD.product_step(TD.case("tiny"), module, "cpu")
    assert calls == []


def test_dropout_struct_matches_the_c_layout():
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "phk.h"\nint main(){printf("%zu %zu %zu", sizeof(phk_dropout_t), ' \
          'offsetof(phk_dropout_t, seed), offsetof(phk_dropout_t, offset));return 0;}'
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "s.c")
        open(path, "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(emu_runtime.ROOT, "include"), path, "-o", os.path.join(d, "s")])
        got = [int(v) for v in subprocess.check_output([os.path.join(d, "s")]).split()]
    assert got == [ctypes.sizeof(L.DropoutT), L.DropoutT.seed.offset, L.DropoutT.offset.offset]
