"""GPU: the differentiable C-ViViT decode -- ``video = cvivit.decode(tokens)`` or ``decode_from_codebook_indices(ids)``,
then ``f(video).backward()`` through phk_cvivit_decode_backward -- against the float64 autograd reference of
tests/decode_grad_cases.py.

fp32 mode (and a split-bf16-mode module, whose backward runs fp32 products) is held to the training step's parity bars:
every gradient tensor, and d(tokens), within 1e-4 of its largest entry (max norm) and 2e-5 (relative Frobenius norm); the
analytically zero position-bias bias within 1e-6 of the largest gradient; the set of gradients left None is the
reference's.  bf16 mode is held to the training step's bf16 closeness bars.  The decode itself is unchanged: the same
values and the same kernel sequence with grad enabled as under no_grad."""
import json
import os
import subprocess
import sys

import pytest
import torch

from phenaki_pytorch_b200 import _lib as L
from tests import decode_grad_cases as DG

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _sync():
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def modules():
    """One product module per case on the GPU, shared by this file's tests (each call sets its own precision)."""
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = DG.build_module(name).to(DEV)
        return cache[name]

    yield get
    cache.clear()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("entry", DG.ENTRIES)
@pytest.mark.parametrize("name", DG.SMALL + ["at_size"])
def test_fp32_decode_gradients_match_fp64_autograd(modules, name, entry):
    worst = DG.check_fp32(DEV, _sync, modules(name), name, entry)
    print(f"\nDECODE_GRAD {name}/{entry} fp32: worst max err / max|ref| {worst:.3e}")


@pytest.mark.parametrize("name,entry", [("rect", "ids"), ("at_size", "tokens")])
def test_split_bf16_mode_differentiates_in_fp32(modules, name, entry):
    worst = DG.check_fp32(DEV, _sync, modules(name), name, entry, precision=L.PREC_BF16X3)
    print(f"\nDECODE_GRAD {name}/{entry} split-bf16: worst max err / max|ref| {worst:.3e}")


@pytest.mark.parametrize("entry", DG.ENTRIES)
@pytest.mark.parametrize("name", ["cfg1", "at_size"])
def test_bf16_decode_gradients_are_close_to_fp64_autograd(modules, name, entry):
    worst = DG.check_bf16(DEV, _sync, modules(name), name, entry)
    print(f"\nDECODE_GRAD {name}/{entry} bf16: worst max err / max|ref| {worst:.3e}")


@pytest.mark.parametrize("name,entry", [("rect", "ids"), ("image", "tokens"), ("cosine_vq", "ids")])
def test_decode_values_are_unchanged_and_no_grad_builds_no_graph(modules, name, entry):
    DG.check_forward_unchanged(DEV, _sync, modules(name), name, entry)


SEQUENCE_CASES = [(name, entry, precision) for name, entry in (("at_size", "ids"), ("rect", "tokens"))
                  for precision in (L.PREC_F32, L.PREC_BF16)]


@pytest.fixture(scope="module")
def kernel_sequences():
    """The profiler traces of tests/decode_grad_cases.py::kernel_sequences, taken in a process of their own: the
    profiler sessions of this file then leave no CUPTI / kineto state behind in the test process, whose later files
    trace kernels too."""
    code = (f"import json, sys; sys.path.insert(0, {ROOT!r}); from tests import decode_grad_cases as DG; "
            f"print(json.dumps(DG.kernel_sequences({SEQUENCE_CASES!r})))")
    flags = ["-s"] if sys.flags.no_user_site else []
    run = subprocess.run([sys.executable, *flags, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert run.returncode == 0, run.stderr[-4000:]
    return json.loads(run.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("name,entry,precision", SEQUENCE_CASES)
def test_decode_kernel_sequence_is_the_same_with_grad_enabled(kernel_sequences, name, entry, precision):
    a, b = kernel_sequences[f"{name}/{entry}/{precision}"]
    assert a and a == b, f"{name}: no_grad decode ran {len(a)} device ops, the graphed decode {len(b)}"


@pytest.mark.parametrize("name,entry", [("rect", "tokens"), ("at_size", "ids")])
def test_two_decodes_then_one_backward_accumulate(modules, name, entry):
    DG.check_two_decodes_then_one_backward(DEV, _sync, modules(name), name, entry)


@pytest.mark.parametrize("name,entry", [("cfg1", "ids"), ("at_size", "tokens")])
def test_decode_backward_is_deterministic_up_to_the_order_of_atomics(modules, name, entry):
    DG.check_deterministic(DEV, _sync, modules(name), name, entry)


def test_create_graph_is_refused(modules):
    DG.check_create_graph_refused(DEV, _sync, modules("rect"), "rect", "ids")


def test_modified_weight_is_refused():
    DG.check_modified_weight_refused(DEV, _sync, DG.build_module("rect").to(DEV), "rect", "tokens")
