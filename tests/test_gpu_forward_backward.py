"""GPU: the differentiable MaskGit / TokenCritic / SelfCritic forwards -- ``out = module(...); f(out).backward()``
through phk_maskgit_backward -- against the float64 autograd reference of tests/forward_grad_cases.py.

fp32 mode (and a split-bf16-mode module, whose backward runs fp32 products) is held to the training step's parity bars:
every gradient tensor, and d(text_embeds), within 1e-4 of its largest entry (max norm) and 2e-5 (relative Frobenius
norm); the analytically zero position-bias bias within 1e-6 of the largest gradient; the set of gradients left None is
the reference's.  bf16 mode is held to the training step's bf16 closeness bars.  The forward itself is unchanged: the
same values and the same kernel sequence with grad enabled as under no_grad."""
import json
import os
import subprocess
import sys

import pytest
import torch
from torch.profiler import ProfilerActivity, profile

from phenaki_pytorch_b200 import _lib as L
from tests import forward_grad_cases as FG
from tests import train_at_size_cases as T

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _sync():
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def lib():
    return L.lib()


@pytest.fixture(scope="module")
def modules():
    """One product module per base case on the GPU, shared by this file's tests (each call sets its own precision)."""
    cache = {}

    def get(name):
        base = FG.ALL_CASES[name]["base"]
        key = id(base)
        if key not in cache:
            cache[key] = T.build_module(base).to(DEV).train()
        return cache[key]

    yield get
    cache.clear()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name", list(FG.CASES))
def test_fp32_forward_gradients_match_fp64_autograd(lib, modules, name):
    worst = FG.check_fp32(lib, DEV, _sync, modules(name), name)
    print(f"\nFORWARD_GRAD {name} fp32: worst max err / max|ref| {worst:.3e}")


@pytest.mark.parametrize("name", FG.BF16_CASES)
def test_bf16_forward_gradients_are_close_to_fp64_autograd(lib, modules, name):
    worst = FG.check_bf16(lib, DEV, _sync, modules(name), name)
    print(f"\nFORWARD_GRAD {name} bf16: worst max err / max|ref| {worst:.3e}")


@pytest.mark.parametrize("base", ["prod_ce", "ragged_ce"])
def test_cross_entropy_through_the_forward_matches_the_train_step(lib, modules, base):
    name = "prod_logits" if base == "prod_ce" else "ragged_logits"
    worst = FG.check_matches_train_step(lib, DEV, _sync, modules(name), base)
    print(f"\nFORWARD_GRAD {base} vs train_step: worst err / bound {worst:.3e}")


@pytest.mark.parametrize("name", ["ragged_logits", "ragged_embeds_cfg", "prod_critic_cfg", "ragged_self_critic"])
def test_forward_values_are_unchanged_and_no_grad_builds_no_graph(lib, modules, name):
    FG.check_forward_unchanged(lib, DEV, _sync, modules(name), name)


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _device_ops(fn):
    """Names of the device ops fn runs, in start order, bracketed by two marker fills: a capture counts only when it
    begins and ends with a marker, i.e. when the profiler kept every record of the session."""
    marker = torch.zeros(1, device=DEV)
    _sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        marker.fill_(1.0)
        fn()
        marker.fill_(2.0)
        _sync()
    ops = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    names = [e.name for e in sorted(ops, key=lambda e: e.time_range.start)]
    assert len(names) >= 2 and "FillFunctor" in names[0] and "FillFunctor" in names[-1], \
        f"incomplete profiler capture: {len(names)} ops, {names[:2]} ... {names[-2:]}"
    return names[1:-1]


def kernel_sequences(name):
    """(device ops of the no_grad forward, device ops of the forward with grad enabled) in bf16 mode, after a warm-up
    of both (position-bias cache, workspace).  Run in a fresh process: late in a long test process the profiler drops
    the first records of a session (a capture once began at the forward's first device-to-host copy)."""
    module = T.build_module(FG.ALL_CASES[name]["base"]).to(DEV).train()
    FG.set_precision(module, L.PREC_BF16)

    def plain():
        with torch.no_grad():
            FG.product_out(name, module, DEV)

    def graphed():
        FG.product_out(name, module, DEV)

    plain(), graphed()
    return _device_ops(plain), _device_ops(graphed)


def _child(fn, *args):
    code = (f"import json, sys; sys.path.insert(0, {ROOT!r}); from tests import test_gpu_forward_backward as T; "
            f"print(json.dumps(T.{fn}(*{args!r})))")
    flags = ["-s"] if sys.flags.no_user_site else []
    run = subprocess.run([sys.executable, *flags, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert run.returncode == 0, run.stderr[-4000:]
    return json.loads(run.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("name", ["ragged_logits_cfg", "prod_critic", "ragged_self_critic_cfg"])
def test_forward_kernel_sequence_is_the_same_with_grad_enabled(name):
    a, b = _child("kernel_sequences", name)
    assert a and a == b, f"{name}: no_grad forward ran {len(a)} device ops, the graphed forward {len(b)}"


@pytest.mark.parametrize("name", ["ragged_logits_cfg", "ragged_self_critic"])
def test_two_forwards_then_one_backward_accumulate(lib, modules, name):
    FG.check_two_forwards_then_one_backward(lib, DEV, _sync, modules(name), name)


@pytest.mark.parametrize("name", ["prod_logits_cfg", "ragged_self_critic_cfg"])
def test_backward_is_deterministic_up_to_the_order_of_atomics(lib, modules, name):
    FG.check_deterministic(lib, DEV, _sync, modules(name), name)


def test_create_graph_is_refused(lib, modules):
    FG.check_create_graph_refused(lib, DEV, _sync, modules("ragged_logits"), "ragged_logits")


def test_unsupported_configuration_raises(lib):
    FG.check_unsupported_configuration_raises(lib, DEV, _sync)
