"""GPU: ``CViViT.encode(tokens)`` -- the encoder's spatial and temporal stacks on patch tokens -- against the unmodified
reference's golden taps and the encode_ids path, and ``f(cvivit.encode(tokens)).backward()`` through
phk_cvivit_encode_backward against the float64 autograd reference of tests/encode_grad_cases.py.

fp32 mode is held to the decode backward's parity bars: every gradient tensor, and d(tokens), within 1e-4 of its largest
entry (max norm) and 2e-5 (relative Frobenius norm); the analytically zero position-bias bias within 1e-6 of the largest
gradient; the set of gradients left None is the reference's.  Split-bf16 mode differentiates in fp32 from the tokens and
must agree with fp32 mode; bf16 mode is held to the training step's bf16 closeness bars.  The encode itself is
unchanged by autograd: the same values and the same kernel sequence with grad enabled as under no_grad.

The file sorts after every other GPU file on purpose.  Several earlier files compare torch.profiler kernel traces taken
in the test process itself, and those traces lose their first kernel records once the process has run long enough: a
one-minute idle wait placed before tests/test_gpu_forward_backward.py makes its trace comparison fail just as this
file's minute of work did.  Running last, this file adds no time ahead of them."""
import json
import os
import subprocess
import sys

import pytest
import torch

import phenaki_pytorch_b200 as P
from phenaki_pytorch_b200 import _lib as L
from tests import cases as CS
from tests import encode_grad_cases as EG

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = {"f32": L.PREC_F32, "bf16x3": L.PREC_BF16X3, "bf16": L.PREC_BF16}


def _sync():
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def modules():
    """One product module per case on the GPU, shared by this file's tests (each call sets its own precision)."""
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = EG.build_module(name).to(DEV)
        return cache[name]

    yield get
    cache.clear()
    torch.cuda.empty_cache()


def _golden_module(name, mode):
    case = CS.CVIVIT_CASES[name]
    torch.manual_seed(case["seed"])
    model = P.CViViT(**case["ctor"]).to(DEV).eval()
    model.precision = MODES[mode]
    return case, model


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", list(CS.CVIVIT_CASES))
def test_encode_matches_reference_golden(golden, name, mode):
    """encode(patch) against the unmodified reference's temporal tap: test_gpu_models.py's fp32 bars in fp32 and
    split-bf16 modes, test_gpu_bf16_mode.py's in bf16 mode."""
    g = golden(f"cvivit_{name}")
    _, model = _golden_module(name, mode)
    with torch.no_grad():
        out = model.encode(g["patch"].to(DEV))
    b, t, h, w, d = g["patch"].shape
    got = out.cpu().permute(0, 2, 3, 1, 4).reshape(b * h * w, t, d)  # -> '(b h w) t d'
    if mode == "bf16":
        err = (got - g["temporal"]).abs() - (0.06 + 0.03 * g["temporal"].abs())
        assert float(err.max()) <= 0, f"{name}: bf16 encode exceeds |err| <= 0.06 + 0.03 |ref| by {float(err.max()):.3e}"
    else:
        torch.testing.assert_close(got, g["temporal"], rtol=2e-4, atol=2e-4)


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", list(CS.CVIVIT_CASES))
def test_encode_runs_the_same_stacks_as_encode_ids(name, mode):
    case, model = _golden_module(name, mode)
    video = CS.seeded_randn(case["video"], case["video_seed"]).to(DEV)
    video = video if video.ndim == 5 else video.unsqueeze(2)
    taps = {}
    model.encode_ids(video, taps=taps)
    with torch.no_grad():
        out = model.encode(taps["patch"])
    top = float(taps["temporal"].abs().max())
    diff = float((out - taps["temporal"]).abs().max())
    assert diff <= 1e-6 * top, f"{name}/{mode}: encode vs the encode_ids tap differ by {diff:.3e} (largest {top:.3e})"


@pytest.mark.parametrize("name", EG.SMALL + ["at_size"])
def test_fp32_encode_gradients_match_fp64_autograd(modules, name):
    worst = EG.check_fp32(DEV, _sync, modules(name), name)
    print(f"\nENCODE_GRAD {name} fp32: worst max err / max|ref| {worst:.3e}")


def test_encode_gradients_reach_only_the_encoder_stacks(modules):
    EG.check_encoder_grads_only(DEV, _sync, modules("rect"), "rect")


@pytest.mark.parametrize("name", ["rect", "at_size"])
def test_split_bf16_mode_gradients_equal_fp32_mode(modules, name):
    EG.check_split_bf16_equals_fp32(DEV, _sync, modules(name), name)


@pytest.mark.parametrize("name", ["cfg1", "at_size"])
def test_bf16_encode_gradients_are_close_to_fp64_autograd(modules, name):
    worst = EG.check_bf16(DEV, _sync, modules(name), name)
    print(f"\nENCODE_GRAD {name} bf16: worst max err / max|ref| {worst:.3e}")


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", ["rect", "image", "cosine_vq"])
def test_encode_values_are_unchanged_and_no_grad_builds_no_graph(modules, name, mode):
    EG.check_forward_unchanged(DEV, _sync, modules(name), name, MODES[mode])


SEQUENCE_CASES = [(name, precision) for name in ("at_size", "rect") for precision in (L.PREC_F32, L.PREC_BF16)]


@pytest.fixture(scope="module")
def kernel_sequences():
    """The profiler traces of tests/encode_grad_cases.py::kernel_sequences, taken in a process of their own (see
    tests/test_gpu_decode_backward.py)."""
    code = (f"import json, sys; sys.path.insert(0, {ROOT!r}); from tests import encode_grad_cases as EG; "
            f"print(json.dumps(EG.kernel_sequences({SEQUENCE_CASES!r})))")
    flags = ["-s"] if sys.flags.no_user_site else []
    run = subprocess.run([sys.executable, *flags, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert run.returncode == 0, run.stderr[-4000:]
    return json.loads(run.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("name,precision", SEQUENCE_CASES)
def test_encode_kernel_sequence_is_the_same_with_grad_enabled(kernel_sequences, name, precision):
    a, b = kernel_sequences[f"{name}/{precision}"]
    assert a and a == b, f"{name}: no_grad encode ran {len(a)} device ops, the graphed encode {len(b)}"


@pytest.mark.parametrize("name", ["rect", "image", "at_size"])
def test_encode_then_decode_gradients_match_fp64_autograd(modules, name):
    worst = EG.check_fp32(DEV, _sync, modules(name), name, then_decode=True)
    print(f"\nENCODE_DECODE_GRAD {name} fp32: worst max err / max|ref| {worst:.3e}")


@pytest.mark.parametrize("name", ["rect", "at_size"])
def test_two_encodes_then_one_backward_accumulate(modules, name):
    EG.check_two_encodes_then_one_backward(DEV, _sync, modules(name), name)


@pytest.mark.parametrize("name,precision", [("cfg1", L.PREC_F32), ("at_size", L.PREC_F32), ("at_size", L.PREC_BF16)])
def test_encode_backward_is_deterministic_up_to_the_order_of_atomics(modules, name, precision):
    EG.check_deterministic(DEV, _sync, modules(name), name, precision)


def test_create_graph_is_refused(modules):
    EG.check_create_graph_refused(DEV, _sync, modules("rect"), "rect")


def test_modified_weight_is_refused():
    EG.check_modified_weight_refused(DEV, _sync, EG.build_module("rect").to(DEV), "rect")


@pytest.mark.parametrize("name", ["rect", "cosine_vq"])
def test_bad_token_shapes_are_refused(modules, name):
    EG.check_bad_shapes_refused(DEV, _sync, modules(name), name)


@pytest.mark.parametrize("name", ["rect", "at_size"])
def test_short_workspace_is_refused(modules, name):
    EG.check_short_workspace_refused(DEV, _sync, modules(name), name)
