"""CPU (tests/cuda_emu): the training products' check bodies of tests/train_products_cases.py on the CPU executor, at
reduced sizes -- the fp32 strided batched product (sgemm_strided_kernel) in every stride / batch / accumulate mode, the
fp32 and bf16 nn.Linear products (the executor runs the real cast / cast-transpose kernels and represents the wgmma GEMM
by its include/phk.h contract, so bf16 mode's padding and transpose wiring is checked here too), the fp32 attention
backward against float64 autograd, colsum, and the scratch layout.  The executor has no hgemm_strided_kernel (bf16
products of the strided product fall back to the fp32 kernel there), so the bf16 strided and attention cases are
GPU-only: tests/test_gpu_train_products.py."""
import pytest
import torch

from phenaki_pytorch_b200 import _lib as L
from tests import train_probe
from tests import train_products_cases as TC

CPU = torch.device("cpu")


def _sync():
    pass


@pytest.fixture(scope="module")
def lib():
    return train_probe.load_emulated()


@pytest.fixture(autouse=True)
def _cpu(lib, monkeypatch):
    monkeypatch.setattr(L, "lib", lambda: lib)  # L.check reads the error message from the library that failed
    monkeypatch.setattr(L, "stream_ptr", lambda: None)


def _s(id_, M, N, K, a_kfast, b_kfast, acc, **kw):
    return dict(id=id_, M=M, N=N, K=K, a_kfast=a_kfast, b_kfast=b_kfast, acc=acc, seed=len(id_) * 7 + M, **kw)


STRIDED = [
    _s("S-dP", 65, 63, 32, True, True, 0, outer=2, div=3),
    _s("dSkh-dgrad", 63, 32, 65, True, False, 1, outer=2, div=2),
    _s("dSTqh-PTdO-wgrad", 64, 64, 31, False, False, 0, outer=1, div=3),
    _s("unused-combination", 1, 65, 33, False, True, 1, outer=2, div=2),
    _s("k1", 63, 1, 1, True, False, 0),
    _s("k15-k-tail", 65, 64, 15, False, False, 1, outer=3, div=1),
    _s("split-K-partial", 64, 64, 16, False, True, 2, k_total=57, count=5),  # slices 16 16 16 9 and one empty
    _s("split-K-1", 1, 33, 32, True, False, 2, k_total=33, count=3),        # slices 32 1 and one empty
]


@pytest.mark.parametrize("c", STRIDED, ids=lambda c: c["id"])
def test_strided_f32(lib, c):
    TC.check_strided(lib, CPU, c, False, _sync)


def _lin(op, M, N, K, **kw):
    return dict(id=f"{M}x{N}x{K}" + "".join(f"-{k}{int(v)}" for k, v in kw.items()), op=op, M=M, N=N, K=K,
                seed=M + N + K, **kw)


LINEAR = [
    _lin("fwd", 37, 96, 77, bias=True), _lin("fwd", 37, 96, 77, residual=True, bias=True),
    _lin("dgrad", 37, 96, 77, acc=0), _lin("dgrad", 37, 96, 77, acc=1), _lin("wgrad", 37, 96, 77),
    _lin("wgrad", 1, 64, 48), _lin("wgrad", 7, 64, 48), _lin("dgrad", 7, 64, 48, acc=1),
    _lin("fwd", 20, 40, 27, bias=True),     # K not a multiple of 8: padded leading dimension
    _lin("dgrad", 20, 27, 40, acc=0),       # N not a multiple of 8: the transposed W's padded rows
    _lin("wgrad", 1025, 64, 64),            # fp32: split-K over 256-row chunks, last chunk of 1 row
    _lin("wgrad", 1100, 16, 3),             # fp32: split-K, last chunk of 76 rows
]


@pytest.mark.parametrize("prec", [L.PREC_F32, L.PREC_BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("c", LINEAR, ids=lambda c: f"{c['op']}-{c['id']}")
def test_linear(lib, c, prec):
    TC.check_linear(lib, CPU, c, prec, _sync)


@pytest.mark.parametrize("op,M,N,K", [("fwd", 37, 96, 77), ("fwd", 96, 37, 77), ("dgrad", 20, 27, 40),
                                      ("dgrad", 40, 27, 20), ("wgrad", 7, 64, 48), ("wgrad", 7, 48, 64)])
def test_linear_refuses_small_scratch(lib, op, M, N, K):
    TC.check_linear_workspace(lib, CPU, dict(op=op, M=M, N=N, K=K), _sync)


def _att(id_, b, H, n, m, **kw):
    return dict(id=id_, b=b, H=H, n=n, m=m, seed=b * 100 + n + m, **kw)


ATTENTION = [
    _att("cross-cfg-null", 2, 2, 40, 20, nnull=2, mask=True, cfg_null=True),
    _att("loop-4095", 1, 2, 63, 63, nnull=2, dh=32, mask=True),      # n * nkt = 4095: warp-per-row contractions
    _att("batched-4096-cpb", 1, 2, 64, 64, dh=32, bias="cpb"),       # n * nkt = 4096: batched products
    _att("temporal-alibi", 6, 2, 9, 9, bias="alibi"),
    _att("dh128", 1, 1, 20, 30, nnull=1, dh=128, bias="cpb"),
]


@pytest.mark.parametrize("c", ATTENTION, ids=lambda c: c["id"])
def test_attention_backward_f32(lib, c):
    TC.check_attention_f32(lib, CPU, c, _sync)


@pytest.mark.parametrize("rows,cols", [(1, 1), (63, 257), (130, 1), (4097, 3), (70, 300)])
def test_colsum(lib, rows, cols):
    TC.check_colsum(lib, CPU, rows, cols, _sync)


def test_scratch_layout(lib):
    for c in ATTENTION + [_att("maskgit-cross", 2, 8, 576, 77, nnull=2)]:
        TC.check_layout(lib, c)
