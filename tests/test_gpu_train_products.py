"""GPU: the training step's products one kernel at a time, against float64 of the operands each kernel consumed
(tests/train_products_ref.py), through the probe library of tests/train_probe.py:

  A. sgemm_batched on sgemm_strided_kernel (fp32) and hgemm_strided_kernel (bf16 mma.sync): the four stride
     combinations, M / N / K across the 64 x 64 x {16, 32} tile edges, two-level (sequence, head) batches, the three
     accumulate modes (NaN-prefilled overwrite, add onto a prefill, split-K with a partial and empty trailing slices),
     ldc > N with bit-exact sentinels;
  B. linear_fwd / dgrad_p / wgrad_p in F32 and BF16 at the shapes the training steps use;
  C. attention_backward in both modes (fp32: against float64 autograd of oracle.attention_core; bf16: scores bit-
     identical to fp32 mode, dS and the batched contractions against float64 of their own bf16 operands);
  D. colsum.
Each bf16 check also proves that a round-toward-zero and an unrounded-operand reference break its bar.  Run with -s to
read the worst err / bar of every case."""
import pytest
import torch

from phenaki_pytorch_b200 import _lib as L
from tests import train_probe
from tests import train_products_cases as TC

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")


def sync():
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def lib():
    return train_probe.load()


@pytest.fixture(autouse=True)
def _probe_errors(lib, monkeypatch):
    monkeypatch.setattr(L, "lib", lambda: lib)  # L.check reads the error message from the library that failed


def _s(id_, M, N, K, a_kfast, b_kfast, acc, **kw):
    return dict(id=id_, M=M, N=N, K=K, a_kfast=a_kfast, b_kfast=b_kfast, acc=acc, seed=len(id_) * 7 + M + K, **kw)


# A k-fast / B k-fast: S and dP (yes, yes), dS.kh and dgrad (yes, no), dS^T.qh, P^T.dO and wgrad (no, no)
STRIDED = [
    _s("S-dP-577x577x64", 577, 577, 64, True, True, 0, outer=2, div=8),
    _s("dP-63x65x32", 63, 65, 32, True, True, 1, outer=2, div=3),
    _s("dP-k1", 65, 63, 1, True, True, 0, outer=1, div=2),
    _s("dSkh-577x64x577", 577, 64, 577, True, False, 0, outer=2, div=2),
    _s("dSkh-65x128x33", 65, 128, 33, True, False, 1, outer=1, div=4),
    _s("dSkh-64x128x577", 64, 128, 577, True, False, 1, outer=2, div=1),
    _s("PTdO-577x64x577", 577, 64, 577, False, False, 0, outer=1, div=8),
    _s("dSTqh-64x32x31", 64, 32, 31, False, False, 1, outer=2, div=2),
    _s("dSTqh-1x64x15", 1, 64, 15, False, False, 0, outer=3, div=1),
    _s("unused-63x1x16", 63, 1, 16, False, True, 0, outer=2, div=2),
    _s("unused-577x63x33", 577, 63, 33, False, True, 1, outer=1, div=3),
    _s("split-K-wgrad-1025", 64, 64, 256, False, False, 2, k_total=1025, count=6),  # 4 x 256, 1, one empty slice
    _s("split-K-wgrad-3825", 64, 3, 256, False, False, 2, k_total=3825, count=16),  # 14 x 256, 241, one empty
    _s("split-K-33", 577, 65, 32, True, True, 2, k_total=33, count=3),              # 32, 1, one empty
]


@pytest.mark.parametrize("bf16", [False, True], ids=["f32", "bf16"])
@pytest.mark.parametrize("c", STRIDED, ids=lambda c: c["id"])
def test_strided_product(lib, c, bf16):
    TC.check_strided(lib, DEV, c, bf16, sync)


def _lin(op, M, N, K, **kw):
    return dict(id=f"{M}x{N}x{K}" + "".join(f"-{k}{int(v)}" for k, v in kw.items()), op=op, M=M, N=N, K=K,
                seed=M + N + K, **kw)


# rows M, nn.Linear(K -> N)
SHAPES = [
    (1152, 512, 512),    # q / out projection, b = 2, n = 576
    (1152, 2730, 512),   # FF1 (2 * inner)
    (1152, 512, 1365),   # FF2: K not a multiple of 8 (padded leading dimension)
    (154, 1024, 768),    # cross k,v on the text rows (2 * 77)
    (37, 96, 77),        # ragged everywhere
    (1, 64, 48),         # wgrad reduction below one MMA k-step and not a multiple of 8
    (7, 64, 48),
    (288, 65536, 512),   # logits head
    (128, 512, 3072),    # C-ViViT patch embeddings K1, K2
    (256, 512, 6144),
    (1025, 64, 64),      # fp32 wgrad split-K, last 256-row chunk of 1 row
    (3825, 64, 3),       # fp32 wgrad split-K, last chunk of 241 rows
]
LINEAR = [c for M, N, K in SHAPES for c in (
    _lin("fwd", M, N, K, bias=True), _lin("fwd", M, N, K, bias=True, residual=True),
    _lin("dgrad", M, N, K, acc=0), _lin("dgrad", M, N, K, acc=1), _lin("wgrad", M, N, K))]


@pytest.mark.parametrize("prec", [L.PREC_F32, L.PREC_BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("c", LINEAR, ids=lambda c: f"{c['op']}-{c['id']}")
def test_linear_product(lib, c, prec):
    TC.check_linear(lib, DEV, c, prec, sync)


@pytest.mark.parametrize("op,M,N,K", [("fwd", 1152, 2730, 512), ("fwd", 2730, 1152, 512), ("dgrad", 1152, 512, 1365),
                                      ("dgrad", 154, 1024, 768), ("wgrad", 7, 64, 48), ("wgrad", 288, 65536, 512)])
def test_linear_refuses_small_scratch(lib, op, M, N, K):
    TC.check_linear_workspace(lib, DEV, dict(op=op, M=M, N=N, K=K), sync)


def _att(id_, b, H, n, m, **kw):
    return dict(id=id_, b=b, H=H, n=n, m=m, seed=b * 100 + n + m, **kw)


ATTENTION = [
    _att("maskgit-self", 2, 8, 576, 576, bias="cpb"),
    _att("maskgit-cross", 2, 8, 576, 77, nnull=2, mask=True, cfg_null=True),
    _att("loop-4095", 2, 4, 63, 63, nnull=2, mask=True),         # n * nkt = 4095: warp-per-row contractions
    _att("batched-4096-cpb", 4, 8, 64, 64, bias="cpb"),          # n * nkt = 4096: the C-ViViT 8 x 8 spatial frame
    _att("cvivit-temporal", 128, 8, 9, 9, bias="alibi"),
    _att("dh32", 2, 4, 100, 98, nnull=2, dh=32, mask=True),
    _att("dh128", 2, 2, 80, 70, nnull=2, dh=128, bias="cpb"),    # all kDPL lane slots
]


@pytest.mark.parametrize("c", ATTENTION, ids=lambda c: c["id"])
def test_attention_backward_f32(lib, c):
    TC.check_attention_f32(lib, DEV, c, sync)


@pytest.mark.parametrize("c", ATTENTION, ids=lambda c: c["id"])
def test_attention_backward_bf16(lib, c):
    TC.check_attention_bf16(lib, DEV, c, sync)


@pytest.mark.parametrize("rows", [1, 63, 4097])
@pytest.mark.parametrize("cols", [1, 257, 65536])
def test_colsum(lib, rows, cols):
    TC.check_colsum(lib, DEV, rows, cols, sync)
