"""GPU: the fp32 single-problem GEMM (phk_gemm_bf16 epilogue 0, gemm_bf16_kernel<0, false>: 64-row ping-pong units,
residual and output through the TMA unit, or from the registers where the TMA unit cannot serve the call) bit for bit
against a reference built from the two-problem launch.

phk_gemm_bf16_x2 with no bias and a trivial second problem writes the fp32 accumulator of every element (same k16 steps
in the same order, the same tensor-core accumulation); the reference then adds the residual and then the bias in fp32,
the order the single-problem epilogue promises: C = (A W^T + residual) + bias."""
import pytest
import torch

from phenaki_pytorch_b200 import _lib as L

pytestmark = pytest.mark.gpu
DEV = "cuda"


def operands(M, N, K, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    a = torch.randn((M, K), generator=g, device=DEV).bfloat16()
    w = torch.randn((N, K), generator=g, device=DEV).bfloat16()
    res = torch.randn((M, N), generator=g, device=DEV)
    bias = torch.randn((N,), generator=g, device=DEV)
    return a, w, res, bias


def accumulator(a, w):
    """A W^T as the fp32 accumulator of the two-problem launch (no bias; the second problem is a dummy)."""
    (M, K), N = a.shape, w.shape[0]
    c = torch.empty((M, N), device=DEV)
    a2, w2, c2 = torch.zeros((1, 8), dtype=torch.bfloat16, device=DEV), torch.zeros((8, 8), dtype=torch.bfloat16,
                                                                                      device=DEV), torch.empty((1, 8), device=DEV)
    L.check(L.lib().phk_gemm_bf16_x2(L.ptr(a), K, L.ptr(w), K, L.ptr(c), N, M, N, K, None, L.ptr(a2), 8, L.ptr(w2), 8,
                                     L.ptr(c2), 8, 1, 8, 8, None, L.stream_ptr()), "phk_gemm_bf16_x2")
    return c


def gemm(a, w, c, ldc, bias=None, residual=None, seg=(0, 0, 0)):
    (M, K), N = a.shape, w.shape[0]
    L.check(L.lib().phk_gemm_bf16(L.ptr(a), K, L.ptr(w), K, L.ptr(c), ldc, M, N, K, L.ptr(bias), L.ptr(residual),
                                  seg[0], seg[1], seg[2], 0, L.stream_ptr()), "phk_gemm_bf16")


def same_bits(x, y):
    return x.shape == y.shape and torch.equal(x.contiguous().view(torch.int32), y.contiguous().view(torch.int32))


def check_modes(M, N, K, seed):
    """Residual in place (C == residual), separate, absent; each with and without a bias; two runs of a call agree."""
    a, w, res, bias = operands(M, N, K, seed)
    acc = accumulator(a, w)
    for b in (None, bias):
        for mode in ("inplace", "separate", "none"):
            ref = acc + res if mode != "none" else acc.clone()
            if b is not None:
                ref = ref + b
            outs = []
            for _ in range(2):
                if mode == "inplace":
                    c = res.clone()
                    gemm(a, w, c, N, bias=b, residual=c)
                else:
                    c = torch.full((M, N), float("nan"), device=DEV)
                    gemm(a, w, c, N, bias=b, residual=res if mode == "separate" else None)
                outs.append(c)
            assert same_bits(outs[0], outs[1]), (mode, b is not None)
            assert same_bits(outs[0], ref), (mode, b is not None)


# every M against every N (K rotating through its list), and every K at two (M, N)
MS = [1, 63, 64, 65, 127, 129, 2304, 4607, 4608, 4609]
NS = [8, 200, 512, 520]
KS = [8, 72, 512, 520, 1408, 1536]
SHAPES = sorted({(m, n, KS[(i + j) % len(KS)]) for i, m in enumerate(MS) for j, n in enumerate(NS)} |
                {(m, n, k) for (m, n) in ((4608, 512), (65, 200)) for k in KS})


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_bit_identical_to_accumulator_plus_residual_plus_bias(M, N, K):
    check_modes(M, N, K, seed=M * 7 + N * 3 + K)


# 64 x 128 units: 1, 12, 131, 132 and 133 of them (one wave, one wave + 1), 144 (two waves, 12 in the last) and 265
# (three waves, 1 in the last) on the 132 persistent CTAs
WAVES = [(64, 128), (768, 128), (131 * 64, 128), (132 * 64, 128), (133 * 64, 128), (72 * 64, 256), (265 * 64, 128)]


@pytest.mark.parametrize("M,N", WAVES)
def test_last_wave_unit_counts(M, N):
    check_modes(M, N, 520, seed=M + N)


def test_row_map():
    """seg (100, 128, 11): row m goes to (m // 100) * 128 + 11 + m % 100; the residual is read through the same map (in
    place) and the rows the map skips are untouched."""
    M, N, K = 1000, 512, 1408
    a, w, _, bias = operands(M, N, K, 5)
    acc = accumulator(a, w)
    rows = ((M + 99) // 100) * 128
    g = torch.Generator(device=DEV).manual_seed(6)
    c0 = torch.randn((rows, N), generator=g, device=DEV)
    idx = torch.tensor([(m // 100) * 128 + 11 + m % 100 for m in range(M)], device=DEV)
    rest = torch.ones(rows, dtype=torch.bool, device=DEV)
    rest[idx] = False
    for b in (None, bias):
        c = c0.clone()
        gemm(a, w, c, N, bias=b, residual=c, seg=(100, 128, 11))
        ref = acc + c0[idx]
        if b is not None:
            ref = ref + b
        assert same_bits(c[idx], ref)
        assert same_bits(c[rest], c0[rest])


@pytest.mark.parametrize("ldc,offset", [(520, 1), (516, 0), (515, 0), (516, 2)],
                         ids=["unaligned C", "ldc > N", "odd ldc", "8-byte aligned C"])
def test_strided_and_unaligned_output(ldc, offset):
    """C at a 4- or 8-byte offset (not 16-byte aligned) or with ldc > N: the residual is C itself; columns >= N of every
    row are untouched."""
    M, N, K = 4609, 512, 520
    a, w, res, bias = operands(M, N, K, 9)
    acc = accumulator(a, w)
    for b in (None, bias):
        buf = torch.full((M * ldc + offset + 8,), -7.0, device=DEV)
        c = buf[offset:offset + M * ldc].view(M, ldc)
        c[:, :N] = res
        gemm(a, w, c, ldc, bias=b, residual=c)
        ref = acc + res
        if b is not None:
            ref = ref + b
        assert same_bits(c[:, :N], ref)
        assert (c[:, N:] == -7.0).all() and (buf[:offset] == -7.0).all() and (buf[offset + M * ldc:] == -7.0).all()
