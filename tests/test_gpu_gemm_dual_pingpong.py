"""GPU: the two-problem wgmma launches (phk_gemm_bf16_qkv, phk_gemm_bf16_x2) on the ping-pong body, bit for bit against
the single-problem launches of the same products, which run the quadrant body.  Both bodies accumulate every output
element in the same k-order (k-blocks of 64 in order, k = 16 steps in order), and the register epilogues round like
the staged ones, so the outputs must be identical -- not merely close.

The schedule cases give CTAs 1, 2, 3 and 5 tiles, a grid where one CTA gets one tile more than the rest, and two
problems whose k-block counts differ by 22x, so the warpgroup that skips the other warpgroup's tile in the ring has to
use the count of that tile's problem."""
import pytest
import torch

from phenaki_pytorch_b200 import _lib as L

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rand(shape, seed, scale=1.0):
    g = torch.Generator(device=DEV)
    g.manual_seed(seed)
    return torch.randn(shape, device=DEV, generator=g) * scale


def operands(M, N, K, seed):
    return rand((M, K), seed).bfloat16(), (rand((N, K), seed + 1) / K ** 0.5).bfloat16()


def gemm(a, w, c, bias=None, epi=0):
    M, K = a.shape
    L.check(L.lib().phk_gemm_bf16(L.ptr(a), K, L.ptr(w), K, L.ptr(c), c.stride(0), M, w.shape[0], K, L.ptr(bias), None,
                                  0, 0, 0, epi, L.stream_ptr()), "phk_gemm_bf16")


def gemm_x2(a1, w1, c1, b1, a2, w2, c2, b2):
    (M1, K1), (N1, _), (M2, K2), (N2, _) = a1.shape, w1.shape, a2.shape, w2.shape
    L.check(L.lib().phk_gemm_bf16_x2(L.ptr(a1), K1, L.ptr(w1), K1, L.ptr(c1), c1.stride(0), M1, N1, K1, L.ptr(b1),
                                     L.ptr(a2), K2, L.ptr(w2), K2, L.ptr(c2), c2.stride(0), M2, N2, K2, L.ptr(b2),
                                     L.stream_ptr()), "phk_gemm_bf16_x2")


def gemm_qkv(xn, xr, wq, wkv, qn, kvn, qs, ks):
    M, K = xn.shape
    L.check(L.lib().phk_gemm_bf16_qkv(L.ptr(xn), L.ptr(xr), K, L.ptr(wq), L.ptr(wkv), K, L.ptr(qn), L.ptr(kvn), M,
                                      wq.shape[0], K, L.ptr(qs), L.ptr(ks), 8.0, L.stream_ptr()), "phk_gemm_bf16_qkv")


def gemm_qnorm(xn, wq, qn, qs, sim_scale):
    M, K = xn.shape
    L.check(L.lib().phk_gemm_bf16_qnorm(L.ptr(xn), K, L.ptr(wq), K, L.ptr(qn), M, wq.shape[0], K, L.ptr(qs), sim_scale,
                                        L.stream_ptr()), "phk_gemm_bf16_qnorm")


def run_qkv(M, I, K, seed):
    xn, wq = operands(M, I, K, seed)
    xr, wkv = operands(M, 2 * I, K, seed + 2)
    qs, ks = rand((64,), seed + 4).abs() + 0.5, rand((64,), seed + 5).abs() + 0.5
    qn = torch.full((M, I), 7.0, dtype=torch.bfloat16, device=DEV)
    kvn = torch.full((M, 2 * I), 7.0, dtype=torch.bfloat16, device=DEV)
    gemm_qkv(xn, xr, wq, wkv, qn, kvn, qs, ks)
    return (xn, xr, wq, wkv, qs, ks), qn, kvn


QKV_SHAPES = ([(M, 512, 512) for M in (4608, 2304, 1152, 384, 1, 129, 1000)] +
              [(1000, 128, 72), (129, 1024, 520), (4608, 1024, 512), (384, 128, 520), (2304, 1024, 72), (1152, 512, 520)])


@pytest.mark.parametrize("M,I,K", QKV_SHAPES)
def test_qkv_equals_the_single_problem_kernels(M, I, K):
    """Qn and the k half of KVn equal phk_gemm_bf16_qnorm of the same operands, the v half equals the bf16 product."""
    (xn, xr, wq, wkv, qs, ks), qn, kvn = run_qkv(M, I, K, 100 + M + I + K)
    q1, k1 = torch.empty_like(qn), torch.empty_like(qn)
    v1 = torch.empty((M, I), dtype=torch.bfloat16, device=DEV)
    gemm_qnorm(xn, wq, q1, qs, 8.0)
    gemm_qnorm(xr, wkv[:I].contiguous(), k1, ks, 1.0)
    gemm(xr, wkv[I:].contiguous(), v1, epi=1)
    assert torch.equal(qn, q1)
    assert torch.equal(kvn[:, :I], k1)
    assert torch.equal(kvn[:, I:], v1)


def x2_against_single(p1, p2, seed, bias=True, offset=0):
    """phk_gemm_bf16_x2 of problems p1 = (M1, N1, K1), p2 against one phk_gemm_bf16 per problem.  offset > 0 writes
    C1 as a column view one float into a wider buffer: an odd ldc and a C that is only 4-byte aligned."""
    (M1, N1, K1), (M2, N2, K2) = p1, p2
    a1, w1 = operands(M1, N1, K1, seed)
    a2, w2 = operands(M2, N2, K2, seed + 2)
    b1, b2 = (rand((N1,), seed + 4), rand((N2,), seed + 5)) if bias else (None, None)

    def out1():
        return torch.full((M1, N1 + offset), 3.0, device=DEV)[:, offset:]

    c1, c2 = out1(), torch.full((M2, N2), 3.0, device=DEV)
    gemm_x2(a1, w1, c1, b1, a2, w2, c2, b2)
    r1, r2 = out1(), torch.full((M2, N2), 3.0, device=DEV)
    gemm(a1, w1, r1, b1)
    gemm(a2, w2, r2, b2)
    assert torch.equal(c1, r1)
    assert torch.equal(c2, r2)
    return c1, c2


def test_x2_patch_embeddings_equal_the_single_problem_kernel():
    x2_against_single((512, 512, 3072), (4096, 512, 6144), 200)


# (problem 1, problem 2): tiles per CTA on the 132-CTA grid in the comment
SCHEDULES = {
    "1 tile, K 64 vs 1408": ((128, 128, 64), (256, 128, 1408)),                  # 3 tiles, 3 CTAs
    "2 tiles": ((1024, 1024, 64), (2560, 1280, 1408)),                           # 64 + 200
    "3 tiles": ((1152, 512, 1408), (4608, 1280, 64)),                            # 36 + 360
    "5 tiles": ((4608, 2048, 64), (1536, 896, 1408)),                            # 576 + 84
    "one CTA gets 2, the rest 1": ((4224, 512, 64), (128, 128, 1408)),           # 132 + 1
    "ragged M, N, K": ((1001, 136, 200), (127, 384, 3072)),
}


@pytest.mark.parametrize("name", list(SCHEDULES))
def test_x2_schedules(name):
    x2_against_single(*SCHEDULES[name], 300 + len(name))


def test_x2_without_bias_and_unaligned_c():
    x2_against_single((300, 130, 72), (1000, 264, 512), 400, bias=False, offset=1)
    x2_against_single((4608, 512, 512), (4608, 1024, 512), 410, bias=True, offset=1)


def test_qkv_and_x2_are_deterministic():
    _, qn, kvn = run_qkv(4608, 512, 512, 500)
    _, qn2, kvn2 = run_qkv(4608, 512, 512, 500)
    assert torch.equal(qn, qn2) and torch.equal(kvn, kvn2)
    c1, c2 = x2_against_single((512, 512, 3072), (4096, 512, 6144), 510)
    d1, d2 = x2_against_single((512, 512, 3072), (4096, 512, 6144), 510)
    assert torch.equal(c1, d1) and torch.equal(c2, d2)
