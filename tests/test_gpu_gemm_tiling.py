"""GPU: the wgmma GEMMs (gemm_bf16_kernel<EPI, DUAL>, gemm_bf16_geglu_kernel) at the production shapes of the C-ViViT encode, the
MaskGit forward and the training step: which kernel instance each entry point launches, results against a float64
product of the same bf16 operands, bit-identical rows whatever the batch a row sits in, and run-to-run determinism.

Error bound of an fp32 output (not fitted): the products of bf16 operands are exact in fp32; each of the K accumulation
steps and the residual / bias additions rounds once, by at most 2u (u = 2^-24; 2u also covers truncating rather than
round-to-nearest tensor-core accumulation) relative to the magnitudes summed so far, and the result is rounded once:
|c - c64| <= 2 (K + 2) u (sum_k |a_k w_k| + |residual| + |bias|) + u |c64|.  A bf16 output adds one bf16 rounding:
2^-8 |c64|."""
import functools
import json
import os
import subprocess
import sys

import pytest
import torch

from phenaki_pytorch_b200 import _lib as L
from tests import cases as TC

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24


def bf16_operands(M, N, K, seed, lda=None, ldw=None):
    lda, ldw = lda or K, ldw or K
    a = torch.zeros((M, lda), dtype=torch.bfloat16)
    w = torch.zeros((N, ldw), dtype=torch.bfloat16)
    a[:, :K] = TC.seeded_randn((M, K), seed).bfloat16()
    w[:, :K] = TC.seeded_randn((N, K), seed + 1).bfloat16()
    return a, w


def ref64(a, w, K):
    a64, w64 = a[:, :K].double(), w[:, :K].double()
    return a64 @ w64.t(), a64.abs() @ w64.abs().t()


def fp32_bound(absdot, K, extra=0.0, exact=None):
    b = 2.0 * (K + 2) * U * (absdot + extra)
    return b + U * exact.abs() if exact is not None else b


def gemm(a, w, c, M, N, K, bias=None, residual=None, seg=(0, 0, 0), epi=0):
    L.check(L.lib().phk_gemm_bf16(L.ptr(a), a.shape[1], L.ptr(w), w.shape[1], L.ptr(c), c.shape[1], M, N, K, L.ptr(bias),
                                  L.ptr(residual), seg[0], seg[1], seg[2], epi, L.stream_ptr()), "phk_gemm_bf16")


def gemm_x2(a1, w1, c1, b1, a2, w2, c2, b2):
    (M1, K1), (N1, _), (M2, K2), (N2, _) = a1.shape, w1.shape, a2.shape, w2.shape
    L.check(L.lib().phk_gemm_bf16_x2(L.ptr(a1), K1, L.ptr(w1), K1, L.ptr(c1), N1, M1, N1, K1, L.ptr(b1), L.ptr(a2), K2,
                                     L.ptr(w2), K2, L.ptr(c2), N2, M2, N2, K2, L.ptr(b2), L.stream_ptr()), "phk_gemm_bf16_x2")


def gemm_qkv(xn, xr, wq, wkv, qn, kvn, qs, ks):
    M, K = xn.shape
    L.check(L.lib().phk_gemm_bf16_qkv(L.ptr(xn), L.ptr(xr), K, L.ptr(wq), L.ptr(wkv), K, L.ptr(qn), L.ptr(kvn), M,
                                      wq.shape[0], K, L.ptr(qs), L.ptr(ks), 8.0, L.stream_ptr()), "phk_gemm_bf16_qkv")


def gemm_qnorm(xn, wq, qn, qs):
    M, K = xn.shape
    L.check(L.lib().phk_gemm_bf16_qnorm(L.ptr(xn), K, L.ptr(wq), K, L.ptr(qn), M, wq.shape[0], K, L.ptr(qs), 8.0,
                                        L.stream_ptr()), "phk_gemm_bf16_qnorm")


def d(*ts):
    return [t.to(DEV) for t in ts]


# ---------------------------------------------------------------------------------------------------------------------
# dispatch: the entry point and epilogue select the instance; shape never does
# ---------------------------------------------------------------------------------------------------------------------
INSTANCES = {"gemm_bf16_kernel<0, false>", "gemm_bf16_kernel<1, false>", "gemm_bf16_geglu_kernel",
             "gemm_bf16_kernel<0, true>", "gemm_bf16_kernel<3, true>", "gemm_bf16_kernel<3, false>"}


def launched_instance(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if "gemm_bf16_" in e.name}
    found = {i for i in INSTANCES if any(i in n for n in names)}
    assert len(found) == 1, names
    return found.pop()


def single_case(M, N, K, epi):
    a, w = d(*bf16_operands(M, N, K, 1))
    if epi == 3:
        qs = torch.ones(64, device=DEV)
        out = torch.empty((M, N), dtype=torch.bfloat16, device=DEV)
        return lambda: gemm_qnorm(a, w, out, qs)
    out = torch.zeros((M, N // 2 if epi == 2 else N), dtype=torch.float32 if epi == 0 else torch.bfloat16, device=DEV)
    return lambda: gemm(a, w, out, M, N, K, residual=out if epi == 0 else None, epi=epi)


def dual_case(kind):
    if kind == "patch-embed x2":
        (a1, w1), (a2, w2) = bf16_operands(512, 512, 3072, 2), bf16_operands(4096, 512, 6144, 4)
        a1, w1, a2, w2 = d(a1, w1, a2, w2)
        c1, c2 = torch.empty((512, 512), device=DEV), torch.empty((4096, 512), device=DEV)
        return lambda: gemm_x2(a1, w1, c1, None, a2, w2, c2, None)
    (xn, wq), (xr, wkv) = bf16_operands(4608, 512, 512, 6), bf16_operands(4608, 1024, 512, 8)
    xn, wq, xr, wkv = d(xn, wq, xr, wkv)
    if kind == "q/kv x2":
        c1, c2 = torch.empty((4608, 512), device=DEV), torch.empty((4608, 1024), device=DEV)
        return lambda: gemm_x2(xn, wq, c1, None, xr, wkv, c2, None)
    qs = torch.ones(64, device=DEV)
    qn = torch.empty((4608, 512), dtype=torch.bfloat16, device=DEV)
    kvn = torch.empty((4608, 1024), dtype=torch.bfloat16, device=DEV)
    return lambda: gemm_qkv(xn, xr, wq, wkv, qn, kvn, qs, qs)


# name -> (launch builder, expected instance): every single-problem production product of the encode, the MaskGit
# forward and the training step, ragged shapes, and the dual launches
DISPATCH = {
    "encode out-proj +res": (lambda: single_case(4608, 512, 512, 0), "gemm_bf16_kernel<0, false>"),
    "encode FF1+GEGLU": (lambda: single_case(4608, 2816, 512, 2), "gemm_bf16_geglu_kernel"),
    "ragged GEGLU": (lambda: single_case(129, 256, 72, 2), "gemm_bf16_geglu_kernel"),
    "encode FF2 +res": (lambda: single_case(4608, 512, 1408, 0), "gemm_bf16_kernel<0, false>"),
    "maskgit cross q (qnorm)": (lambda: single_case(4608, 512, 512, 3), "gemm_bf16_kernel<3, false>"),
    "train bf16 out": (lambda: single_case(2304, 512, 512, 1), "gemm_bf16_kernel<1, false>"),
    "ragged tiny": (lambda: single_case(1, 8, 8, 0), "gemm_bf16_kernel<0, false>"),
    "ragged bf16": (lambda: single_case(129, 200, 72, 1), "gemm_bf16_kernel<1, false>"),
    "split-bf16 K' = 3 Kp": (lambda: single_case(4608, 512, 3 * 512, 0), "gemm_bf16_kernel<0, false>"),
    "patch-embed x2": (lambda: dual_case("patch-embed x2"), "gemm_bf16_kernel<0, true>"),
    "q/kv x2": (lambda: dual_case("q/kv x2"), "gemm_bf16_kernel<0, true>"),
    "qkv": (lambda: dual_case("qkv"), "gemm_bf16_kernel<3, true>"),
}


@functools.lru_cache(maxsize=1)
def observed_instances():
    """The kernel trace of every DISPATCH case, taken in a fresh process: a CUDA-activity trace taken after other GPU
    work of a long test session can come back empty."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-m", "tests.test_gpu_gemm_tiling"], cwd=root, capture_output=True,
                         text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-3000:]
    return json.loads(out.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("name", list(DISPATCH))
def test_dispatch(name):
    assert observed_instances()[name] == DISPATCH[name][1]


def test_dispatch_every_instance_reached():
    assert set(observed_instances().values()) == INSTANCES


# ---------------------------------------------------------------------------------------------------------------------
# against float64
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,N,K", [(1, 8, 8), (127, 130, 64), (129, 256, 72), (4609, 512, 520), (300, 1000, 1365)])
def test_fp32_bias_inplace_residual_against_float64(M, N, K):
    Kp = (K + 7) // 8 * 8
    a, w = bf16_operands(M, N, K, 10, lda=Kp, ldw=Kp)
    bias, res = TC.seeded_randn((N,), 12), TC.seeded_randn((M, N), 13)
    exact, absdot = ref64(a, w, K)
    exact = exact + res.double() + bias.double()
    ad, wd, bd = d(a, w, bias)
    c = res.clone().to(DEV)
    gemm(ad, wd, c, M, N, K, bias=bd, residual=c)
    err = (c.cpu().double() - exact).abs()
    assert (err <= fp32_bound(absdot, K, res.double().abs() + bias.double().abs(), exact)).all()


def test_row_map_against_float64():
    M, N, K = 1000, 384, 1408
    a, w = bf16_operands(M, N, K, 20)
    exact, absdot = ref64(a, w, K)
    ad, wd = d(a, w)
    c = torch.full((((M + 99) // 100) * 128, N), 5.0, device=DEV)
    gemm(ad, wd, c, M, N, K, seg=(100, 128, 11))
    idx = torch.tensor([(m // 100) * 128 + 11 + m % 100 for m in range(M)])
    assert ((c.cpu()[idx].double() - exact).abs() <= fp32_bound(absdot, K, exact=exact)).all()
    rest = torch.ones(c.shape[0], dtype=torch.bool)
    rest[idx] = False
    assert (c.cpu()[rest] == 5.0).all()


@pytest.mark.parametrize("M,N,K", [(129, 264, 200), (4608, 512, 512)])
def test_bf16_out_against_float64(M, N, K):
    a, w = bf16_operands(M, N, K, 30)
    bias = TC.seeded_randn((N,), 31)
    exact, absdot = ref64(a, w, K)
    exact = exact + bias.double()
    ad, wd, bd = d(a, w, bias)
    c = torch.empty((M, N), dtype=torch.bfloat16, device=DEV)
    gemm(ad, wd, c, M, N, K, bias=bd, epi=1)
    bound = fp32_bound(absdot, K, bias.double().abs()) * (1 + 2.0 ** -8) + 2.0 ** -8 * exact.abs()
    assert ((c.cpu().double() - exact).abs() <= bound).all()


def gelu64(x):
    return 0.5 * x * (1.0 + torch.erf(x / 2.0 ** 0.5))


@pytest.mark.parametrize("M", [127, 4608])
def test_geglu_against_float64(M):
    """The fitted GELU adds at most 2.4e-4 |v| (see the kernel) on top of the accumulation bound, propagated through
    gelu(g) v: |d/dg| <= 1.13 |v|, |d/dv| = |gelu(g)|."""
    N, K = 2816, 512
    a = TC.seeded_randn((M, K), 40).bfloat16()
    w = (TC.seeded_randn((N, K), 41) / K ** 0.5).bfloat16()
    exact, absdot = ref64(a, w, K)
    out = torch.empty((M, N // 2), dtype=torch.bfloat16, device=DEV)
    ad, wd = d(a, w)
    gemm(ad, wd, out, M, N, K, epi=2)
    ev, eg = exact.reshape(M, -1, 2, 64)[:, :, 0].reshape(M, -1), exact.reshape(M, -1, 2, 64)[:, :, 1].reshape(M, -1)
    bv, bg = absdot.reshape(M, -1, 2, 64)[:, :, 0].reshape(M, -1), absdot.reshape(M, -1, 2, 64)[:, :, 1].reshape(M, -1)
    ref = gelu64(eg) * ev
    bound = (1.13 * ev.abs() * fp32_bound(bg, K) + gelu64(eg).abs() * fp32_bound(bv, K) + 2.4e-4 * ev.abs() * (eg.abs() + 1)
             + 2.0 ** -8 * ref.abs() + 1e-30)
    assert ((out.cpu().double() - ref).abs() <= bound * 1.01).all()


def test_qkv_against_float64():
    """Epilogue 3: per-head l2 normalisation; the normalised values are O(1), so the accumulation error relative to the
    head's norm bounds the result, then one bf16 rounding."""
    M, I, K = 4609, 512, 512
    xn, wq = bf16_operands(M, I, K, 50)
    xr, wkv = bf16_operands(M, 2 * I, K, 52)
    qs, ks = TC.seeded_randn((64,), 54).abs() + 0.5, TC.seeded_randn((64,), 55).abs() + 0.5
    q64, qabs = ref64(xn, wq, K)
    kv64, kvabs = ref64(xr, wkv, K)

    def norm(x, s, mul):
        h = x.reshape(M, -1, 64)
        return (h / h.norm(dim=-1, keepdim=True) * s.double() * mul).reshape(M, -1)

    ref_q, ref_k, ref_v = norm(q64, qs, 8.0), norm(kv64[:, :I], ks, 1.0), kv64[:, I:]
    dd = d(xn, xr, wq, wkv, qs, ks)
    qn = torch.empty((M, I), dtype=torch.bfloat16, device=DEV)
    kvn = torch.empty((M, 2 * I), dtype=torch.bfloat16, device=DEV)
    gemm_qkv(*dd[:4], qn, kvn, dd[4], dd[5])

    def rel_bound(x, absdot, s, mul):  # relative accumulation error of a head (2x: the norm moves too) + fp32 steps
        hn = x.reshape(M, -1, 64).norm(dim=-1, keepdim=True)
        e = (fp32_bound(absdot, K).reshape(M, -1, 64).norm(dim=-1, keepdim=True) / hn)
        return ((2 * e + 8 * U) * s.double().max() * mul).expand(-1, -1, 64).reshape(M, -1)

    for got, ref, b in ((qn, ref_q, rel_bound(q64, qabs, qs, 8.0)), (kvn[:, :I], ref_k, rel_bound(kv64[:, :I], kvabs[:, :I], ks, 1.0)),
                        (kvn[:, I:], ref_v, fp32_bound(kvabs[:, I:], K))):
        assert ((got.cpu().double() - ref).abs() <= b + 2.0 ** -8 * ref.abs()).all()
    qn1 = torch.empty_like(qn)
    gemm_qnorm(dd[0], dd[2], qn1, dd[4])
    assert torch.equal(qn1, qn)


def test_dual_problems_differ_in_m_n_k_and_bias():
    (a1, w1), (a2, w2) = bf16_operands(127, 384, 3072, 60), bf16_operands(1001, 136, 200, 62)
    b1, b2 = TC.seeded_randn((384,), 64), TC.seeded_randn((136,), 65)
    dd = d(a1, w1, a2, w2, b1, b2)
    c1, c2 = torch.zeros((127, 384), device=DEV), torch.zeros((1001, 136), device=DEV)
    gemm_x2(dd[0], dd[1], c1, dd[4], dd[2], dd[3], c2, dd[5])
    for c, a, w, b, K in ((c1, a1, w1, b1, 3072), (c2, a2, w2, b2, 200)):
        exact, absdot = ref64(a, w, K)
        exact = exact + b.double()
        assert ((c.cpu().double() - exact).abs() <= fp32_bound(absdot, K, b.double().abs(), exact)).all()


# ---------------------------------------------------------------------------------------------------------------------
# row invariance and determinism
# ---------------------------------------------------------------------------------------------------------------------
PRODUCTS = [("out-proj +res", 512, 512, 0), ("FF2 +res", 512, 1408, 0), ("FF1+GEGLU", 2816, 512, 2),
            ("bf16 out", 512, 512, 1), ("qnorm", 512, 512, 3), ("patch-embed rest", 512, 6144, 0)]


def run_product(kind, N, K, epi, a, w, res):
    M = a.shape[0]
    if epi == 3:
        out = torch.empty((M, N), dtype=torch.bfloat16, device=DEV)
        gemm_qnorm(a, w, out, torch.full((64,), 1.25, device=DEV))
        return out
    out = res.clone() if epi == 0 else torch.empty((M, N // 2 if epi == 2 else N), dtype=torch.bfloat16, device=DEV)
    gemm(a, w, out, M, N, K, residual=out if epi == 0 else None, epi=epi)
    return out


@pytest.mark.parametrize("kind,N,K,epi", PRODUCTS, ids=[p[0] for p in PRODUCTS])
def test_rows_do_not_depend_on_the_batch(kind, N, K, epi):
    """Rows [576 i, 576 (i + 1)) of the M = 4608 product equal the M = 576 product of the same rows bit for bit, and
    rows near the tile edges equal the same rows inside a larger product; two calls give identical bits."""
    a, w = bf16_operands(4609, N, K, 70)
    a, w = d(a, w)
    res = TC.seeded_randn((4609, N), 72).to(DEV)
    full = run_product(kind, N, K, epi, a[:4608], w, res[:4608])
    assert torch.equal(full, run_product(kind, N, K, epi, a[:4608], w, res[:4608]))
    for i in (0, 3, 7):
        r = slice(576 * i, 576 * (i + 1))
        assert torch.equal(run_product(kind, N, K, epi, a[r].contiguous(), w, res[r].contiguous()), full[r]), i
    for m in (1, 127, 129):
        assert torch.equal(run_product(kind, N, K, epi, a[:m].contiguous(), w, res[:m].contiguous()), full[:m]), m
    big = run_product(kind, N, K, epi, a, w, res)
    assert torch.equal(big[:4608], full)


def test_dual_rows_do_not_depend_on_the_batch():
    (xn, wq), (xr, wkv) = bf16_operands(4608, 512, 512, 80), bf16_operands(4608, 1024, 512, 82)
    xn, wq, xr, wkv = d(xn, wq, xr, wkv)
    qs = torch.full((64,), 1.25, device=DEV)

    def qkv(m):
        qn = torch.empty((m, 512), dtype=torch.bfloat16, device=DEV)
        kvn = torch.empty((m, 1024), dtype=torch.bfloat16, device=DEV)
        gemm_qkv(xn[:m].contiguous(), xr[:m].contiguous(), wq, wkv, qn, kvn, qs, qs)
        return qn, kvn

    q_full, kv_full = qkv(4608)
    q_576, kv_576 = qkv(576)
    assert torch.equal(q_576, q_full[:576]) and torch.equal(kv_576, kv_full[:576])
    q_again, kv_again = qkv(4608)
    assert torch.equal(q_again, q_full) and torch.equal(kv_again, kv_full)


if __name__ == "__main__":
    print(json.dumps({name: launched_instance(build()) for name, (build, _) in DISPATCH.items()}))
