"""GPU: the wgmma/TMA bf16 GEMM (phk_gemm_bf16) against torch fp32 matmul of the SAME bf16-rounded
operands (so the only difference is fp32 summation order: tolerance 2e-3 * sqrt(K/512) absolute on O(sqrt(K)) sums)."""
import pytest
import torch

from phenaki_pytorch_b200 import _lib as L
from tests import cases as TC

pytestmark = pytest.mark.gpu
DEV = "cuda"


def operands(M, N, K, lda=None, ldw=None, seed=0):
    lda, ldw = lda or K, ldw or K
    a = torch.zeros((M, lda))
    w = torch.zeros((N, ldw))
    a[:, :K] = TC.seeded_randn((M, K), seed)
    w[:, :K] = TC.seeded_randn((N, K), seed + 1)
    return a.bfloat16(), w.bfloat16()


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 128, 512), (4608, 512, 512), (300, 200, 520), (77, 64, 48),
                                   (129, 1024, 768), (512, 512, 3072), (1000, 40, 136)])
def test_gemm_bf16_fp32_out_bias_residual(M, N, K):
    a, w = operands(M, N, K)
    bias, res = TC.seeded_randn((N,), 5), TC.seeded_randn((M, N), 6)
    ref = a.float() @ w.float().t() + bias + res
    ad, wd, bd = a.to(DEV), w.to(DEV), bias.to(DEV)
    c = res.clone().to(DEV)
    L.check(L.lib().phk_gemm_bf16(L.ptr(ad), K, L.ptr(wd), K, L.ptr(c), N, M, N, K, L.ptr(bd), L.ptr(c), 0, 0, 0, 0,
                                  L.stream_ptr()), "phk_gemm_bf16")
    torch.cuda.synchronize()
    torch.testing.assert_close(c.cpu(), ref, rtol=1e-4, atol=2e-3 * max(1.0, (K / 512) ** 0.5))


def test_gemm_bf16_padded_leading_dims_and_row_map():
    M, N, K = 130, 96, 1365           # FF second linear of the reference: K = int(4*2/3*512) (attention.py:46)
    a, w = operands(M, N, K, lda=1408, ldw=1408)
    ref = a[:, :K].float() @ w[:, :K].float().t()
    ad, wd = a.to(DEV), w.to(DEV)
    c = torch.zeros((400, N), device=DEV)
    L.check(L.lib().phk_gemm_bf16(L.ptr(ad), 1408, L.ptr(wd), 1408, L.ptr(c), N, M, N, K, None, None, 10, 30, 7, 0,
                                  L.stream_ptr()), "phk_gemm_bf16")
    idx = torch.tensor([(m // 10) * 30 + 7 + m % 10 for m in range(M)])
    torch.testing.assert_close(c.cpu()[idx], ref, rtol=1e-4, atol=4e-3)
    rest = torch.ones(400, dtype=torch.bool)
    rest[idx] = False
    assert (c.cpu()[rest] == 0).all()


@pytest.mark.parametrize("M,N,K", [(256, 256, 512), (100, 72, 200)])
def test_gemm_bf16_bf16_out(M, N, K):
    a, w = operands(M, N, K, seed=3)
    bias = TC.seeded_randn((N,), 9)
    ref = (a.float() @ w.float().t() + bias)
    ad, wd, bd = a.to(DEV), w.to(DEV), bias.to(DEV)
    c = torch.empty((M, N), dtype=torch.bfloat16, device=DEV)
    L.check(L.lib().phk_gemm_bf16(L.ptr(ad), K, L.ptr(wd), K, L.ptr(c), N, M, N, K, L.ptr(bd), None, 0, 0, 0, 1,
                                  L.stream_ptr()), "phk_gemm_bf16")
    torch.testing.assert_close(c.cpu().float(), ref, rtol=1e-2, atol=5e-2)  # one bf16 rounding of O(sqrt(K)) values


@pytest.mark.parametrize("M,inner,K", [(300, 1365, 512), (64, 170, 64)])
def test_gemm_bf16_geglu_epilogue(M, inner, K):
    """W rows packed [64 value | 64 gate] per 128-column tile; out = gelu(gate) * value (attention.py:40-43)."""
    inner_pad = (inner + 63) // 64 * 64
    a = TC.seeded_randn((M, K), 11).bfloat16()
    w1 = (TC.seeded_randn((2 * inner, K), 12) / K ** 0.5).bfloat16()
    packed = torch.zeros((2 * inner_pad, K), dtype=torch.bfloat16)
    for g in range(inner_pad // 64):
        lo, hi = g * 64, min(g * 64 + 64, inner)
        if hi > lo:
            packed[g * 128: g * 128 + (hi - lo)] = w1[lo:hi]                       # values
            packed[g * 128 + 64: g * 128 + 64 + (hi - lo)] = w1[inner + lo: inner + hi]   # gates
    h = a.float() @ w1.float().t()
    ref = torch.nn.functional.gelu(h[:, inner:]) * h[:, :inner]
    ad, wd = a.to(DEV), packed.to(DEV)
    out = torch.full((M, inner_pad), 7.0, dtype=torch.bfloat16, device=DEV)
    L.check(L.lib().phk_gemm_bf16(L.ptr(ad), K, L.ptr(wd), K, L.ptr(out), inner_pad, M, 2 * inner_pad, K, None, None,
                                  0, 0, 0, 2, L.stream_ptr()), "phk_gemm_bf16")
    o = out.cpu().float()
    torch.testing.assert_close(o[:, :inner], ref, rtol=1e-2, atol=1e-2)
    assert (o[:, inner:] == 0).all()  # K-padding of the next GEMM must be exact zeros


@pytest.mark.parametrize("n_seq,n,heads,with_bias", [(2, 576, 8, True), (3, 64, 2, True), (1, 200, 4, False), (2, 640, 8, True)])
def test_attention_tensor_core_matches_oracle(n_seq, n, heads, with_bias):
    """wgmma attention (bf16 operands, fp32 softmax) vs the fp32 oracle core: |err| <= 0.02 on O(1) outputs."""
    from oracle import phenaki_oracle as O
    dh, I = 64, heads * 64
    q, kv = TC.seeded_randn((n_seq, n, I), 200), TC.seeded_randn((n_seq, n, 2 * I), 201)
    qs, ks = TC.seeded_randn((dh,), 202).abs() * 0.3 + 0.7, TC.seeded_randn((dh,), 203).abs() * 0.3 + 0.7
    bias = TC.seeded_randn((heads, n, n), 204) if with_bias else None
    split = lambda t: t.reshape(n_seq, n, heads, dh).permute(0, 2, 1, 3)
    k, v = kv.chunk(2, dim=-1)
    ref = O.attention_core(split(q), split(k), split(v), qs, ks, heads=heads, attn_bias=bias)
    ref = ref.permute(0, 2, 1, 3).reshape(n_seq, n, I)
    lib = L.lib()
    qd, kvd, qsd, ksd = q.to(DEV), kv.to(DEV), qs.to(DEV), ks.to(DEV)
    bd = bias.to(DEV) if with_bias else None
    out = torch.empty((n_seq, n, I), dtype=torch.bfloat16, device=DEV)
    nbytes = lib.phk_attention_tc_scratch_bytes(n_seq, n, heads)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    L.check(lib.phk_attention_tc(L.ptr(qd), L.ptr(kvd), L.ptr(qsd), L.ptr(ksd), L.ptr(bd), L.ptr(out), n_seq, n, heads,
                                 8.0, L.ptr(scratch), nbytes, L.stream_ptr()), "phk_attention_tc")
    torch.cuda.synchronize()
    err = (out.cpu().float() - ref).abs().max().item()
    assert err <= 0.02, f"max |err| {err}"


@pytest.mark.parametrize("M,N,K", [(256, 256, 64), (600, 700, 200), (4608, 512, 512), (1300, 1000, 1408), (129, 96, 72)])
def test_gemm_variants_fp32_out_bias_residual_rowmap(M, N, K):
    """Ragged M / N / K, with bias, in-place residual and the output row map."""
    Kp = (K + 7) // 8 * 8
    a, w = operands(M, N, K, lda=Kp, ldw=Kp, seed=20)
    bias, res = TC.seeded_randn((N,), 25), TC.seeded_randn((M, N), 26)
    ref = a[:, :K].float() @ w[:, :K].float().t() + bias + res
    ad, wd, bd = a.to(DEV), w.to(DEV), bias.to(DEV)
    c = res.clone().to(DEV)
    L.check(L.lib().phk_gemm_bf16(L.ptr(ad), Kp, L.ptr(wd), Kp, L.ptr(c), N, M, N, K, L.ptr(bd), L.ptr(c), 0, 0, 0, 0,
                                  L.stream_ptr()), "phk_gemm_bf16")
    torch.testing.assert_close(c.cpu(), ref, rtol=1e-4, atol=2e-3 * max(1.0, (K / 512) ** 0.5))
    # row map: output row = (m // 50) * 64 + 3 + m % 50
    rows = (M + 49) // 50 * 64 + 8
    c2 = torch.zeros((rows, N), device=DEV)
    L.check(L.lib().phk_gemm_bf16(L.ptr(ad), Kp, L.ptr(wd), Kp, L.ptr(c2), N, M, N, K, None, None, 50, 64, 3, 0,
                                  L.stream_ptr()), "phk_gemm_bf16")
    idx = torch.tensor([(m // 50) * 64 + 3 + m % 50 for m in range(M)])
    torch.testing.assert_close(c2.cpu()[idx], ref - bias - res, rtol=1e-4, atol=2e-3 * max(1.0, (K / 512) ** 0.5))


def test_gemm_variants_bf16_out_and_geglu():
    M, N, K = 700, 520, 256
    a, w = operands(M, N, K, seed=30)
    bias = TC.seeded_randn((N,), 31)
    ref = a.float() @ w.float().t() + bias
    c = torch.empty((M, N), dtype=torch.bfloat16, device=DEV)
    ad, wd, bd = a.to(DEV), w.to(DEV), bias.to(DEV)   # named: the device copies must outlive the launch
    L.check(L.lib().phk_gemm_bf16(L.ptr(ad), K, L.ptr(wd), K, L.ptr(c), N, M, N, K, L.ptr(bd), None, 0, 0, 0, 1,
                                  L.stream_ptr()), "phk_gemm_bf16")
    torch.testing.assert_close(c.cpu().float(), ref, rtol=1e-2, atol=5e-2)
    # GEGLU: W rows packed [64 value | 64 gate]; 5 groups, the last one ragged
    inner, K2 = 300, 512
    inner_pad = (inner + 63) // 64 * 64
    a2 = TC.seeded_randn((M, K2), 32).bfloat16()
    w1 = (TC.seeded_randn((2 * inner, K2), 33) / K2 ** 0.5).bfloat16()
    packed = torch.zeros((2 * inner_pad, K2), dtype=torch.bfloat16)
    for g in range(inner_pad // 64):
        lo, hi = g * 64, min(g * 64 + 64, inner)
        packed[g * 128: g * 128 + (hi - lo)] = w1[lo:hi]
        packed[g * 128 + 64: g * 128 + 64 + (hi - lo)] = w1[inner + lo: inner + hi]
    h = a2.float() @ w1.float().t()
    ref2 = torch.nn.functional.gelu(h[:, inner:]) * h[:, :inner]     # exact erf GELU (attention.py:40-43)
    out = torch.full((M, inner_pad), 7.0, dtype=torch.bfloat16, device=DEV)
    a2d, pd = a2.to(DEV), packed.to(DEV)
    L.check(L.lib().phk_gemm_bf16(L.ptr(a2d), K2, L.ptr(pd), K2, L.ptr(out), inner_pad, M, 2 * inner_pad, K2, None, None,
                                  0, 0, 0, 2, L.stream_ptr()), "phk_gemm_bf16")
    o = out.cpu().float()
    torch.testing.assert_close(o[:, :inner], ref2, rtol=1e-2, atol=1e-2)
    assert (o[:, inner:] == 0).all()


def test_geglu_epilogue_activation_error_is_below_bf16_rounding():
    """The epilogue's sigmoid-form fit of erf-GELU: |gelu_fit(g) * v - gelu_erf(g) * v| stays within one bf16 ulp of the
    result (+1e-4 * |v| absolute near zero) over the whole gate range, including |g| > 8 where the fit is clamped."""
    M, K = 256, 64
    gates = torch.linspace(-12.0, 12.0, M)
    a = torch.zeros((M, K))
    a[:, 0] = gates            # gate pre-activation = a[:,0] * 1
    a[:, 1] = 1.0              # value pre-activation = 1 * v_j
    w = torch.zeros((128, K))
    vals = torch.linspace(0.25, 2.0, 64)
    w[:64, 1] = vals           # value rows
    w[64:, 0] = 1.0            # gate rows
    ab, wb = a.bfloat16(), w.bfloat16()
    g = ab[:, 0].float()[:, None]
    v = wb[:64, 1].float()[None, :]
    ref = torch.nn.functional.gelu(g.double()).float() * v
    out = torch.empty((M, 64), dtype=torch.bfloat16, device=DEV)
    abd, wbd = ab.to(DEV), wb.to(DEV)
    L.check(L.lib().phk_gemm_bf16(L.ptr(abd), K, L.ptr(wbd), K, L.ptr(out), 64, M, 128, K, None, None, 0, 0, 0, 2,
                                  L.stream_ptr()), "phk_gemm_bf16")
    err = (out.cpu().float() - ref).abs()
    bound = ref.abs() * 2.0 ** -8 + 1e-4 * v
    assert (err <= bound).all(), f"max excess {(err - bound).max():.2e}"


@pytest.mark.parametrize("M,N1,N2,K1,K2", [(4608, 512, 1024, 512, 512), (300, 200, 130, 72, 136), (129, 64, 64, 64, 64)])
def test_gemm_x2_two_problems_in_one_launch(M, N1, N2, K1, K2):
    """phk_gemm_bf16_x2 (q and k,v projections of one attention block in a single persistent launch) equals the fp32
    product of the bf16 operands, and two separate phk_gemm_bf16 calls bit for bit (same tiles, same K order)."""
    a1, w1 = operands(M, N1, K1, seed=50)
    a2, w2 = operands(M, N2, K2, seed=52)
    d = [t.to(DEV) for t in (a1, w1, a2, w2)]
    c1 = torch.full((M, N1), 3.0, device=DEV)
    c2 = torch.full((M, N2), 3.0, device=DEV)
    lib = L.lib()
    L.check(lib.phk_gemm_bf16_x2(L.ptr(d[0]), K1, L.ptr(d[1]), K1, L.ptr(c1), N1, M, N1, K1, None, L.ptr(d[2]), K2, L.ptr(d[3]),
                                 K2, L.ptr(c2), N2, M, N2, K2, None, L.stream_ptr()), "phk_gemm_bf16_x2")
    torch.testing.assert_close(c1.cpu(), a1.float() @ w1.float().t(), rtol=1e-4, atol=2e-3)
    torch.testing.assert_close(c2.cpu(), a2.float() @ w2.float().t(), rtol=1e-4, atol=2e-3)
    s1, s2 = torch.empty_like(c1), torch.empty_like(c2)
    L.check(lib.phk_gemm_bf16(L.ptr(d[0]), K1, L.ptr(d[1]), K1, L.ptr(s1), N1, M, N1, K1, None, None, 0, 0, 0, 0, L.stream_ptr()))
    L.check(lib.phk_gemm_bf16(L.ptr(d[2]), K2, L.ptr(d[3]), K2, L.ptr(s2), N2, M, N2, K2, None, None, 0, 0, 0, 0, L.stream_ptr()))
    assert torch.equal(s1, c1) and torch.equal(s2, c2)


def test_gemm_x2_different_row_counts_and_biases():
    """The two problems of one launch may differ in M, N, K and bias: first-frame (512 x 3072) and rest-frames
    (4096 x 6144) patch embeddings of cfg2 (cvivit.py:542-549), scaled down."""
    M1, N1, K1, M2, N2, K2 = 128, 256, 384, 1000, 256, 768
    a1, w1 = operands(M1, N1, K1, seed=60)
    a2, w2 = operands(M2, N2, K2, seed=62)
    b1, b2 = TC.seeded_randn((N1,), 64), TC.seeded_randn((N2,), 65)
    d = [t.to(DEV) for t in (a1, w1, a2, w2, b1, b2)]
    c1, c2 = torch.zeros((M1, N1), device=DEV), torch.zeros((M2, N2), device=DEV)
    L.check(L.lib().phk_gemm_bf16_x2(L.ptr(d[0]), K1, L.ptr(d[1]), K1, L.ptr(c1), N1, M1, N1, K1, L.ptr(d[4]), L.ptr(d[2]), K2,
                                     L.ptr(d[3]), K2, L.ptr(c2), N2, M2, N2, K2, L.ptr(d[5]), L.stream_ptr()), "phk_gemm_bf16_x2")
    torch.testing.assert_close(c1.cpu(), a1.float() @ w1.float().t() + b1, rtol=1e-4, atol=3e-3)
    torch.testing.assert_close(c2.cpu(), a2.float() @ w2.float().t() + b2, rtol=1e-4, atol=3e-3)
