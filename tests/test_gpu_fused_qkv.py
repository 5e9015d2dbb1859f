"""GPU: the fused self-attention operand path of bf16 mode (round 2): phk_gemm_bf16_qkv (q / k,v projections whose
epilogue writes the l2-normalised, scaled bf16 operands of the attention core, attention.py:146-157), consumed by
phk_attention_tc_bf16 (4-D tensor maps over token-major rows, V as an MN-major wgmma operand) and
phk_attention_small_bf16 (temporal transformer, one warp per (sequence, head)) -- against torch fp32 references of the
same ops computed from the same bf16 inputs."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from phenaki_pytorch_b200 import _lib as L
from tests import cases as TC

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _qkv_reference(xn, xraw, wq, wkv, qs, ks, heads, sim_scale):
    q = xn.float() @ wq.float().t()
    kv = xraw.float() @ wkv.float().t()
    k, v = kv.chunk(2, dim=-1)
    M = q.shape[0]
    qn = F.normalize(q.reshape(M, heads, 64), dim=-1) * qs * sim_scale
    kn = F.normalize(k.reshape(M, heads, 64), dim=-1) * ks
    return qn.reshape(M, -1), torch.cat((kn.reshape(M, -1), v), dim=-1)


@pytest.mark.parametrize("M,heads,K", [(4608, 8, 512), (300, 2, 256), (129, 4, 64), (2304, 8, 512)])
def test_qkv_projection_with_normalising_epilogue(M, heads, K):
    I = heads * 64
    xn, xraw = TC.seeded_randn((M, K), 400).bfloat16(), (TC.seeded_randn((M, K), 401) * 1.7).bfloat16()
    wq, wkv = (TC.seeded_randn((I, K), 402) / K ** 0.5).bfloat16(), (TC.seeded_randn((2 * I, K), 403) / K ** 0.5).bfloat16()
    qs, ks = TC.seeded_randn((64,), 404).abs() * 0.3 + 0.7, TC.seeded_randn((64,), 405).abs() * 0.3 + 0.7
    ref_q, ref_kv = _qkv_reference(xn, xraw, wq, wkv, qs, ks, heads, 8.0)
    d = lambda t: t.to(DEV)
    xnd, xrd, wqd, wkvd, qsd, ksd = d(xn), d(xraw), d(wq), d(wkv), d(qs), d(ks)
    qn = torch.full((M, I), 9.0, dtype=torch.bfloat16, device=DEV)
    kvn = torch.full((M, 2 * I), 9.0, dtype=torch.bfloat16, device=DEV)
    L.check(L.lib().phk_gemm_bf16_qkv(L.ptr(xnd), L.ptr(xrd), K, L.ptr(wqd), L.ptr(wkvd), K, L.ptr(qn), L.ptr(kvn), M, I, K,
                                      L.ptr(qsd), L.ptr(ksd), 8.0, L.stream_ptr()), "phk_gemm_bf16_qkv")
    torch.cuda.synchronize()
    # one bf16 rounding of values of magnitude <= 8 (q), <= 1 (k), O(1) (v)
    torch.testing.assert_close(qn.cpu().float(), ref_q, rtol=1e-2, atol=2e-2)
    torch.testing.assert_close(kvn.cpu().float()[:, :I], ref_kv[:, :I], rtol=1e-2, atol=4e-3)
    torch.testing.assert_close(kvn.cpu().float()[:, I:], ref_kv[:, I:], rtol=1e-2, atol=2e-2)


def _core_reference(qn, kvn, n_seq, n, heads, bias=None, causal_slopes=None):
    I = heads * 64
    q = qn.float().reshape(n_seq, n, heads, 64).permute(0, 2, 1, 3)
    k = kvn.float()[:, :I].reshape(n_seq, n, heads, 64).permute(0, 2, 1, 3)
    v = kvn.float()[:, I:].reshape(n_seq, n, heads, 64).permute(0, 2, 1, 3)
    sim = q @ k.transpose(-1, -2)
    if bias is not None:
        sim = sim + bias
    if causal_slopes is not None:
        idx = torch.arange(n)
        sim = sim - (idx[None, :] - idx[:, None]).abs() * causal_slopes[:, None, None]
        sim = sim.masked_fill(torch.ones(n, n, dtype=torch.bool).triu(1), -torch.finfo(torch.float32).max)
    out = sim.softmax(dim=-1) @ v
    return out.permute(0, 2, 1, 3).reshape(n_seq * n, I)


@pytest.mark.parametrize("n_seq,n,heads,with_bias", [(72, 64, 8, True), (2, 576, 8, True), (1, 200, 4, False), (3, 130, 2, True),
                                                     (8, 576, 8, True), (2, 1024, 8, True), (5, 199, 3, True)])
def test_attention_tc_on_prenormalised_token_major_operands(n_seq, n, heads, with_bias):
    """(8, 576, 8): the MaskGit shape; n = 199: odd bias rows (scalar loads) and a ragged last chunk."""
    _attention_tc_case(n_seq, n, heads, with_bias)


@pytest.mark.parametrize("n_seq,n,heads,with_bias", [(72, 64, 8, True), (5, 49, 3, True), (3, 17, 2, False), (2, 64, 4, False),
                                                     (4, 36, 8, True)])
def test_attention_mid_mma_on_prenormalised_token_major_operands(n_seq, n, heads, with_bias):
    """phk_attention_mid_bf16 (16 < n <= 64, one CTA of four warps per (sequence, head), mma.sync): the spatial transformer's
    72 x 64 shape, odd lengths (scalar bias loads, warps without rows), no bias."""
    _attention_tc_case(n_seq, n, heads, with_bias, entry="phk_attention_mid_bf16")


def _attention_tc_case(n_seq, n, heads, with_bias, entry="phk_attention_tc_bf16"):
    I = heads * 64
    rows = n_seq * n
    qn = (F.normalize(TC.seeded_randn((rows, heads, 64), 410), dim=-1) * 8.0).reshape(rows, I).bfloat16()
    kn = F.normalize(TC.seeded_randn((rows, heads, 64), 411), dim=-1).reshape(rows, I)
    kvn = torch.cat((kn, TC.seeded_randn((rows, I), 412)), dim=-1).bfloat16()
    bias = TC.seeded_randn((heads, n, n), 413) if with_bias else None
    ref = _core_reference(qn, kvn, n_seq, n, heads, bias=bias)
    qd, kvd = qn.to(DEV), kvn.to(DEV)
    bd = bias.to(DEV) if with_bias else None
    out = torch.empty((rows, I), dtype=torch.bfloat16, device=DEV)
    L.check(getattr(L.lib(), entry)(L.ptr(qd), I, L.ptr(kvd), 2 * I, L.ptr(bd), L.ptr(out), n_seq, n, heads, L.stream_ptr()), entry)
    torch.cuda.synchronize()
    err = (out.cpu().float() - ref).abs().max().item()
    assert err <= 0.02, f"max |err| {err}"


@pytest.mark.parametrize("n_outer,n_inner,n,heads,causal", [(8, 64, 9, 8, True), (3, 4, 5, 2, True), (2, 6, 16, 4, False)])
def test_small_attention_on_prenormalised_operands(n_outer, n_inner, n, heads, causal):
    """The temporal layout: sequence (outer, inner) has its token t at row (outer * n + t) * n_inner + inner."""
    I = heads * 64
    rows = n_outer * n * n_inner
    qn = (F.normalize(TC.seeded_randn((rows, heads, 64), 420), dim=-1) * 8.0).reshape(rows, I).bfloat16()
    kn = F.normalize(TC.seeded_randn((rows, heads, 64), 421), dim=-1).reshape(rows, I)
    kvn = torch.cat((kn, TC.seeded_randn((rows, I), 422)), dim=-1).bfloat16()
    slopes = torch.tensor([2.0 ** (-8.0 * (i + 1) / heads) for i in range(heads)]) if causal else None
    # gather every sequence into (n_seq * n) contiguous rows for the reference
    idx = torch.arange(rows).reshape(n_outer, n, n_inner).permute(0, 2, 1).reshape(-1)
    ref = _core_reference(qn[idx], kvn[idx], n_outer * n_inner, n, heads, causal_slopes=slopes)
    g = L.AttnGeomT()
    g.n_outer, g.n_inner, g.n_q, g.n_k, g.heads, g.dim_head, g.causal = n_outer, n_inner, n, n, heads, 64, int(causal)
    g.q_outer, g.q_inner, g.q_tok = n * n_inner * I, I, n_inner * I
    g.k_outer, g.k_inner, g.k_tok = n * n_inner * 2 * I, 2 * I, n_inner * 2 * I
    g.o_outer, g.o_inner, g.o_tok = g.q_outer, g.q_inner, g.q_tok
    g.mask_off_from, g.out_bf16, g.scale = -1, 1, 8.0
    qd, kvd = qn.to(DEV), kvn.to(DEV)
    sd = slopes.to(DEV) if causal else None
    out = torch.empty((rows, I), dtype=torch.bfloat16, device=DEV)
    L.check(L.lib().phk_attention_small_bf16(L.ptr(qd), L.ptr(kvd), L.ptr(sd), L.ptr(out), C.byref(g), L.stream_ptr()),
            "phk_attention_small_bf16")
    torch.cuda.synchronize()
    err = (out.cpu().float()[idx] - ref).abs().max().item()
    assert err <= 0.02, f"max |err| {err}"


@pytest.mark.parametrize("b,n,ctx_len,heads,cfg", [(4, 576, 16, 8, True), (2, 130, 29, 4, False), (3, 64, 7, 2, True)])
def test_cross_attention_bf16_output_on_warp_mma(b, n, ctx_len, heads, cfg):
    """phk_attention's bf16-output cross-attention path (attention_cross_mma_kernel: null-kv + text keys <= 32 slots) against
    the fp32 oracle core: text masks, the CFG null half (sequences >= mask_off_from see only the null keys), ragged tails."""
    from oracle import phenaki_oracle as O
    I, nnull = heads * 64, 2
    seqs = 2 * b if cfg else b
    q = TC.seeded_randn((seqs, n, I), 440)
    ctx_kv = TC.seeded_randn((b, ctx_len, 2 * I), 441)
    null_kv = TC.seeded_randn((heads, 2 * nnull, 64), 442)
    qs, ks = TC.seeded_randn((64,), 443).abs() * 0.3 + 0.7, TC.seeded_randn((64,), 444).abs() * 0.3 + 0.7
    tmask = torch.ones((b, ctx_len), dtype=torch.bool)
    for i in range(b):
        tmask[i, max(1, ctx_len - 3 * i):] = False
    split = lambda t_: t_.reshape(t_.shape[0], t_.shape[1], heads, 64).permute(0, 2, 1, 3)
    kvs = ctx_kv.repeat(2, 1, 1) if cfg else ctx_kv
    k, v = kvs.chunk(2, dim=-1)
    nk = null_kv[:, 0::2].unsqueeze(0).expand(seqs, -1, -1, -1)
    nv = null_kv[:, 1::2].unsqueeze(0).expand(seqs, -1, -1, -1)
    mask = torch.cat((tmask, torch.zeros_like(tmask)), dim=0) if cfg else tmask
    ref = O.attention_core(split(q), torch.cat((nk, split(k)), dim=-2), torch.cat((nv, split(v)), dim=-2), qs, ks, heads=heads,
                           num_null_kv=nnull, mask=mask)
    ref = ref.permute(0, 2, 1, 3).reshape(seqs, n, I)
    g = L.AttnGeomT()
    g.n_outer, g.n_inner, g.n_q, g.n_k, g.heads, g.dim_head, g.num_null_kv = seqs, 1, n, ctx_len, heads, 64, nnull
    g.q_outer, g.q_tok = n * I, I
    g.k_outer, g.k_tok = ctx_len * 2 * I, 2 * I
    g.o_outer, g.o_tok = n * I, I
    g.kv_outer_mod, g.mask_outer_mod, g.mask_off_from = b, b, (b if cfg else -1)
    g.out_bf16, g.scale = 1, 8.0
    d = lambda t_: t_.contiguous().to(DEV)
    qd, kvd, nd, qsd, ksd, md = d(q), d(ctx_kv), d(null_kv), d(qs), d(ks), d(tmask.to(torch.uint8))
    out = torch.empty((seqs, n, I), dtype=torch.bfloat16, device=DEV)
    L.check(L.lib().phk_attention(L.ptr(qd), L.ptr(kvd), L.ptr(nd), L.ptr(qsd), L.ptr(ksd), None, L.ptr(md), None, L.ptr(out),
                                  C.byref(g), L.stream_ptr()), "phk_attention")
    torch.cuda.synchronize()
    err = (out.cpu().float() - ref).abs().max().item()
    assert err <= 0.03, f"max |err| {err}"


@pytest.mark.parametrize("b,n,ctx_len,heads,cfg", [(4, 576, 16, 8, True), (2, 130, 29, 4, False), (3, 64, 7, 2, True)])
def test_cross_attention_on_packed_operands(b, n, ctx_len, heads, cfg):
    """phk_cross_kv_pack (keys l2-normalised * k_scale, values, dead flags; two layers packed in one launch) +
    phk_attention_cross_packed on pre-normalised bf16 queries, against the fp32 oracle core: text masks, the CFG null half,
    ragged query tails."""
    from oracle import phenaki_oracle as O
    I, nnull, depth = heads * 64, 2, 2
    seqs = 2 * b if cfg else b
    q = TC.seeded_randn((seqs, n, I), 450)
    qs, ks = TC.seeded_randn((64,), 453).abs() * 0.3 + 0.7, TC.seeded_randn((64,), 454).abs() * 0.3 + 0.7
    tmask = torch.ones((b, ctx_len), dtype=torch.bool)
    for i in range(b):
        tmask[i, max(1, ctx_len - 3 * i):] = False
    split = lambda t_: t_.reshape(t_.shape[0], t_.shape[1], heads, 64).permute(0, 2, 1, 3)
    layers = [(TC.seeded_randn((b, ctx_len, 2 * I), 460 + l), TC.seeded_randn((heads, 2 * nnull, 64), 470 + l)) for l in range(depth)]
    d = lambda t_: t_.contiguous().to(DEV)
    kv_d = [d(kv) for kv, _ in layers]
    nk_d = [d(nkv) for _, nkv in layers]
    ks_d = d(ks)
    PtrArr = C.c_void_p * depth
    pack = torch.empty((depth, b, heads, 2 * 32 * 64), dtype=torch.bfloat16, device=DEV)
    dead = torch.empty((depth, b, 32), dtype=torch.float32, device=DEV)
    md = d(tmask.to(torch.uint8))
    L.check(L.lib().phk_cross_kv_pack(PtrArr(*[t.data_ptr() for t in kv_d]), PtrArr(*[t.data_ptr() for t in nk_d]),
                                      PtrArr(*[ks_d.data_ptr()] * depth), depth, L.ptr(md), b, ctx_len, heads, nnull,
                                      L.ptr(pack), L.ptr(dead), L.stream_ptr()), "phk_cross_kv_pack")
    # what phk_gemm_bf16_qnorm's epilogue writes: per-head l2-normalised queries * q_scale * 8, bf16
    qn = (F.normalize(q.reshape(seqs, n, heads, 64), dim=-1) * qs * 8.0).reshape(seqs * n, I).bfloat16()
    qd = d(qn)
    mask = torch.cat((tmask, torch.zeros_like(tmask)), dim=0) if cfg else tmask
    for l, (ctx_kv, null_kv) in enumerate(layers):
        kvs = ctx_kv.repeat(2, 1, 1) if cfg else ctx_kv
        k, v = kvs.chunk(2, dim=-1)
        nk = null_kv[:, 0::2].unsqueeze(0).expand(seqs, -1, -1, -1)
        nv = null_kv[:, 1::2].unsqueeze(0).expand(seqs, -1, -1, -1)
        ref = O.attention_core(split(q), torch.cat((nk, split(k)), dim=-2), torch.cat((nv, split(v)), dim=-2), qs, ks, heads=heads,
                               num_null_kv=nnull, mask=mask)
        ref = ref.permute(0, 2, 1, 3).reshape(seqs * n, I)
        out = torch.full((seqs * n, I), 7.0, dtype=torch.bfloat16, device=DEV)
        L.check(L.lib().phk_attention_cross_packed(L.ptr(qd), I, L.ptr(pack[l]), L.ptr(dead[l]), L.ptr(out), I, seqs, n, heads, b,
                                                   nnull, b if cfg else -1, L.stream_ptr()), "phk_attention_cross_packed")
        torch.cuda.synchronize()
        err = (out.cpu().float() - ref).abs().max().item()
        assert err <= 0.04, f"layer {l}: max |err| {err}"
