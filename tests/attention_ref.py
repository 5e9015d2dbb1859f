"""float64 reference of the attention forward core (oracle.phenaki_oracle.attention_core) and a per-element error bound
derived from the arithmetic of each kernel of csrc/attention.cu and csrc/attention_tc.cu.

Notation, for one (sequence, head, query row i): q^_i and k^_j are the normalised, scaled operands (F.normalize(q) *
q_scale * scale and F.normalize(k) * k_scale, or the bf16 Qn / KVn the bf16 entry points take), s_ij = q^_i . k^_j + b_ij
(b: position bias, ALiBi, 0 on null keys), L_i the live keys (key mask, causal mask, CFG null half), m_i = max_{j in L_i}
s_ij, a_ij = softmax over L_i, o_id = sum_j a_ij v_jd.  u = 2^-24 (fp32), and a bf16 rounding of x moves it by at most
half an ulp <= 2^-8 |x|.

1. Score perturbations.  If every live exponent p_ij = exp(s_ij - m_i) the kernel forms carries a relative error
   e^{+-d_ij}, then a'_ij / a_ij lies in [e^{-2 D_i}, e^{2 D_i}] with D_i = max_{j in L_i} d_ij, and since
   sum_j (a'_ij - a_ij) = 0,
       |o'_id - o_id| = |sum_j (a'_ij - a_ij)(v_jd - o_id)| <= (e^{2 D_i} - 1) (T_id + |o_id|),   T_id = sum_j a_ij |v_jd|.
   d_ij collects, with S_ij = sum_d |q^_id k^_jd|:
     * bf16 rounding of q^ and k^ (attention_prep_kernel ahead of the wgmma kernel, the cross MMA kernel, the packed
       cross keys): (1 + 2^-9)^2 - 1 <= 2^-8, times S_ij;
     * fp32 l2-normalisation of fp32 projections (sum of dim_head squares, sqrt or rsqrt, divide, two scale
       multiplies): (dim_head / 2 + 8) u relative on each of q^, k^, so 2 (dim_head / 2 + 8) u S_ij;
     * the fp32 dot product of dim_head terms (FFMA chains or tensor-core accumulation; exact bf16 x bf16 products):
       (dim_head + 2) 2u S_ij;
     * the scale multiply, the bias / ALiBi add and the fmaf(s, log2 e, -m log2 e) argument of ex2: 2u (|s_ij| + |b_ij|)
       and 2^-22 (|s_ij| + |m_i|);
     * ex2.approx / __expf / expf themselves, once per key chunk (the online-softmax rescale exp(m_old - m_new) is one
       more exponential per chunk): chunks x 2^-21.
2. P rounded to bf16 before P.V while the row sum l uses the unrounded p (every MMA kernel): 2^-8 T_id.
3. V rounded to bf16 from fp32 (attention_prep_kernel, the cross MMA kernel, the packed cross values): 2^-8 T_id.
4. fp32 accumulation of P.V and of l over |L_i| keys, and 1 / l times the accumulator: (|L_i| + 8) 2u T_id.
5. Exponentials that flush to zero in fp32 (weights below 2^-126): 2^-126 |L_i| max |v|.
6. The output rounding: 2^-8 (|o_id| + E_id) in bf16, u (|o_id| + E_id) in fp32, E_id the sum of 1-5.

Exact probes (census, dominant key) reuse the same reference; tests/attention_cases.py builds their inputs.
"""
import math

import torch
import torch.nn.functional as F

from oracle import phenaki_oracle as O

U = 2.0 ** -24
BF16 = 2.0 ** -8
F64 = torch.float64


class Model:
    """Error model of one kernel (see the module docstring): which operands it rounds to bf16, whether it normalises fp32
    projections itself, and its key-chunk width (online-softmax passes)."""

    def __init__(self, *, fp32_norm, qk_bf16=False, v_bf16=False, p_bf16=False, out_bf16=False, chunk=None):
        self.fp32_norm, self.qk_bf16, self.v_bf16, self.p_bf16, self.out_bf16 = fp32_norm, qk_bf16, v_bf16, p_bf16, out_bf16
        self.chunk = chunk

    def chunks(self, n_keys):
        return 1 if self.chunk is None else max(1, -(-n_keys // self.chunk))


def normalised(x, scale_vec, scale=1.0):
    """F.normalize(x, dim=-1) * scale_vec * scale in float64 (attention.py:153-157)."""
    return F.normalize(x.to(F64), dim=-1) * scale_vec.to(F64) * scale


def oracle_core(q, k, v, q_scale, k_scale, live, bias, scale):
    """oracle.attention_core in float64 on split heads: q (S,h,i,d), k / v (S,h,j,d) with the null keys first.  `live`
    (S,1|h,1|i,j) bool marks the live keys; `bias` (1|S,h,i,j) float64 or None carries the position bias and the ALiBi
    term.  A key that is dead for some rows only (causal) is folded into the bias as -finfo.max, which is what the
    oracle's causal masked_fill adds."""
    neg = -torch.finfo(F64).max
    S, h, i, _ = q.shape
    j = k.shape[-2]
    live = live.expand(S, h, i, j)
    extra = torch.zeros((S, h, i, j), dtype=F64) if bias is None else bias.to(F64).expand(S, h, i, j).clone()
    extra = extra.masked_fill(~live, neg)
    return O.attention_core(q.to(F64), k.to(F64), v.to(F64), q_scale.to(F64), k_scale.to(F64), heads=h,
                            attn_bias=extra, scale=scale)


def prenormalised_core(qh, kh, v, live, bias):
    """The same core on already normalised and scaled operands (the bf16 entry points' Qn / KVn): returns o and the
    attention weights a, the scores s (bias included, -inf on dead keys) and the row maxima m the bound needs."""
    s = torch.einsum("shid,shjd->shij", qh.to(F64), kh.to(F64))
    b = torch.zeros_like(s) if bias is None else bias.to(F64).expand_as(s)
    s = s + b
    sm = s.masked_fill(~live.expand_as(s), -math.inf)
    m = sm.amax(dim=-1, keepdim=True)
    p = torch.exp(sm - m)
    a = p / p.sum(dim=-1, keepdim=True)
    return torch.einsum("shij,shjd->shid", a, v.to(F64)), a, s, m, b


def bound(model, qh, kh, v, live, bias, o=None):
    """Per-element bound |out - o| (S,h,i,d) for the kernel `model`, from the reference operands (module docstring).
    Returns (o, bound); o is the prenormalised core's output unless given."""
    o_pre, a, s, m, b = prenormalised_core(qh, kh, v, live, bias)
    o = o_pre if o is None else o
    dh = qh.shape[-1]
    liv = live.expand_as(s)
    Sij = torch.einsum("shid,shjd->shij", qh.abs().to(F64), kh.abs().to(F64))
    per_s = (BF16 if model.qk_bf16 else 0.0) + (2 * (dh / 2 + 8) * U if model.fp32_norm else 0.0) + (dh + 2) * 2 * U
    n_keys = s.shape[-1]
    d = per_s * Sij + 2 * U * (s.abs() + b.abs()) + 2.0 ** -22 * (s.abs() + m.abs()) + model.chunks(n_keys) * 2.0 ** -21
    D = torch.where(liv, d, torch.zeros_like(d)).amax(dim=-1, keepdim=True)
    va = v.abs().to(F64)
    T = torch.einsum("shij,shjd->shid", a, va)
    n_live = liv.sum(dim=-1, keepdim=True).to(F64)
    E = torch.expm1(2 * D) * (T + o.abs())
    E = E + ((BF16 if model.p_bf16 else 0.0) + (BF16 if model.v_bf16 else 0.0) + (n_live + 8) * 2 * U) * T
    E = E + 2.0 ** -126 * n_live * va.amax(dim=(-2, -1), keepdim=True)
    return o, E + (BF16 if model.out_bf16 else U) * (o.abs() + E)


def census_expected(v, live):
    """q = 0: every live score is 0, every live key has p = 1 exactly: out = sum_{j live} v_j / |L|.  live (S,h,i,j)."""
    w = live.to(F64)
    return torch.einsum("shij,shjd->shid", w, v.to(F64)) / w.sum(-1, keepdim=True)


def census_tolerance(expected, v, live, out_bf16):
    """One ulp of the expected value in the output type, plus the fp32 rounding of the partial sums of the terms
    p_j v_j / l or p_j (v_j / l) ((|L| + 2) 2u of the mean |v|, for the kernels that scale P before P.V): far below the
    1 / |L| that one wrong key moves the average by."""
    e = expected.abs()
    ex = torch.floor(torch.log2(torch.where(e > 0, e, torch.ones_like(e))))
    ulp = torch.where(e > 0, torch.pow(2.0, ex - (7 if out_bf16 else 23)), torch.zeros_like(e))
    w = live.to(F64)
    n = w.sum(-1, keepdim=True)
    mean_abs = torch.einsum("shij,shjd->shid", w, v.abs().to(F64)) / n
    return ulp + (n + 2) * 2 * U * mean_abs
