"""Check bodies of the attention-forward tests, shared by the H100 file (tests/test_gpu_attention_forward.py) and the CPU
executor file (tests/test_attention_forward_emulated_cpu.py): every body takes (lib, device, sync).

A case is a dict naming the entry point, the kernel it must reach (`kernel`, the demangled name of the kernel template
instance) and the shape.  Each case runs in up to three input modes:
  * "random"   : random operands, every element within the bound of tests/attention_ref.py;
  * "census"   : q = 0, so every live key has weight exactly 1; v in {-1, 0, +1} with column sums in -2..2 over the live
                 keys, keys behind the key mask hold 64.  out = bf16(sum_live v / |live|) within one ulp: a key that is
                 missing, doubled or read from another sequence / head / row moves a column sum by an integer;
  * "dominant" : q = 0 and bias[h, i, pi_h(i)] = +40 (pi_h a permutation reaching every key position, the last key of a
                 ragged chunk included) or, for causal kernels, ALiBi slopes 30 (the diagonal): out_i is one value row
                 to rounding, which pins the bias row / column / head indexing and the V row addressing.
Every input buffer holds NaN wherever the geometry does not address an operand (padding columns, gaps between
sequences), and every output buffer starts as a sentinel that must survive everywhere the kernel has nothing to write."""
import ctypes as C
import math

import torch

from oracle import phenaki_oracle as O
from phenaki_pytorch_b200 import _lib as L
from tests import attention_ref as R

F64 = torch.float64
SENTINEL = -320.0  # exact in fp32 and bf16
DOMINANT_BIAS, DOMINANT_SLOPE = 40.0, 30.0
CENSUS_DEAD = 64.0  # value of a key behind the key mask: any leak of it is far outside one ulp
REF_ELEMS = 2 ** 24  # fp64 score elements per reference chunk (several temporaries of this size)
WORST = {}  # kernel -> worst err / bound seen in this process (reported by the test files)

# ---- error models of the kernels (tests/attention_ref.py) ---------------------------------------------------------------
_PRENORM_MMA = dict(fp32_norm=False, p_bf16=True, out_bf16=True)
_FP32_MMA = dict(fp32_norm=True, qk_bf16=True, v_bf16=True, p_bf16=True, out_bf16=True)


def model(kernel, out_bf16):
    if kernel.startswith("attention_kernel<"):
        return R.Model(fp32_norm=True, out_bf16=out_bf16, chunk=64)
    if kernel.startswith(("attention_small_kernel<", "attention_rows_kernel<", "attention_fewkeys_kernel<")) or \
            (kernel.startswith("attention_warp64_kernel<") and kernel.endswith("false>")):
        return R.Model(fp32_norm=True, out_bf16=out_bf16)
    if kernel.startswith("attention_warp64_kernel<"):  # PRE: the bf16 operands of phk_gemm_bf16_qkv
        return R.Model(fp32_norm=False, out_bf16=out_bf16)
    if kernel in ("attention_small_mma_kernel", "attention_mid_mma_kernel"):
        return R.Model(**_PRENORM_MMA)
    if kernel == "attention_tc_kernel":
        return R.Model(**_PRENORM_MMA, chunk=64)
    if kernel == "attention_prep_kernel":  # phk_attention_tc: fp32 projections -> bf16 operands -> attention_tc_kernel
        return R.Model(**_FP32_MMA, chunk=64)
    if kernel in ("attention_cross_mma_kernel", "attention_cross_packed_kernel"):
        return R.Model(**_FP32_MMA)
    raise KeyError(kernel)


def _defaults(case):
    bf16_out = case["entry"] in ("small_bf16", "mid_bf16", "tc_bf16", "tc", "cross_packed")  # default (only one for 3 of them)
    c = dict(n_inner=1, dh=64, nnull=0, causal=False, bias=False, mask=False, ctx_b=0, cfg=False, out_bf16=int(bf16_out),
             pad_q=0, pad_k=0, pad_o=0, temporal=False, layers=1)
    c.update(case)
    c.setdefault("n_k", c["n_q"])
    if c["entry"] in ("mid_bf16", "tc_bf16", "tc", "cross_packed"):
        c["out_bf16"] = 1
    return c


def _rng(seed):
    return torch.Generator().manual_seed(seed)


def _bf16(x):
    return x.to(torch.bfloat16).to(torch.float32)


# ---- census values ----------------------------------------------------------------------------------------------------

def balanced(live, g):
    """live (..., n) bool -> values (..., n) in {-1, 0, +1} on the live keys with sum in -2..2 (not all 0) and
    CENSUS_DEAD on the others: P (+1, -1) pairs and |t| values sign(t) at random live positions."""
    n_live = live.sum(-1, keepdim=True)
    key = torch.rand(live.shape, generator=g) + (~live).float() * 2.0  # dead keys rank last
    rank = key.argsort(-1).argsort(-1)
    t = torch.randint(-2, 3, n_live.shape, generator=g)
    t = torch.where(t == 0, torch.ones_like(t), t) if n_live.numel() == 1 else t
    t = torch.clamp(t, -n_live, n_live)
    P = (torch.rand(n_live.shape, generator=g) * ((n_live - t.abs()) // 2 + 1).float()).floor().long()
    pair = torch.where(rank % 2 == 0, 1.0, -1.0)
    v = torch.where(rank < 2 * P, pair, torch.where(rank < 2 * P + t.abs(), torch.sign(t).float(), 0.0))
    return torch.where(live, v, torch.full_like(v, CENSUS_DEAD))


def _coprime_step(n):
    a = max(1, n // 2 - 1) | 1
    while math.gcd(a, n) != 1:
        a += 2
    return a


def dominant_bias(heads, n_q, n_k):
    """bias[h, i, pi_h(i)] = +40, 0 elsewhere; pi_h(i) = (a i + 7 h + 1) mod n_k, a coprime to n_k."""
    b = torch.zeros((heads, n_q, n_k))
    a = _coprime_step(n_k)
    i = torch.arange(n_q)
    for h in range(heads):
        b[h, i, (a * i + 7 * h + 1) % n_k] = DOMINANT_BIAS
    return b


# ---- logical problem ----------------------------------------------------------------------------------------------------

class Problem:
    """Logical operands of one call: q (S, h, n_q, dh); text keys / values (S_kv, h, n_k, dh); null keys / values
    (h, nnull, dh); key mask (rows, n_k) or None; bias (h, n_q, n_k) or None; ALiBi slopes (h,) or None; per sequence the
    text row it reads (kv_of), its mask row (mask_of) and whether it is the CFG null half."""


def make_problem(case, mode, seed):
    c = _defaults(case)
    g = _rng(seed)
    e = c["entry"]
    h, dh, nq, nk, nnull = c["heads"], c["dh"], c["n_q"], c["n_k"], c["nnull"]
    P = Problem()
    if e == "cross_packed":
        S = 2 * c["ctx_b"] if c["cfg"] else c.get("n_seq", c["ctx_b"])
        S_kv = c["ctx_b"]
    else:
        S = c["n_outer"] * c["n_inner"]
        S_kv = c["ctx_b"] if c["ctx_b"] else S
    P.S, P.S_kv = S, S_kv
    seqs = torch.arange(S)
    so = seqs // c["n_inner"]
    P.kv_of = so % c["ctx_b"] if c["ctx_b"] else seqs
    P.mask_of = so % c["ctx_b"] if c["ctx_b"] else so
    off_from = c["ctx_b"] if c["cfg"] else -1
    if e == "cross_packed":
        P.null_half = (so >= off_from) if off_from >= 0 else torch.zeros(S, dtype=torch.bool)
    else:  # phk_attention drops the text keys of the null half through the key mask only
        P.null_half = (so >= off_from) if (off_from >= 0 and c["mask"]) else torch.zeros(S, dtype=torch.bool)
    prenorm_q = e in ("small_bf16", "mid_bf16", "tc_bf16", "cross_packed")
    prenorm_k = e in ("small_bf16", "mid_bf16", "tc_bf16")
    P.q_scale = torch.rand(dh, generator=g) * 0.6 + 0.7
    P.k_scale = [torch.rand(dh, generator=g) * 0.6 + 0.7 for _ in range(c["layers"])]
    P.scale = 8.0
    P.key_mask = None
    if c["mask"] and nk > 0:
        rows = c["ctx_b"] if c["ctx_b"] else c["n_outer"]
        P.key_mask = torch.rand((rows, nk), generator=g) < 0.7
        P.key_mask[:, 0] = True
        P.key_mask[0, :] = True  # one row with every key live (the full ragged tail)
        if rows > 1 and nk > 1:
            P.key_mask[1, nk - 1] = False  # and one whose last key is masked
    P.bias = torch.randn((h, nq, nk), generator=g) if c["bias"] else None
    P.slopes = torch.tensor(O.alibi_slopes(h), dtype=torch.float32) if c["causal"] else None

    def q_values():
        x = torch.randn((S, h, nq, dh), generator=g)
        return _bf16(R.normalised(x, P.q_scale, P.scale).float()) if prenorm_q else x

    P.q = q_values()
    P.layers = []
    for layer in range(c["layers"]):
        kt = torch.randn((S_kv, h, nk, dh), generator=g)
        nkey = torch.randn((h, nnull, dh), generator=g)
        if prenorm_k:
            kt = _bf16(R.normalised(kt, P.k_scale[layer]).float())
        vt = torch.randn((S_kv, h, nk, dh), generator=g)
        nval = torch.randn((h, nnull, dh), generator=g)
        if prenorm_k:
            vt = _bf16(vt)
        P.layers.append([kt, vt, nkey, nval])
    if mode in ("census", "dominant"):
        P.q = torch.zeros_like(P.q)
    if mode == "census":
        if P.bias is not None:
            P.bias = torch.zeros_like(P.bias)
        if P.slopes is not None:
            P.slopes = torch.zeros_like(P.slopes)
        for lay in P.layers:
            live_txt = torch.ones((S_kv, 1, 1, nk), dtype=torch.bool)
            if P.key_mask is not None:  # mask row r pairs with text row r in every census case
                live_txt = P.key_mask[:S_kv].reshape(S_kv, 1, 1, nk).clone()
            vt = balanced(live_txt.expand(S_kv, h, dh, nk).clone(), g).permute(0, 1, 3, 2)
            lay[1] = vt.contiguous()
            lay[3] = balanced(torch.ones((h, dh, nnull), dtype=torch.bool), g).permute(0, 2, 1).contiguous()
    if mode == "dominant":
        if P.bias is not None:
            P.bias = dominant_bias(h, nq, nk)
        if P.slopes is not None:
            P.slopes = torch.full((h,), DOMINANT_SLOPE)
        for lay in P.layers:
            lay[1], lay[3] = _bf16(lay[1]), _bf16(lay[3])
    P.prenorm_q, P.prenorm_k = prenorm_q, prenorm_k
    return c, P


def reference_operands(c, P, layer, seqs):
    """q^, k^ (normalised and scaled, float64), v, live (S, 1, n_q, J) and bias (1, h, n_q, J) of the sequences `seqs`,
    null keys first; plus the raw q / k for the oracle when the kernel normalises fp32 projections itself."""
    kt, vt, nkey, nval = P.layers[layer]
    h, nq, nk, nnull = c["heads"], c["n_q"], c["n_k"], c["nnull"]
    S = len(seqs)
    kv = P.kv_of[seqs]
    k = torch.cat((nkey.unsqueeze(0).expand(S, -1, -1, -1), kt[kv]), dim=2).to(F64)
    v = torch.cat((nval.unsqueeze(0).expand(S, -1, -1, -1), vt[kv]), dim=2).to(F64)
    q = P.q[seqs].to(F64)
    J = nnull + nk
    live = torch.ones((S, 1, nq, J), dtype=torch.bool)
    if P.key_mask is not None:
        live[:, :, :, nnull:] &= P.key_mask[P.mask_of[seqs]].reshape(S, 1, 1, nk)
    live[:, :, :, nnull:] &= ~P.null_half[seqs].reshape(S, 1, 1, 1)
    bias = None
    if P.bias is not None:
        bias = torch.cat((torch.zeros((h, nq, nnull)), P.bias), dim=-1).to(F64).unsqueeze(0)
    if c["causal"]:
        pos = torch.arange(nq) + (nk - nq)
        j = torch.arange(J)
        dist = (j[None, :] - pos[:, None]).abs().to(F64)
        alibi = -dist.unsqueeze(0) * P.slopes.to(F64).reshape(h, 1, 1)
        bias = alibi.unsqueeze(0) if bias is None else bias + alibi
        live &= (j[None, :] <= pos[:, None]).reshape(1, 1, nq, J)
    qh = q if P.prenorm_q else R.normalised(q, P.q_scale, P.scale)
    kh = k if P.prenorm_k else R.normalised(k, P.k_scale[layer])
    return q, k, v, qh, kh, live, bias


# ---- device buffers -----------------------------------------------------------------------------------------------------

def _idx(n_out, n_in, n, h, dh, outer, inner, tok):
    so = torch.arange(n_out).view(-1, 1, 1, 1, 1)
    si = torch.arange(n_in).view(1, -1, 1, 1, 1)
    t = torch.arange(n).view(1, 1, -1, 1, 1)
    hh = torch.arange(h).view(1, 1, 1, -1, 1)
    d = torch.arange(dh).view(1, 1, 1, 1, -1)
    return (so * outer + si * inner + t * tok + hh * dh + d).reshape(n_out * n_in, n, h, dh).permute(0, 2, 1, 3)


def _strides(c, n, row):
    """(outer, inner, token) element strides of a sequence-of-tokens operand: sequence-major rows, or the temporal view
    '(b h w) t' of '(b t) (h w)' rows (token stride n_inner rows)."""
    if c["temporal"]:
        return n * c["n_inner"] * row, row, c["n_inner"] * row
    return c["n_inner"] * n * row, n * row, row


def _scatter(idx, values, extra, dtype, dev):
    """A NaN buffer holding `values` at `idx` (flat element offsets), `extra` trailing elements, never empty."""
    size = max(int(idx.max()) + 1 if idx.numel() else 0, 0) + extra
    buf = torch.full((max(size, 1),), float("nan"), dtype=torch.float32)
    if idx.numel():
        buf[idx.reshape(-1)] = values.reshape(-1).float()
    return buf.to(dtype).to(dev)


class Layout:
    pass


def layout(c, P):
    h, dh, nq, nk = c["heads"], c["dh"], c["n_q"], c["n_k"]
    I = h * dh
    lay = Layout()
    lay.rq, lay.rk, lay.ro = I + c["pad_q"], 2 * I + c["pad_k"], I + c["pad_o"]
    lay.q = _strides(c, nq, lay.rq)
    lay.o = _strides(c, nq, lay.ro)
    if c["ctx_b"]:
        lay.k = (nk * lay.rk, 0, lay.rk)
        lay.kidx = _idx(c["ctx_b"], 1, nk, h, dh, *lay.k)
    else:
        lay.k = _strides(c, nk, lay.rk)
        lay.kidx = _idx(c["n_outer"], c["n_inner"], nk, h, dh, *lay.k)
    lay.qidx = _idx(c["n_outer"], c["n_inner"], nq, h, dh, *lay.q)
    lay.oidx = _idx(c["n_outer"], c["n_inner"], nq, h, dh, *lay.o)
    return lay


def _geom(c, lay):
    g = L.AttnGeomT()
    g.n_outer, g.n_inner, g.n_q, g.n_k = c["n_outer"], c["n_inner"], c["n_q"], c["n_k"]
    g.heads, g.dim_head, g.num_null_kv, g.causal = c["heads"], c["dh"], c["nnull"], int(c["causal"])
    g.q_outer, g.q_inner, g.q_tok = lay.q
    g.k_outer, g.k_inner, g.k_tok = lay.k
    g.o_outer, g.o_inner, g.o_tok = lay.o
    g.kv_outer_mod = c["ctx_b"]
    g.mask_outer_mod = c["ctx_b"] if (c["mask"] and c["ctx_b"]) else 0
    g.mask_off_from = c["ctx_b"] if c["cfg"] else -1
    g.out_bf16, g.scale = int(c["out_bf16"]), 8.0
    return g


def _null_kv(nkey, nval):
    """(h, 2 nnull, dh), interleaved k0 v0 k1 v1 ... ('h (n r) d', attention.py:148)"""
    h, nnull, dh = nkey.shape
    return torch.stack((nkey, nval), dim=2).reshape(h, 2 * nnull, dh).contiguous()


def run(lib, dev, c, P, sync):
    """Runs the case's entry point; returns per layer the output gathered to (S, h, n_q, dh) float64, and asserts that
    every output element outside the written set still holds the sentinel."""
    e = c["entry"]
    d = lambda t: t.contiguous().to(dev)
    ptr = L.ptr
    odt = torch.bfloat16 if c["out_bf16"] else torch.float32
    h, dh, nq, nk, nnull = c["heads"], c["dh"], c["n_q"], c["n_k"], c["nnull"]
    I = h * dh
    outs = []
    if e in ("attention", "small_bf16", "mid_bf16", "tc_bf16"):
        lay = layout(c, P)
        kt, vt, nkey, nval = P.layers[0]
        dt = torch.float32 if e == "attention" else torch.bfloat16
        qb = _scatter(lay.qidx, P.q, c["pad_q"], dt, dev)
        kvb = _scatter(torch.cat((lay.kidx, lay.kidx + I)), torch.cat((kt, vt)), c["pad_k"], dt, dev)
        ob = torch.full((int(lay.oidx.max()) + 1 + c["pad_o"],), SENTINEL, dtype=odt, device=dev)
        bias = d(P.bias) if P.bias is not None else None
        if e == "attention":
            g = _geom(c, lay)
            nkv = d(_null_kv(nkey, nval)) if nnull else None
            mask = d(P.key_mask.to(torch.uint8)) if P.key_mask is not None else None
            slopes = d(P.slopes) if P.slopes is not None else None
            qs, ks = d(P.q_scale), d(P.k_scale[0])
            L.check(lib.phk_attention(ptr(qb), ptr(kvb), ptr(nkv), ptr(qs), ptr(ks), ptr(bias), ptr(mask), ptr(slopes),
                                      ptr(ob), C.byref(g), L.stream_ptr()), "phk_attention")
        elif e == "small_bf16":
            g = _geom(c, lay)
            slopes = d(P.slopes) if P.slopes is not None else None
            L.check(lib.phk_attention_small_bf16(ptr(qb), ptr(kvb), ptr(slopes), ptr(ob), C.byref(g), L.stream_ptr()),
                    "phk_attention_small_bf16")
        else:
            fn = getattr(lib, "phk_attention_" + e)
            L.check(fn(ptr(qb), lay.rq, ptr(kvb), lay.rk, ptr(bias), ptr(ob), c["n_outer"], nq, h, L.stream_ptr()),
                    "phk_attention_" + e)
        sync()
        outs.append(_gather(ob, lay.oidx))
    elif e == "tc":
        kt, vt, _, _ = P.layers[0]
        S = c["n_outer"]
        q = d(P.q.permute(0, 2, 1, 3).reshape(S * nq, I))
        kv = d(torch.cat((kt.permute(0, 2, 1, 3).reshape(S * nk, I), vt.permute(0, 2, 1, 3).reshape(S * nk, I)), dim=1))
        ob = torch.full((S * nq * I + c["pad_o"],), SENTINEL, dtype=odt, device=dev)
        nb = int(lib.phk_attention_tc_scratch_bytes(S, nq, h))
        scratch = torch.empty(nb, dtype=torch.uint8, device=dev)
        qs, ks = d(P.q_scale), d(P.k_scale[0])  # held until the call has run (a freed block is reused at once)
        bias = d(P.bias) if P.bias is not None else None
        L.check(lib.phk_attention_tc(ptr(q), ptr(kv), ptr(qs), ptr(ks), ptr(bias), ptr(ob), S, nq, h, 8.0, ptr(scratch), nb,
                                     L.stream_ptr()), "phk_attention_tc")
        sync()
        outs.append(_gather(ob, _idx(S, 1, nq, h, dh, nq * I, 0, I)))
    elif e == "cross_packed":
        S, b, depth = P.S, c["ctx_b"], c["layers"]
        ld_q, ld_o = I + c["pad_q"], I + c["pad_o"]
        qidx = _idx(S, 1, nq, h, dh, nq * ld_q, 0, ld_q)
        oidx = _idx(S, 1, nq, h, dh, nq * ld_o, 0, ld_o)
        qb = _scatter(qidx, P.q, c["pad_q"], torch.bfloat16, dev)
        kv_d, nkv_d, ks_d = [], [], []
        for layer, (kt, vt, nkey, nval) in enumerate(P.layers):
            rows = torch.cat((kt, vt), dim=1).permute(0, 2, 1, 3).reshape(b * nk, 2 * I) if nk else torch.full((1, 2 * I), float("nan"))
            kv_d.append(d(rows))
            nkv_d.append(d(_null_kv(nkey, nval)))
            ks_d.append(d(P.k_scale[layer]))
        Arr = C.c_void_p * depth
        pack = torch.empty((depth, b, h, 2 * 32 * 64), dtype=torch.bfloat16, device=dev)
        dead = torch.empty((depth, b, 32), dtype=torch.float32, device=dev)
        mask = d(P.key_mask.to(torch.uint8)) if P.key_mask is not None else None
        L.check(lib.phk_cross_kv_pack(Arr(*[t.data_ptr() for t in kv_d]), Arr(*[t.data_ptr() for t in nkv_d]),
                                      Arr(*[t.data_ptr() for t in ks_d]), depth, ptr(mask), b, nk, h, nnull, ptr(pack),
                                      ptr(dead), L.stream_ptr()), "phk_cross_kv_pack")
        for layer in range(depth):
            ob = torch.full((int(oidx.max()) + 1 + c["pad_o"],), SENTINEL, dtype=odt, device=dev)
            L.check(lib.phk_attention_cross_packed(ptr(qb), ld_q, ptr(pack[layer]), ptr(dead[layer]), ptr(ob), ld_o, S, nq, h,
                                                   b, nnull, b if c["cfg"] else -1, L.stream_ptr()), "phk_attention_cross_packed")
            sync()
            outs.append(_gather(ob, oidx))
    else:
        raise KeyError(e)
    return outs


def _gather(ob, oidx):
    o = ob.cpu().float()
    untouched = torch.ones(o.numel(), dtype=torch.bool)
    untouched[oidx.reshape(-1)] = False
    bad = int((o[untouched] != SENTINEL).sum())
    assert bad == 0, f"{bad} output elements outside the written rows / columns were overwritten"
    return o[oidx].to(F64)


# ---- judging ------------------------------------------------------------------------------------------------------------

def judge(c, P, outs, mode, kernel):
    """Every element within the bound (all modes), census values within one ulp; returns the worst err / bound."""
    mdl = model(kernel, bool(c["out_bf16"]))
    h, nq, J = c["heads"], c["n_q"], c["nnull"] + c["n_k"]
    step = max(1, REF_ELEMS // max(1, h * nq * J))
    worst = 0.0
    for layer, out in enumerate(outs):
        for s0 in range(0, P.S, step):
            seqs = torch.arange(s0, min(P.S, s0 + step))
            q, k, v, qh, kh, live, bias = reference_operands(c, P, layer, seqs)
            ref = None
            if not P.prenorm_q:  # the oracle core itself (float64) where the kernel sees the fp32 projections
                ref = R.oracle_core(q, k, v, P.q_scale, P.k_scale[layer], live, bias, P.scale)
            ref, bnd = R.bound(mdl, qh, kh, v, live, bias, o=ref)
            got = out[seqs]
            assert torch.isfinite(got).all(), f"{kernel} {mode}: non-finite outputs (a NaN padding element was read)"
            err = (got - ref).abs()
            ratio = err / bnd
            r_max = float(ratio.max()) if ratio.numel() else 0.0
            if r_max > 1.0:
                at = tuple(int(x) for x in torch.nonzero(ratio == ratio.max())[0])
                at = (int(seqs[at[0]]),) + at[1:]
                raise AssertionError(f"{kernel} {mode} layer {layer}: err / bound {r_max:.3g} at (seq, head, row, d) {at}: "
                                     f"got {float(got[tuple([at[0] - s0, *at[1:]])]):.6g} want {float(ref[tuple([at[0] - s0, *at[1:]])]):.6g}")
            worst = max(worst, r_max)
            if mode == "census":
                liv = live.expand(len(seqs), h, nq, J)
                want = R.census_expected(v, liv)
                tol = R.census_tolerance(want, v, liv, bool(c["out_bf16"]))
                miss = (got - want).abs() > tol
                assert not bool(miss.any()), f"{kernel} census layer {layer}: {int(miss.sum())} elements off the exact average" \
                                             f" (first at {tuple(int(x) for x in torch.nonzero(miss)[0])})"
    WORST[kernel] = max(WORST.get(kernel, 0.0), worst)
    return worst


MODES = ("random", "census", "dominant")


def check(lib, dev, case, sync, modes=MODES, seed=0):
    """Runs `case` in each applicable mode and judges it; returns {mode: worst err / bound}."""
    result = {}
    for mode in modes:
        c = _defaults(case)
        if mode == "dominant" and not (c["bias"] or c["causal"]):
            continue  # no way to single out one key without a bias or ALiBi
        c, P = make_problem(case, mode, seed + 1000 * MODES.index(mode))
        outs = run(lib, dev, c, P, sync)
        result[mode] = judge(c, P, outs, mode, _model_kernel(case))
    return result


def _model_kernel(case):
    """The kernel whose arithmetic the output carries: the last of the case's kernels, or the prep kernel of
    phk_attention_tc (its bf16 roundings come before the wgmma kernel)."""
    k = case["kernel"]
    if isinstance(k, tuple):
        return "attention_prep_kernel" if "attention_prep_kernel" in k else k[-1]
    return k


def kernels_of(case):
    k = case["kernel"]
    return set(k) if isinstance(k, tuple) else {k}
