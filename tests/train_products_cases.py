"""Check bodies of the training products, shared by tests/test_gpu_train_products.py (H100) and
tests/test_train_products_emulated_cpu.py (the CPU executor): each drives one internal function of csrc/train.cu
through the probe library (tests/train_probe.py) and compares it with the float64 references and bars of
tests/train_products_ref.py.

Outputs the kernel must overwrite are prefilled with NaN, outputs it accumulates into with random values, and every
buffer carries sentinels around (and, for strided products, between) the output rows, which must come back bit-exact."""
import ctypes as C

import torch

from oracle import phenaki_oracle as O
from phenaki_pytorch_b200 import _lib as L
from tests import train_products_ref as R

NAN = float("nan")
SENT = 16  # sentinel floats before and after every output buffer


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _randn(shape, seed, dev, scale=1.0):
    return (torch.randn(shape, generator=_g(seed)) * scale).to(dev)


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _guarded(n, seed, dev):
    """a buffer of n floats with SENT random sentinels on each side: (whole buffer, its initial copy, the inner view)"""
    buf = _randn((n + 2 * SENT,), seed, dev)
    return buf, buf.clone(), buf[SENT:SENT + n]


def _same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# ---------------------------------------------------------------------------------------------------------------------
# A. strided batched product: sgemm_strided_kernel / hgemm_strided_kernel through sgemm_batched
# ---------------------------------------------------------------------------------------------------------------------
def check_strided(lib, dev, c, bf16, sync):
    """c: M, N, K, a_kfast, b_kfast, acc (0 | 1 | 2), outer, div; split-K (acc 2): K is the slice, k_total the length,
    count the batch entries (trailing ones may have an empty slice).  The operands are token-major with the `div` inner
    entries (heads) interleaved within each row, as dO, P and the key / query blocks of the attention backward."""
    M, N, K, acc = c["M"], c["N"], c["K"], c["acc"]
    split = acc == 2
    outer, div = (1, 1) if split else (c.get("outer", 1), c.get("div", 1))
    k_len = c["k_total"] if split else K  # the reduction length of one output element
    count = c["count"] if split else outer * div
    if c["a_kfast"]:  # A(m, k) = A[m * sam + k * sak]
        sam, sak, a_in, a_out = div * k_len, 1, k_len, M * div * k_len
    else:
        sam, sak, a_in, a_out = 1, div * M, M, k_len * div * M
    if c["b_kfast"]:  # B(k, n) = B[k * sbk + n * sbn]
        sbk, sbn, b_in, b_out = 1, div * k_len, k_len, N * div * k_len
    else:
        sbk, sbn, b_in, b_out = div * N, 1, N, k_len * div * N
    A = _randn((outer * div * M * k_len,), c["seed"], dev)
    B = _randn((outer * div * N * k_len,), c["seed"] + 1, dev)
    ldc = N + 3  # columns N .. ldc - 1 of every row are sentinels, as are SENT floats on either side
    c_in, c_out = M * ldc, div * M * ldc
    cbuf, _, Cv = _guarded(outer * div * M * ldc, c["seed"] + 2, dev)
    is_out = torch.zeros(cbuf.numel(), dtype=torch.bool, device=dev)
    is_out[SENT:SENT + Cv.numel()].view(-1, ldc)[:, :N] = True
    if acc == 0:
        cbuf[is_out] = NAN
    cbuf0 = cbuf.clone()
    prefill = Cv.view(outer * div, M, ldc)[:, :, :N].clone()
    if split:  # batch entry z reads K range [z * K, ...): the operands advance by K along k
        gb = (count, 1, K * sak, 0, K * sbk, 0, 0, 0, k_len)
    else:
        gb = (count, div, a_out, a_in, b_out, b_in, c_out, c_in, 0)
    sync()
    L.check(lib.probe_sgemm_batched(_p(A), sam, sak, _p(B), sbk, sbn, _p(Cv), ldc, M, N, K, acc, *gb, int(bf16),
                                    L.stream_ptr()), "probe_sgemm_batched")
    sync()
    got = Cv.view(outer * div, M, ldc)[:, :, :N]
    name = f"strided {'bf16' if bf16 else 'f32'} {c['id']}"
    assert _same_bits(cbuf[~is_out], cbuf0[~is_out]), f"{name}: sentinel overwritten"
    entries = [(0, 0)] if split else [(o, i) for o in range(outer) for i in range(div)]
    for e, (o, i) in enumerate(entries):
        Ae = torch.as_strided(A, (M, k_len), (sam, sak), o * a_out + i * a_in)
        Be = torch.as_strided(B, (k_len, N), (sbk, sbn), o * b_out + i * b_in)
        pre = prefill[e].double() if acc else None
        base = pre if pre is not None else 0.0
        adds = (count if split else 1)
        if bf16:
            ah, bh = R.rne(Ae), R.rne(Be)
            ref = ah @ bh + base
            bar = R.bf16_bar(ah, bh, pre, adds)
            alts = {"round-toward-zero": R.rtz(Ae) @ R.rtz(Be) + base, "unrounded": R.exact(Ae) @ R.exact(Be) + base}
            R.assert_within(f"{name} [{o},{i}]", got[e], ref, bar, alts)
        else:
            ref = Ae.double() @ Be.double() + base
            R.assert_within(f"{name} [{o},{i}]", got[e], ref, R.f32_bar(Ae, Be, k_len, pre, adds))


# ---------------------------------------------------------------------------------------------------------------------
# B. nn.Linear products: linear_fwd / dgrad_p / wgrad_p, fp32 and bf16 (operands cast to bf16, wgmma GEMM)
# ---------------------------------------------------------------------------------------------------------------------
def _pad8(v):
    return (v + 7) // 8 * 8


def tc_need(op, M, N, K):
    """bf16 operand elements of each of the two scratch buffers (leading dimension padded to 8)"""
    if op == "fwd":    # X [M, K], W [N, K]
        return max(M * _pad8(K), N * _pad8(K))
    if op == "dgrad":  # dY [M, N], W^T [K, N]
        return max(M * _pad8(N), K * _pad8(N))
    return max(N * _pad8(M), K * _pad8(M))  # wgrad: dY^T [N, M], X^T [K, M]


OPS = {"fwd": 0, "dgrad": 1, "wgrad": 2}


def _tc_scratch(elems, dev):
    # 0xFFFF bf16 = NaN: a product that read padding or stale scratch would come out NaN
    return torch.full((2 * elems,), -1, dtype=torch.int16, device=dev)


def check_linear(lib, dev, c, prec, sync):
    """c: op (fwd | dgrad | wgrad), M rows, N, K as nn.Linear(K -> N) over M rows; fwd: bias, residual; dgrad: acc"""
    op, M, N, K, seed = c["op"], c["M"], c["N"], c["K"], c["seed"]
    bf16 = prec == L.PREC_BF16
    W = _randn((N, K), seed, dev, K ** -0.5)
    bias = None
    if op == "fwd":
        a, b = _randn((M, K), seed + 1, dev), W
        shape, adds = (M, N), 0
        if c.get("bias"):
            bias = _randn((N,), seed + 2, dev)
            adds += 1
        if c.get("residual"):
            adds += 1
    elif op == "dgrad":
        a, b = _randn((M, N), seed + 1, dev), W
        shape, adds = (M, K), int(c.get("acc", 0))
    else:
        a, b = _randn((M, N), seed + 1, dev), _randn((M, K), seed + 2, dev)
        shape, adds = (N, K), 1
    buf, buf0, out = _guarded(shape[0] * shape[1], seed + 3, dev)
    out = out.view(shape)
    accumulates = (op == "fwd" and c.get("residual")) or (op == "dgrad" and c.get("acc")) or op == "wgrad"
    if not accumulates:
        out.fill_(NAN)
    prefill = out.clone() if accumulates else None
    elems = tc_need(op, M, N, K)
    scratch = _tc_scratch(elems, dev) if bf16 else None
    sync()
    L.check(lib.probe_linear(OPS[op], prec, _p(scratch), elems if bf16 else 0, _p(a), _p(b), _p(out), M, N, K, _p(bias),
                             _p(out) if (op == "fwd" and c.get("residual")) else None, int(c.get("acc", 0)),
                             L.stream_ptr()), "probe_linear")
    sync()
    name = f"linear {op} {'bf16' if bf16 else 'f32'} {c['id']}"
    assert _same_bits(buf[:SENT], buf0[:SENT]) and _same_bits(buf[-SENT:], buf0[-SENT:]), f"{name}: sentinel overwritten"
    # as products  X . W^T  (fwd),  dY . W  (dgrad),  dY^T . X  (wgrad)
    if op == "fwd":
        lhs, rhs, k_len = a, b.t(), K
    elif op == "dgrad":
        lhs, rhs, k_len = a, b, N
    else:
        lhs, rhs, k_len = a.t(), b, M
    extra = 0.0
    mag_extra = None
    if prefill is not None:
        extra = prefill.double()
        mag_extra = prefill.double().abs()
    if bias is not None:
        extra = extra + bias.double()
        mag_extra = bias.double().abs() if mag_extra is None else mag_extra + bias.double().abs()
    mag_pre = None if mag_extra is None else mag_extra.expand(shape)
    if bf16:
        ah, bh = R.rne(lhs), R.rne(rhs)
        ref = ah @ bh + extra
        bar = R.bf16_bar(ah, bh, mag_pre, max(adds, 1))
        alts = {"round-toward-zero": R.rtz(lhs) @ R.rtz(rhs) + extra, "unrounded": R.exact(lhs) @ R.exact(rhs) + extra}
        R.assert_within(name, out, ref, bar, alts)
    else:
        ref = lhs.double() @ rhs.double() + extra
        parts = -(-M // 256) if (op == "wgrad" and N * K <= 4 * 64 * 64 and M >= 1024) else 1  # split-K wgrad
        R.assert_within(name, out, ref, R.f32_bar(lhs, rhs, k_len, mag_pre, adds + parts))


def check_linear_workspace(lib, dev, c, sync):
    """bf16 mode with an operand scratch one element too small: PHK_E_WORKSPACE, and no kernel launched"""
    op, M, N, K = c["op"], c["M"], c["N"], c["K"]
    elems = tc_need(op, M, N, K) - 1
    scratch = _tc_scratch(elems, dev)
    a_shape, b_shape, out_shape = {"fwd": ((M, K), (N, K), (M, N)), "dgrad": ((M, N), (N, K), (M, K)),
                                   "wgrad": ((M, N), (M, K), (N, K))}[op]
    a, b, out = (torch.zeros(s_, device=dev) for s_ in (a_shape, b_shape, out_shape))
    sync()
    before = lib.phk_launch_count()
    rc = lib.probe_linear(OPS[op], L.PREC_BF16, _p(scratch), elems, _p(a), _p(b), _p(out), M, N, K, None, None, 0,
                          L.stream_ptr())
    assert rc == -4, f"linear {op} {M}x{N}x{K}: scratch of {elems} elements accepted (rc {rc})"
    assert lib.phk_launch_count() == before, f"linear {op} {M}x{N}x{K}: a refused call launched kernels"
    sync()


# ---------------------------------------------------------------------------------------------------------------------
# C. attention backward
# ---------------------------------------------------------------------------------------------------------------------
class AttnProblem:
    def __init__(self, c, dev):
        b, H, n, m, nnull, dh = c["b"], c["H"], c["n"], c["m"], c.get("nnull", 0), c.get("dh", 64)
        self.c, self.dev = c, dev
        self.b, self.H, self.n, self.m, self.nnull, self.dh = b, H, n, m, nnull, dh
        self.nkt, I = nnull + m, H * dh
        self.I = I
        s = c["seed"]
        self.q = _randn((b * n, I), s, dev)
        self.kv = _randn((b * m, 2 * I), s + 1, dev)
        self.null_kv = _randn((H, 2 * max(nnull, 1), dh), s + 2, dev)
        self.q_scale = (1.0 + 0.25 * torch.randn(dh, generator=_g(s + 3))).to(dev)
        self.k_scale = (1.0 + 0.25 * torch.randn(dh, generator=_g(s + 4))).to(dev)
        self.dO = _randn((b * n, I), s + 5, dev)
        self.bias = None
        if c.get("bias") == "cpb":
            self.bias = _randn((H, n, m), s + 6, dev)
        elif c.get("bias") == "alibi":  # alibi_causal_bias_kernel: -|j - i| * slope for j <= i, -FLT_MAX above
            slopes = torch.tensor([2.0 ** (-8.0 * (h + 1) / H) for h in range(H)])
            i = torch.arange(n)[:, None]
            j = torch.arange(m)[None, :]
            al = -(j - i).abs().float()[None] * slopes[:, None, None]
            self.bias = torch.where(j > i, torch.full_like(al, -torch.finfo(torch.float32).max), al).to(dev)
        self.key_mask = None
        if c.get("mask"):
            km = torch.rand((b, m), generator=_g(s + 7)) < 0.7
            km[:, 0] = True
            if c.get("cfg_null"):  # the CFG null half: one sequence's text fully masked (only the null keys stay live)
                km[-1] = False
            self.key_mask = km.to(torch.uint8).to(dev)

    def attn_t(self, null_kv, q_scale, k_scale):
        a = L.AttnT()
        a.null_kv, a.q_scale, a.k_scale = _p(null_kv), _p(q_scale), _p(k_scale)
        a.num_null_kv = self.nnull
        return a

    def layout(self, lib):
        out = (C.c_int64 * 9)()
        L.check(lib.probe_attn_bwd_layout(self.b, self.H, self.n, self.m, self.nnull, self.dh, out), "layout")
        return list(out)

    def run(self, lib, bf16, sync, seed):
        """one attention_backward call: (outputs, accumulator prefills, scratch)"""
        dev, H, dh = self.dev, self.H, self.dh
        lay = self.layout(lib)
        scratch = torch.full((lay[8],), NAN, device=dev)
        dq = torch.full((self.b * self.n, self.I), NAN, device=dev)
        dkv = torch.full((self.b * self.m, 2 * self.I), NAN, device=dev)
        pre = {"null_kv": _randn(self.null_kv.shape, seed, dev, 1e-2), "q_scale": _randn((dh,), seed + 1, dev, 1e-2),
               "k_scale": _randn((dh,), seed + 2, dev, 1e-2)}
        if self.bias is not None:
            pre["bias"] = _randn(self.bias.shape, seed + 3, dev, 1e-4)
        guarded = {k: _guarded(v.numel(), 0, dev) for k, v in pre.items()}  # accumulators with sentinels around them
        out = {}
        for k, (_, _, inner) in guarded.items():
            inner.copy_(pre[k].reshape(-1))
            out[k] = inner.view(pre[k].shape)
        A = self.attn_t(self.null_kv, self.q_scale, self.k_scale)
        G = self.attn_t(out["null_kv"], out["q_scale"], out["k_scale"])
        sync()
        L.check(lib.probe_attention_backward(_p(self.q), _p(self.kv), C.byref(A), C.byref(G), _p(self.bias),
                                             _p(self.key_mask), _p(self.dO), _p(dq), _p(dkv), _p(out.get("bias")),
                                             self.b, H, self.n, self.m, self.nnull, dh, _p(scratch), int(bf16),
                                             L.stream_ptr()), "probe_attention_backward")
        sync()
        for k, (buf, buf0, _) in guarded.items():
            assert _same_bits(buf[:SENT], buf0[:SENT]) and _same_bits(buf[-SENT:], buf0[-SENT:]), f"d{k}: sentinel overwritten"
        out["q"], out["kv"] = dq, dkv
        return out, pre, scratch, lay

    def scratch_views(self, scratch, lay):
        bh, n, nkt, dh = self.b * self.H, self.n, self.nkt, self.dh
        shapes = [(n, dh), (nkt, dh), (nkt, dh), (n, nkt), (n, nkt), (n, dh), (nkt, dh), (nkt, dh)]
        names = ["qh", "kh", "vv", "P", "dS", "preQ", "preK", "preV"]
        return {k: scratch[o:o + bh * r * cc].view(bh, r, cc) for k, o, (r, cc) in zip(names, lay, shapes)}

    def autograd(self):
        """float64 autograd of oracle.attention_core: gradients of sum(O * dO)"""
        b, H, n, m, nnull, dh = self.b, self.H, self.n, self.m, self.nnull, self.dh
        q = self.q.double().requires_grad_()
        kv = self.kv.double().requires_grad_()
        nkv = self.null_kv.double().requires_grad_()
        qs = self.q_scale.double().requires_grad_()
        ks = self.k_scale.double().requires_grad_()
        bias = self.bias.double().requires_grad_() if self.bias is not None else None
        qq = q.view(b, n, H, dh).permute(0, 2, 1, 3)
        kk = kv.view(b, m, 2, H, dh)[:, :, 0].permute(0, 2, 1, 3)
        vv = kv.view(b, m, 2, H, dh)[:, :, 1].permute(0, 2, 1, 3)
        if nnull:
            kk = torch.cat((nkv[:, 0:2 * nnull:2].unsqueeze(0).expand(b, -1, -1, -1), kk), dim=2)
            vv = torch.cat((nkv[:, 1:2 * nnull:2].unsqueeze(0).expand(b, -1, -1, -1), vv), dim=2)
        mask = self.key_mask.bool() if self.key_mask is not None else None
        o = O.attention_core(qq, kk, vv, qs, ks, heads=H, num_null_kv=nnull, mask=mask, attn_bias=bias)
        (o * self.dO.double().view(b, n, H, dh).permute(0, 2, 1, 3)).sum().backward()
        g = {"q": q.grad, "kv": kv.grad, "q_scale": qs.grad, "k_scale": ks.grad}
        g["null_kv"] = nkv.grad if nnull else torch.zeros_like(nkv, dtype=torch.float64)
        if bias is not None:
            g["bias"] = bias.grad
        return g

    def grads_from_products(self, preQ, preK, preV, dS):
        """float64 l2norm / scale backward applied to the dq / dk / dv contractions [b*H, rows, dh] (and dbias from dS)"""
        b, H, n, m, nnull, dh, nkt = self.b, self.H, self.n, self.m, self.nnull, self.dh, self.nkt
        q = self.q.double().view(b, n, H, dh).permute(0, 2, 1, 3)
        kraw = self.kv.double().view(b, m, 2, H, dh)[:, :, 0].permute(0, 2, 1, 3)
        if nnull:
            kraw = torch.cat((self.null_kv.double()[:, 0:2 * nnull:2].unsqueeze(0).expand(b, -1, -1, -1), kraw), dim=2)
        dq, dqs = R.l2norm_scale_bwd(q, self.q_scale, 8.0 * preQ.view(b, H, n, dh))
        dk, dks = R.l2norm_scale_bwd(kraw, self.k_scale, 8.0 * preK.view(b, H, nkt, dh))
        dv = preV.view(b, H, nkt, dh)
        g = {"q": dq.permute(0, 2, 1, 3).reshape(b * n, H * dh), "q_scale": dqs.sum((0, 1, 2)),
             "k_scale": dks.sum((0, 1, 2))}
        kv = torch.stack((dk[:, :, nnull:], dv[:, :, nnull:]), dim=1)  # [b, 2, H, m, dh]
        g["kv"] = kv.permute(0, 3, 1, 2, 4).reshape(b * m, 2 * H * dh)
        nk = torch.zeros((H, 2 * max(nnull, 1), dh), dtype=torch.float64, device=self.dev)
        if nnull:
            nk[:, 0:2 * nnull:2] = dk[:, :, :nnull].sum(0)
            nk[:, 1:2 * nnull:2] = dv[:, :, :nnull].sum(0)
        g["null_kv"] = nk
        if self.bias is not None:
            g["bias"] = dS.view(b, H, n, nkt)[..., nnull:].sum(0)
        return g


def _compare_grads(name, out, pre, ref, check):
    """outputs the kernel accumulates into hold prefill + gradient (the fp32 sum is compared, not a difference)"""
    for k in ref:
        check(f"{name} d{k}", out[k], ref[k] + pre[k].double() if k in pre else ref[k])


def check_attention_f32(lib, dev, c, sync):
    P = AttnProblem(c, dev)
    out, pre, _, _ = P.run(lib, False, sync, c["seed"] + 10)
    _compare_grads(f"attention f32 {c['id']}", out, pre, P.autograd(), R.assert_close_norms)


def check_attention_bf16(lib, dev, c, sync):
    P = AttnProblem(c, dev)
    name = f"attention bf16 {c['id']}"
    out32, _, scr32, lay = P.run(lib, False, sync, c["seed"] + 10)
    out, pre, scr, _ = P.run(lib, True, sync, c["seed"] + 10)
    V32, V = P.scratch_views(scr32, lay), P.scratch_views(scr, lay)
    # the score product stays fp32 in bf16 mode: the recomputed operands and probabilities are bit-identical
    for k in ("qh", "kh", "vv", "P"):
        assert _same_bits(V[k], V32[k]), f"{name}: {k} differs from the fp32-mode call"
    b, H, n, nkt, dh = P.b, P.H, P.n, P.nkt, P.dh
    dO = P.dO.view(b, n, H, dh).permute(0, 2, 1, 3).reshape(b * H, n, dh)
    Pk, dS, vv = V["P"].double(), V["dS"], V["vv"]
    # dP = bf16(dO) . bf16(vv)^T on hgemm_strided_kernel, then dS = P (dP - sum_j P dP) in fp32
    def ds_of(dp):
        return Pk * (dp - (Pk * dp).sum(-1, keepdim=True))
    dp_ref = R.rne(dO) @ R.rne(vv).transpose(1, 2)
    bar_dp = R.bf16_bar(R.rne(dO), R.rne(vv).transpose(1, 2))
    # the dP bar carried through the softmax backward, plus its own fp32 rounding (the row dot product over nkt terms)
    mag = (Pk * dp_ref.abs()).sum(-1, keepdim=True)
    bar_ds = Pk * (bar_dp + (Pk * bar_dp).sum(-1, keepdim=True) + (nkt + 2) * R.U * (mag + dp_ref.abs()))
    alts = {"round-toward-zero": ds_of(R.rtz(dO) @ R.rtz(vv).transpose(1, 2)),
            "unrounded": ds_of(R.exact(dO) @ R.exact(vv).transpose(1, 2))}
    R.assert_within(f"{name} dS", dS, ds_of(dp_ref), bar_ds, alts)
    if n * nkt >= 64 * 64:  # the three contractions on hgemm_strided_kernel, operands read back from the scratch
        kh, qh = V["kh"], V["qh"]
        for k, a, bb in (("preQ", dS, kh), ("preK", dS.transpose(1, 2), qh), ("preV", V["P"].transpose(1, 2), dO)):
            ah, bh = R.rne(a), R.rne(bb)
            R.assert_within(f"{name} {k}", V[k], ah @ bh, R.bf16_bar(ah, bh),
                            {"round-toward-zero": R.rtz(a) @ R.rtz(bb), "unrounded": R.exact(a) @ R.exact(bb)})
        fin = P.grads_from_products(V["preQ"].double(), V["preK"].double(), V["preV"].double(), dS.double())
    else:  # loop path: the contractions run in fp32 on the kernel's own dS and P
        dSd = dS.double()
        fin = P.grads_from_products(dSd @ V["kh"].double(), dSd.transpose(1, 2) @ V["qh"].double(),
                                    Pk.transpose(1, 2) @ dO.double(), dSd)
    _compare_grads(f"{name} (from its own products)", out, pre, fin, R.assert_close_norms)
    _compare_grads(f"{name} (closeness)", out, pre, P.autograd(), R.assert_step_grade)


def check_layout(lib, c, dev="cpu"):
    """attn_bwd_bufs carves eight consecutive buffers, and attn_bwd_scratch_floats covers them"""
    P = AttnProblem(c, dev)
    lay = P.layout(lib)
    bh, n, nkt, dh = P.b * P.H, P.n, P.nkt, P.dh
    sizes = [n * dh, nkt * dh, nkt * dh, n * nkt, n * nkt, n * dh, nkt * dh, nkt * dh]
    off = 0
    for o, s in zip(lay[:8], sizes):
        assert o == off
        off += bh * s
    assert off <= lay[8]


# ---------------------------------------------------------------------------------------------------------------------
# D. colsum (bias gradients): out[c] += sum_r x[r, c]
# ---------------------------------------------------------------------------------------------------------------------
def check_colsum(lib, dev, rows, cols, sync, seed=7):
    ld = cols + 5
    x = _randn((rows, ld), seed, dev)
    buf, buf0, out = _guarded(cols, seed + 1, dev)
    pre = out.clone()
    sync()
    L.check(lib.probe_colsum(_p(x), rows, cols, ld, _p(out), L.stream_ptr()), "probe_colsum")
    sync()
    name = f"colsum {rows}x{cols}"
    assert _same_bits(buf[:SENT], buf0[:SENT]) and _same_bits(buf[-SENT:], buf0[-SENT:]), f"{name}: sentinel overwritten"
    xs = x[:, :cols].double()
    ref = xs.sum(0) + pre.double()
    # serial fp32 sums over row chunks, at most 64 chunks meet through atomics onto the prefill
    bar = (rows + 65) * R.U * (xs.abs().sum(0) + pre.double().abs())
    R.assert_within(name, out, ref, bar)
