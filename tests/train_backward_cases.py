"""Check bodies of the rest of the training backward, shared by tests/test_gpu_train_backward.py (H100) and
tests/test_train_backward_emulated_cpu.py (the CPU executor): LayerNorm (E), GEGLU with dropout (F), PEG (G), the
embeddings (H), the position-bias MLP (I) and the head losses (J), each one function of csrc/train.cu driven through the
probe library (tests/train_probe.py) and compared with float64 torch autograd of an independent statement of the
forward (oracle/phenaki_oracle.py, F.gelu, F.cross_entropy, F.binary_cross_entropy_with_logits), applied to the exact
fp32 inputs the kernel received.  As in tests/train_products_cases.py, outputs the kernel overwrites are prefilled with
NaN, outputs it accumulates into with random values (the reference adds them), every output carries SENT sentinels on
both sides that must come back bit-exact, and every case prints its worst err / bar.

Bars, per output element; U = 2^-23 (one fp32 ulp relative, twice the unit roundoff), first order in U:
  sums      (k + adds) U sum|terms|: the recursive-summation bound of k terms plus the `adds` further additions (atomics
            or slots across row chunks, the prefill).  It holds for any order.  For the warp-per-row kernels
            (LayerNorm dx, the BCE score) k is the depth of the order they use, ceil(dim / 32) lane-serial terms plus 5
            shuffle levels.
  LayerNorm dx = rstd (a' - c1 - xhat c2), a' = dy g, c1 = mean(a'), c2 = mean(a' xhat).  With a = |dy g|,
            A1 = mean a, A2 = mean(a |xhat|), m = mean|x| rstd and k = ceil(dim / 32) + 5: the fp32 mean is off by at
            most (k + 1) U mean|x| (a shift s <= (k + 1) U m of every xhat), rstd by ((k + 4) / 2 + 2) U relative (the
            variance sum, rsqrtf's 2 ulp), xhat by |xhat| (k + 12) / 2 U + s, c1 and c2 by (k + 2) U A1|2 plus the
            propagated xhat error, the final expression by 4 roundings.  Collecting the coefficients:
                bar = 3 (k + 8) U (1 + m) rstd (a + A1 + |xhat| A1 + (1 + |xhat|) A2)   (+ U |dx| prefill, accumulate)
            dgamma / dbeta: column sums over rows of dy xhat / dy (row chunks meet through <= 64 atomics or slots):
                (rows + 66) U (sum|dy xhat| + |prefill|) + (k + 8) U sum_r |dy| (|xhat| + m_r).
  GEGLU     g = 0.5 gate (1 + erff(z)) val M, z = gate / sqrt 2, M the dropout multiplier; erff is within 2 ulp, expf
            within 2 ulp (CUDA C Programming Guide, no --use_fast_math).  With Phi = 0.5 (1 + erf z), phi the normal
            density and E = |z| exp(-z^2) (erf's sensitivity to z's rounding):
                g:     U |gate val M| (1 + 5 Phi + E)
                dval:  U |dg M gate| (1 + 4 Phi + E)
                dgate: U |dg M val| (1 + 5 Phi + E + |gate| phi (8 + gate^2))
  PEG       dx = dy + 27 fused taps: 28 U (|dy| + sum_tap |w| |dy_o|); dw: (P + 17) U (sum_o |dy x_src| + |prefill|)
            (16 chunks of positions meet through atomics or slots); db: colsum, (P + 65) U (sum|dy| + |prefill|).
  embeddings  dtok[id]: (count_id + 3) U (sum |alpha dx| + |prefill|); dpos[p]: (sequences + 3) U (same).
  position-bias MLP  a running-error bound: every fp32 value is within (its own bound) + (the propagated bounds of its
            operands) of float64, each product / sum of k terms adding k U times the same product on absolute values
            (|A| |B|), logf 1 ulp, leaky ReLU's slope 1 or 0.1.  A pre-activation within its error bound of 0 may take
            the other slope in fp32: its 0.9 |gradient| is added to the bound and carried on like any other error.
  CE        p = expf(l - mx) / s with s a block sum of V terms (depth ceil(V / 256) + 10): p is within
            (|l - mx| + 6 + depth + sum_v p_v |l_v - mx|) U p; dlogits = (p - onehot) k within
            |k| (that + 3 U |p - onehot| + 2^-126), the last term for a p below fp32's normal range (expf underflows);
            the row loss (mx + logf s - l_t) / count within (the sum's relative error + 4 U |terms|) / count; the
            reduced loss (ceil(R / 1024) + 10) U sum|row| + sum of the row bars.
  BCE       a = emb . w + b within ea = (ceil(D / 32) + 6) U (|emb| |w| + |b|); sigmoid within
            sigma (1 - sigma) ea + sigma ((1 - sigma)(2 + |a|) + 3) U; dscore = (sigma - y) scale / R within
            |scale / R| (that + 3 U |sigma - y| + 2^-126), the last term for a sigma below fp32's normal range (expf(100)
            overflows to inf and sigma(-100) comes out 0).  Row loss (max(a, 0) - a y + log1pf(expf(-|a|))) / R within
            (ea + (2 + |a|) U e^-|a| + U (|max(a, 0)| + |a y| + 3 |l|)) / R.
Each section also asserts that a slipped float64 reference (the alternatives listed there) breaks the same bar, so the
bars are tight enough to see those slips.
"""
import ctypes as C
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import phenaki_oracle as O
from phenaki_pytorch_b200 import _lib as L
from tests import dropout_ref
from tests import train_products_ref as R
from tests.train_products_cases import NAN, SENT, _g, _p, _randn, _same_bits

U = R.U
E_UNSUPPORTED, E_WORKSPACE = -3, -4


class Guarded:
    """named output buffers, each with SENT random sentinels on both sides; fill: 'nan' (overwritten) or 'rand'
    (accumulated into; the prefill is kept)"""

    def __init__(self, dev, seed):
        self.dev, self.seed, self.bufs = dev, seed, {}

    def add(self, name, shape, fill, scale=1.0):
        n = int(np.prod(shape))
        self.seed += 1
        buf = _randn((n + 2 * SENT,), self.seed, self.dev)
        inner = buf[SENT:SENT + n]
        if fill == "nan":
            inner.fill_(NAN)
        else:
            inner.mul_(scale)
        self.bufs[name] = (buf, buf.clone(), inner.view(shape))
        return inner.view(shape)

    def pre(self, name):
        return self.bufs[name][1][SENT:-SENT].view(self.bufs[name][2].shape).double()

    def check(self, what):
        for k, (buf, buf0, _) in self.bufs.items():
            assert _same_bits(buf[:SENT], buf0[:SENT]) and _same_bits(buf[-SENT:], buf0[-SENT:]), \
                f"{what}: sentinel of {k} overwritten"

    def untouched(self, what):
        for k, (buf, buf0, _) in self.bufs.items():
            assert _same_bits(buf, buf0), f"{what}: {k} written by a refused call"


class Det:
    """the deterministic-mode reduction scratch (t_det) of the probe for the duration of a `with` block"""

    def __init__(self, lib, dev, floats):
        self.lib, self.floats = lib, int(floats)
        self.buf = torch.full((max(self.floats, 1),), NAN, device=dev) if floats else None

    def __enter__(self):
        if self.buf is not None:
            self.lib.probe_set_det_scratch(_p(self.buf), self.floats)
        return self

    def __exit__(self, *exc):
        self.lib.probe_set_det_scratch(None, 0)


def _modes(lib, dev, det_floats, run, sync):
    """run(mode) under the default path and twice under the fixed-order path: the two fixed-order runs must be
    bit-identical.  Returns [(mode, outputs)] for the bar checks."""
    out = [("default", run("default"))]
    fixed = []
    for _ in range(2):
        with Det(lib, dev, det_floats):
            fixed.append(run("fixed"))
            sync()
    for k in (k for k in fixed[0] if not k.startswith("_")):
        assert _same_bits(fixed[0][k], fixed[1][k]), f"fixed-order {k} differs between two identical calls"
    out.append(("fixed", fixed[0]))
    return out


def _within(name, got, ref, bar, alts=None):
    """got within bar of ref everywhere (prints the margin); each alternative (a slipped reference) breaks the bar"""
    w = R.worst(got, ref, bar)
    print(f"[train-backward] {name}: worst err/bar {w:.3g}")
    assert w <= 1.0, f"{name}: error {w:.3g} x the bar"
    for label, alt in (alts or {}).items():
        wa = R.worst(alt, ref, bar)
        assert wa > 1.0, f"{name}: the {label} reference stays within the bar ({wa:.3g}): the bar cannot see it"


def _sizes(lib, cpb=None, d=(1, 1, 1), rows=1, dim=1):
    out = (C.c_int64 * 3)()
    c = cpb if cpb is not None else L.CpbT()
    L.check(lib.probe_scratch_floats(C.byref(c), d[0], d[1], d[2], rows, dim, out), "probe_scratch_floats")
    return list(out)


# ---------------------------------------------------------------------------------------------------------------------
# E. LayerNorm backward: ln_backward (ln_bwd_dx_kernel, ln_bwd_dgb_kernel | ln_bwd_dgb_fixed_kernel + add_slots)
# ---------------------------------------------------------------------------------------------------------------------
def _ln_inputs(rows, dim, seed, dev):
    """rows of very different scales (10^-2.5 .. 10^0.5, row 0 the narrowest) around random offsets: eps matters in
    the narrow rows"""
    gen = _g(seed)
    scale = 10.0 ** (torch.rand((rows, 1), generator=gen) * 3.0 - 2.5)
    scale[0] = 10.0 ** -2.5  # at least one row whose variance is comparable to eps
    x = (torch.randn((rows, dim), generator=gen) * scale + 0.5 * torch.randn((rows, 1), generator=gen)).to(dev)
    g = (1.0 + 0.5 * torch.randn((dim,), generator=gen)).to(dev)
    dy = torch.randn((rows, dim), generator=gen).to(dev)
    return x, g, dy


def _ln_ref(x, g, dy, unbiased=False, eps=1e-5):
    """float64 autograd of O.layer_norm (or a slipped statement of it): (dx, dgamma, dbeta)"""
    xd = x.double().requires_grad_()
    gd = g.double().requires_grad_()
    bd = torch.zeros_like(gd).requires_grad_()
    if not unbiased and eps == 1e-5:
        y = O.layer_norm(xd, gd, bd)
    else:
        mu = xd.mean(-1, keepdim=True)
        var = xd.var(-1, keepdim=True, unbiased=unbiased)
        y = (xd - mu) / torch.sqrt(var + eps) * gd + bd
    (y * dy.double()).sum().backward()
    return xd.grad, gd.grad, bd.grad


def check_layernorm(lib, dev, c, sync):
    """c: rows, dim, dx ('write' | 'acc' | None), dbeta (bool), seed"""
    rows, dim, seed = c["rows"], c["dim"], c["seed"]
    x, g, dy = _ln_inputs(rows, dim, seed, dev)
    ref_dx, ref_dg, ref_db = _ln_ref(x, g, dy)
    name = f"layernorm {c['id']}"
    # bars (module docstring)
    xd = x.double()
    mu = xd.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(xd.var(-1, keepdim=True, unbiased=False) + 1e-5)
    xh = (xd - mu) * rstd
    a = (dy.double() * g.double()).abs()
    A1, A2 = a.mean(-1, keepdim=True), (a * xh.abs()).mean(-1, keepdim=True)
    k = -(-dim // 32) + 5
    m = xd.abs().mean(-1, keepdim=True) * rstd
    bar_dx = 3 * (k + 8) * U * (1 + m) * rstd * (a + A1 + xh.abs() * A1 + (1 + xh.abs()) * A2)
    dyd = dy.double()
    bar_g_rows = (k + 8) * U * (dyd.abs() * (xh.abs() + m)).sum(0)
    alts_dx = {"variance 1/(dim-1)": _ln_ref(x, g, dy, unbiased=True)[0], "eps dropped": _ln_ref(x, g, dy, eps=0.0)[0]}

    def run(mode):
        G = Guarded(dev, seed + 100)
        dx = None
        if c["dx"] == "write":
            dx = G.add("dx", (rows, dim), "nan")
        elif c["dx"] == "acc":
            dx = G.add("dx", (rows, dim), "rand")
        dg = G.add("dgamma", (dim,), "rand")
        db = G.add("dbeta", (dim,), "rand") if c["dbeta"] else None
        stats = torch.full((2 * rows,), NAN, device=dev)
        sync()
        L.check(lib.probe_ln_backward(_p(x), _p(g), _p(dy), _p(dx), int(c["dx"] == "acc"), _p(dg), _p(db), _p(stats),
                                      rows, dim, L.stream_ptr()), "probe_ln_backward")
        sync()
        G.check(f"{name} ({mode})")
        out = {"dgamma": dg.clone()}
        for k_, v in (("dx", dx), ("dbeta", db)):
            if v is not None:
                out[k_] = v.clone()
        out["_G"] = G
        return out

    results = _modes(lib, dev, _sizes(lib, rows=rows, dim=dim)[1], run, sync)
    for mode, out in results:
        G = out.pop("_G")
        nm = f"{name} ({mode})"
        if "dx" in out:
            pre = G.pre("dx") if c["dx"] == "acc" else 0.0
            bar = bar_dx + (U * (G.pre("dx").abs() + ref_dx.abs()) if c["dx"] == "acc" else 0.0)
            # the slips change dx by ~ eps / (2 var) (eps dropped: ~15 % in the narrow row 0) and ~ 1 / (2 dim) relative
            # (1/(dim-1)), which the bar (~ (dim / 32 + 13) 2^-20 relative) resolves up to dim 512
            alts = {k_: v + pre for k_, v in alts_dx.items() if dim <= 512 or k_ == "eps dropped"}
            _within(f"{nm} dx", out["dx"], ref_dx + pre, bar, alts)
        pg = G.pre("dgamma")
        _within(f"{nm} dgamma", out["dgamma"], ref_dg + pg,
                (rows + 66) * U * ((dyd * xh).abs().sum(0) + pg.abs()) + bar_g_rows)
        if "dbeta" in out:
            pb = G.pre("dbeta")
            _within(f"{nm} dbeta", out["dbeta"], ref_db + pb, (rows + 66) * U * (dyd.abs().sum(0) + pb.abs()))


def check_layernorm_workspace(lib, dev, rows, dim, sync):
    """fixed-order path with one float less scratch than ln_det_floats: PHK_E_WORKSPACE, dgamma untouched"""
    x, g, dy = _ln_inputs(rows, dim, 5, dev)
    G = Guarded(dev, 11)
    dx = G.add("dx", (rows, dim), "nan")
    dg = G.add("dgamma", (dim,), "rand")
    db = G.add("dbeta", (dim,), "rand")
    stats = torch.full((2 * rows,), NAN, device=dev)
    need = _sizes(lib, rows=rows, dim=dim)[1]
    assert need == 2 * (-(-rows // 256)) * dim
    sync()
    with Det(lib, dev, need - 1):
        rc = lib.probe_ln_backward(_p(x), _p(g), _p(dy), _p(dx), 0, _p(dg), _p(db), _p(stats), rows, dim,
                                   L.stream_ptr())
    sync()
    assert rc == E_WORKSPACE, f"layernorm {rows}x{dim}: a scratch of {need - 1} floats accepted (rc {rc})"
    G.check(f"layernorm workspace {rows}x{dim}")
    for k in ("dgamma", "dbeta"):
        buf, buf0, _ = G.bufs[k]
        assert _same_bits(buf, buf0), f"layernorm workspace: {k} written by a refused call"


# ---------------------------------------------------------------------------------------------------------------------
# F. GEGLU forward with dropout (geglu_dropout_fwd: geglu_dropout_kernel | phk_geglu) and backward (geglu_bwd_kernel)
# ---------------------------------------------------------------------------------------------------------------------
SEED_K = 0x1234_5678_9ABC_DEF1


def _site(p):
    """(p, scale, k0, k1, base) as the training step's DropSite: scale = 1 / (1 - p) in fp32 (inf at p = 1)"""
    with np.errstate(divide="ignore"):
        scale = float(np.float32(1.0) / (np.float32(1.0) - np.float32(p))) if p > 0 else 0.0
    return float(p), scale, SEED_K & 0xFFFFFFFF, SEED_K >> 32, 77


def check_geglu(lib, dev, c, sync):
    """c: rows, inner, p, seed"""
    rows, inner, p, seed = c["rows"], c["inner"], c["p"], c["seed"]
    h = _randn((rows, 2 * inner), seed, dev, 2.0)
    dg = _randn((rows, inner), seed + 1, dev)
    site = _site(p)
    if p > 0:
        Mk = dropout_ref.multiplier(dropout_ref.keep(SEED_K, site[4], rows * inner, p), p, torch.float64)
        Mk = Mk.view(rows, inner).to(dev)
    else:
        Mk = torch.ones((rows, inner), dtype=torch.float64, device=dev)
    name = f"geglu {c['id']}"
    G = Guarded(dev, seed + 10)
    g = G.add("g", (rows, inner), "nan")
    dh = G.add("dh", (rows, 2 * inner), "nan")
    sync()
    L.check(lib.probe_geglu_dropout_fwd(_p(h), _p(g), rows, inner, *site, L.stream_ptr()), "probe_geglu_dropout_fwd")
    L.check(lib.probe_geglu_backward(_p(h), _p(dg), _p(dh), rows, inner, *site, L.stream_ptr()), "probe_geglu_backward")
    sync()
    G.check(name)

    def ref(approx):
        hd = h.double().requires_grad_()
        val, gate = hd[:, :inner], hd[:, inner:]
        out = F.gelu(gate, approximate=approx) * val * Mk
        (out * dg.double()).sum().backward()
        return out.detach(), hd.grad

    g_ref, dh_ref = ref("none")
    g_tanh, dh_tanh = ref("tanh")
    hd = h.double()
    val, gate = hd[:, :inner], hd[:, inner:]
    z = gate / math.sqrt(2.0)
    Phi = 0.5 * (1.0 + torch.erf(z))
    phi = torch.exp(-0.5 * gate * gate) / math.sqrt(2.0 * math.pi)
    E = z.abs() * torch.exp(-z * z)
    dM = (dg.double() * Mk).abs()
    bar_g = U * (gate * val * Mk).abs() * (1 + 5 * Phi + E)
    bar_dval = U * dM * gate.abs() * (1 + 4 * Phi + E)
    bar_dgate = U * dM * val.abs() * (1 + 5 * Phi + E + gate.abs() * phi * (8 + gate * gate))
    tanh_visible = p < 1  # p = 1: everything is 0 whichever GELU
    _within(f"{name} g", g, g_ref, bar_g, {"tanh-GELU": g_tanh} if tanh_visible else None)
    _within(f"{name} dh", dh, dh_ref, torch.cat((bar_dval, bar_dgate), 1),
            {"tanh-GELU": dh_tanh} if tanh_visible else None)
    if p >= 1:
        assert not torch.isnan(g).any() and not (g != 0).any() and not (dh != 0).any(), f"{name}: p = 1 is not zeros"


# ---------------------------------------------------------------------------------------------------------------------
# G. PEG backward: peg_backward (colsum for db, peg_bwd_dw_kernel | peg_bwd_dw_fixed_kernel + add_slots, peg_bwd_kernel)
# ---------------------------------------------------------------------------------------------------------------------
def _peg_y(x, W, b, shape, causal, flip=False, pad_causal=None):
    """O.peg + residual on x [B, THW, D]; W the parameter [D, 1, 3, 3, 3]; the slips: flip (convolution in place of
    correlation), pad_causal (the other temporal padding)"""
    sd = {"dsconv.weight": W.flip(2, 3, 4) if flip else W, "dsconv.bias": b}
    return O.peg(x, shape, sd, "", pad_causal if pad_causal is not None else causal) + x


def _peg_ref(x, W, b, dy, shape, causal, **slip):
    xd, Wd, bd = (t.double().requires_grad_() for t in (x, W, b))
    (_peg_y(xd, Wd, bd, shape, causal, **slip) * dy.double()).sum().backward()
    return xd.grad, Wd.grad.reshape(W.shape[0], 27), bd.grad


def check_peg(lib, dev, c, sync):
    """c: B, T, H, W, D, causal, seed"""
    B, T, H, Wd_, D, causal, seed = c["B"], c["T"], c["H"], c["W"], c["D"], c["causal"], c["seed"]
    shape = (B, T, H, Wd_)
    P = B * T * H * Wd_
    x = _randn((B, T * H * Wd_, D), seed, dev)
    W = _randn((D, 1, 3, 3, 3), seed + 1, dev, 0.2)
    b = _randn((D,), seed + 2, dev)
    dy = _randn((B, T * H * Wd_, D), seed + 3, dev)
    w27 = W.reshape(D, 27).t().contiguous()  # the forward's tap-major layout
    pad_t0 = 2 if causal else 1
    ref = _peg_ref(x, W, b, dy, shape, causal)
    alts = {"taps flipped": _peg_ref(x, W, b, dy, shape, causal, flip=True)}
    if T > 1:
        alts["causal pad 1" if causal else "causal pad 2 on a non-causal PEG"] = _peg_ref(x, W, b, dy, shape, causal,
                                                                                          pad_causal=not causal)
    # magnitudes: the same linear maps on absolute values
    Wa = W.double().abs()
    xa = x.double().abs().requires_grad_()
    Wm = Wa.clone().requires_grad_()
    zero = torch.zeros(D, dtype=torch.float64, device=dev)
    (O.peg(xa, shape, {"dsconv.weight": Wm, "dsconv.bias": zero}, "", causal) * dy.double().abs()).sum().backward()
    mag_dx, mag_dw = xa.grad, Wm.grad.reshape(D, 27)  # sum_tap |w| |dy_o| ; sum_o |dy| |x_src|
    name = f"peg {c['id']}"

    def run(mode):
        G = Guarded(dev, seed + 20)
        dx = G.add("dx", (P, D), "nan")
        dw = G.add("dw", (D, 27), "rand", 0.1)
        db = G.add("db", (D,), "rand", 0.1)
        sync()
        L.check(lib.probe_peg_backward(_p(x), _p(w27), _p(dy), _p(dx), _p(dw), _p(db), P, T, H, Wd_, D, pad_t0,
                                       L.stream_ptr()), "probe_peg_backward")
        sync()
        G.check(f"{name} ({mode})")
        return {"dx": dx.clone(), "dw": dw.clone(), "db": db.clone(), "_G": G}

    det = max(_sizes(lib, dim=D)[2], -(-P // 256) * D)
    for mode, out in _modes(lib, dev, det, run, sync):
        G = out.pop("_G")
        nm = f"{name} ({mode})"
        _within(f"{nm} dx", out["dx"], ref[0].reshape(P, D), 28 * U * (dy.double().abs() + mag_dx).reshape(P, D),
                {k: v[0].reshape(P, D) for k, v in alts.items()})
        pw, pb = G.pre("dw"), G.pre("db")
        _within(f"{nm} dw", out["dw"], ref[1] + pw, (P + 17) * U * (mag_dw + pw.abs()),
                {k: v[1] + pw for k, v in alts.items()})
        _within(f"{nm} db", out["db"], ref[2] + pb, (P + 65) * U * (dy.double().abs().sum((0, 1)) + pb.abs()))


def check_peg_refused(lib, dev, sync):
    """D = 1025: PHK_E_UNSUPPORTED before anything is written or launched"""
    B, T, H, W, D = 1, 2, 3, 3, 1025
    P = B * T * H * W
    x, dy = _randn((P, D), 1, dev), _randn((P, D), 2, dev)
    w27 = _randn((27, D), 3, dev)
    G = Guarded(dev, 40)
    dx, dw, db = G.add("dx", (P, D), "nan"), G.add("dw", (D, 27), "rand"), G.add("db", (D,), "rand")
    sync()
    before = lib.phk_launch_count()
    rc = lib.probe_peg_backward(_p(x), _p(w27), _p(dy), _p(dx), _p(dw), _p(db), P, T, H, W, D, 1, L.stream_ptr())
    sync()
    assert rc == E_UNSUPPORTED, f"peg D = 1025 accepted (rc {rc})"
    assert lib.phk_launch_count() == before, "peg D = 1025: a refused call launched kernels"
    G.untouched("peg D = 1025")


# ---------------------------------------------------------------------------------------------------------------------
# H. embeddings: embed_backward (embed_bwd_kernel | embed_tok_fixed_kernel + embed_pos_fixed_kernel)
# ---------------------------------------------------------------------------------------------------------------------
def _embed_ref(ids, dx, vocab, n, D, alpha, pos_of_row=None):
    """float64 autograd of x = alpha (tok[clamp(ids)] + pos[row % n]) (the shrink trick's gradient path)"""
    tok = torch.zeros((vocab, D), dtype=torch.float64, device=dx.device, requires_grad=True)
    pos = torch.zeros((n, D), dtype=torch.float64, device=dx.device, requires_grad=True)
    rows = ids.numel()
    p = pos_of_row if pos_of_row is not None else torch.arange(rows, device=dx.device) % n
    keep = p < n
    xt = alpha * tok[ids.clamp(0, vocab - 1)]
    xp = alpha * pos[p[keep]]
    ((xt * dx.double()).sum() + (xp * dx.double()[keep]).sum()).backward()
    return tok.grad, pos.grad


def check_embed(lib, dev, c, sync):
    """c: b, n, D, vocab (table rows), ids ('random' | 'mask' | 'clamp'), alpha, seed"""
    b, n, D, vocab, alpha, seed = c["b"], c["n"], c["D"], c["vocab"], c["alpha"], c["seed"]
    rows = b * n
    gen = _g(seed)
    if c["ids"] == "mask":  # every row the mask id (the table's last row)
        ids = torch.full((rows,), vocab - 1, dtype=torch.int64)
    else:
        ids = torch.randint(0, vocab, (rows,), generator=gen)
        if c["ids"] == "clamp":  # -1 and >= vocab: the forward's clamp
            sel = torch.rand((rows,), generator=gen)
            ids = torch.where(sel < 0.2, torch.full_like(ids, -1), ids)
            ids = torch.where(sel > 0.8, vocab + torch.randint(0, 5, (rows,), generator=gen), ids)
    ids = ids.to(dev)
    dx = _randn((rows, D), seed + 1, dev)
    ref_tok, ref_pos = _embed_ref(ids, dx, vocab, n, D, alpha)
    alt_tok, alt_pos = _embed_ref(ids, dx, vocab, n, D, 1.0)
    _, row_pos = _embed_ref(ids, dx, vocab, n, D, alpha, pos_of_row=torch.arange(rows, device=dev))
    cnt = torch.zeros((vocab,), dtype=torch.float64, device=dev).index_add_(
        0, ids.clamp(0, vocab - 1), torch.ones(rows, dtype=torch.float64, device=dev))
    mag_tok = torch.zeros((vocab, D), dtype=torch.float64, device=dev).index_add_(
        0, ids.clamp(0, vocab - 1), (alpha * dx.double()).abs())
    mag_pos = (alpha * dx.double()).abs().view(b, n, D).sum(0)
    name = f"embed {c['id']}"

    def run(mode):
        G = Guarded(dev, seed + 30)
        dtok = G.add("dtok", (vocab, D), "rand", 0.1)
        dpos = G.add("dpos", (n, D), "rand", 0.1)
        sync()
        L.check(lib.probe_embed_backward(_p(ids), _p(dx), _p(dtok), _p(dpos), rows, n, D, alpha, vocab,
                                         L.stream_ptr()), "probe_embed_backward")
        sync()
        G.check(f"{name} ({mode})")
        return {"dtok": dtok.clone(), "dpos": dpos.clone(), "_G": G}

    for mode, out in _modes(lib, dev, 1, run, sync):
        G = out.pop("_G")
        nm = f"{name} ({mode})"
        pt, pp = G.pre("dtok"), G.pre("dpos")
        _within(f"{nm} dtok", out["dtok"], ref_tok + pt, (cnt[:, None] + 3) * U * (mag_tok + pt.abs()),
                {"alpha not applied": alt_tok + pt})
        _within(f"{nm} dpos", out["dpos"], ref_pos + pp, (b + 3) * U * (mag_pos + pp.abs()),
                {"alpha not applied": alt_pos + pp, "position = row": row_pos + pp} if b > 1 else
                {"alpha not applied": alt_pos + pp})


# ---------------------------------------------------------------------------------------------------------------------
# I. position-bias MLP: cpb_backward (cpb_inputs_kernel, bias_lrelu_kernel, cpb_dtable_kernel | cpb_dtable_fixed_kernel,
#    lrelu_bwd_kernel and the fp32 products)
# ---------------------------------------------------------------------------------------------------------------------
_CPB_KEYS = ("w0", "b0", "w1", "b1", "w2", "b2")


def _cpb_sd(P):
    return {"net.0.0.weight": P["w0"], "net.0.0.bias": P["b0"], "net.1.0.weight": P["w1"], "net.1.0.bias": P["b1"],
            "net.2.weight": P["w2"], "net.2.bias": P["b2"]}


def _cpb_slipped(P, dims, slope=0.1, signed=True):
    """an own statement of the MLP with the slips: the leaky slope, sign(delta) dropped"""
    pos = [torch.arange(d, device=P["w0"].device) for d in dims]
    grid = torch.stack(torch.meshgrid(*pos, indexing="ij")).reshape(len(dims), -1).t()
    rel = (grid[:, None, :] - grid[None, :, :]).to(P["w0"].dtype)
    h = torch.log(rel.abs() + 1)
    if signed:
        h = torch.sign(rel) * h
    h = F.leaky_relu(F.linear(h, P["w0"], P["b0"]), slope)
    h = F.leaky_relu(F.linear(h, P["w1"], P["b1"]), slope)
    return F.linear(h, P["w2"], P["b2"]).permute(2, 0, 1)


def _cpb_grads(params, dbias, dims, fn):
    P = {k: v.double().requires_grad_() for k, v in params.items()}
    (fn(P) * dbias.double()).sum().backward()
    return {k: P[k].grad for k in _CPB_KEYS}


def _cpb_bars(params, dbias, dims, nd, hid, H):
    """the running-error bound of the module docstring, on the U distinct deltas"""
    dev = dbias.device
    d3 = list(dims) + [1] * (3 - len(dims))
    s = [2 * d - 1 for d in d3]
    Un = s[0] * s[1] * s[2]
    u = torch.arange(Un, device=dev)
    delta = torch.stack((u // (s[1] * s[2]) - (d3[0] - 1), (u // s[2]) % s[1] - (d3[1] - 1), u % s[2] - (d3[2] - 1)), 1)
    delta = delta[:, :nd].double()
    inp = torch.sign(delta) * torch.log(delta.abs() + 1)
    e_in = 2 * U * inp.abs()  # logf's 1 ulp, the product with the sign and the conversion exact
    W0, b0, W1, b1, W2, b2 = (params[k].double() for k in _CPB_KEYS)
    z1 = inp @ W0.t() + b0
    a1 = F.leaky_relu(z1, 0.1)
    e_z1 = (nd + 2) * U * (inp.abs() @ W0.abs().t() + b0.abs()) + e_in @ W0.abs().t()
    e_a1 = e_z1 + U * a1.abs()
    z2 = a1 @ W1.t() + b1
    a2 = F.leaky_relu(z2, 0.1)
    e_z2 = (hid + 2) * U * (a1.abs() @ W1.abs().t() + b1.abs()) + e_a1 @ W1.abs().t()
    e_a2 = e_z2 + U * a2.abs()
    # dtable[u, h]: the pairs (i, j) with delta u, i = (i0, i1, i2) over the grid d3
    n = d3[0] * d3[1] * d3[2]
    gi = torch.stack(torch.meshgrid(*[torch.arange(d, device=dev) for d in d3], indexing="ij")).reshape(3, -1).t()
    rel = gi[:, None, :] - gi[None, :, :]
    uid = ((rel[..., 0] + d3[0] - 1) * s[1] + rel[..., 1] + d3[1] - 1) * s[2] + rel[..., 2] + d3[2] - 1
    db = dbias.double().reshape(H, n * n)
    dt = torch.zeros((Un, H), dtype=torch.float64, device=dev).index_add_(0, uid.reshape(-1), db.t())
    dt_abs = torch.zeros((Un, H), dtype=torch.float64, device=dev).index_add_(0, uid.reshape(-1), db.abs().t())
    cnt = torch.zeros((Un,), dtype=torch.float64, device=dev).index_add_(
        0, uid.reshape(-1), torch.ones(n * n, dtype=torch.float64, device=dev))
    e_dt = (cnt[:, None] + 1) * U * dt_abs
    adds = Un // 256 + 3  # split-K slices / slots of the wgrad, the prefill
    sum_k = Un + adds

    def layer(dout, e_dout, act, e_act):
        """bars of one Linear's weight and bias gradients from d/d(its output) and its input, with their bounds"""
        bar_w = sum_k * U * (dout.abs().t() @ act.abs()) + e_dout.t() @ act.abs() + dout.abs().t() @ e_act
        bar_b = (Un + 65) * U * dout.abs().sum(0) + e_dout.sum(0)
        return bar_w, bar_b

    bars = {}
    bars["w2"], bars["b2"] = layer(dt, e_dt, a2, e_a2)
    g2 = dt @ W2  # d/d a2
    e_g2 = (H + 1) * U * (dt.abs() @ W2.abs()) + e_dt @ W2.abs()
    s2 = torch.where(z2 > 0, 1.0, 0.1).double()
    amb2 = (z2.abs() <= e_z2).double()
    da2 = g2 * s2
    e_da2 = e_g2 * torch.maximum(s2, amb2) + U * da2.abs() + 0.9 * amb2 * g2.abs()
    bars["w1"], bars["b1"] = layer(da2, e_da2, a1, e_a1)
    g1 = da2 @ W1
    e_g1 = (hid + 1) * U * (da2.abs() @ W1.abs()) + e_da2 @ W1.abs()
    s1 = torch.where(z1 > 0, 1.0, 0.1).double()
    amb1 = (z1.abs() <= e_z1).double()
    da1 = g1 * s1
    e_da1 = e_g1 * torch.maximum(s1, amb1) + U * da1.abs() + 0.9 * amb1 * g1.abs()
    bars["w0"], bars["b0"] = layer(da1, e_da1, inp, e_in)
    return bars, int(amb1.sum() + amb2.sum())


def cpb_params(nd, hid, H, seed, dev):
    return {"w0": _randn((hid, nd), seed, dev, 1.0), "b0": _randn((hid,), seed + 1, dev, 0.5),
            "w1": _randn((hid, hid), seed + 2, dev, hid ** -0.5), "b1": _randn((hid,), seed + 3, dev, 0.5),
            "w2": _randn((H, hid), seed + 4, dev, hid ** -0.5), "b2": _randn((H,), seed + 5, dev, 0.5)}


def _cpb_t(P, nd, hid, H):
    t = L.CpbT()
    for k in _CPB_KEYS:
        setattr(t, k, _p(P[k]))
    t.num_dims, t.hidden, t.heads = nd, hid, H
    return t


def check_cpb(lib, dev, c, sync):
    """c: dims (2 or 3 entries), hidden, heads, seed"""
    dims, hid, H, seed = tuple(c["dims"]), c["hidden"], c["heads"], c["seed"]
    nd = len(dims)
    d3 = list(dims) + [1] * (3 - nd)
    n = d3[0] * d3[1] * d3[2]
    params = cpb_params(nd, hid, H, seed, dev)
    dbias = _randn((H, n, n), seed + 9, dev)
    ref = _cpb_grads(params, dbias, dims, lambda P: O.continuous_position_bias(_cpb_sd(P), "", dims))
    alts = {"slope 0.01": _cpb_grads(params, dbias, dims, lambda P: _cpb_slipped(P, dims, slope=0.01)),
            "sign(delta) dropped": _cpb_grads(params, dbias, dims, lambda P: _cpb_slipped(P, dims, signed=False))}
    bars, amb = _cpb_bars(params, dbias, dims, nd, hid, H)
    ct = _cpb_t(params, nd, hid, H)
    scratch_floats = _sizes(lib, ct, d3)[0]
    Un = (2 * d3[0] - 1) * (2 * d3[1] - 1) * (2 * d3[2] - 1)
    name = f"cpb {c['id']}"
    print(f"[train-backward] {name}: U = {Un}, {amb} pre-activations within their error bound of 0")

    def run(mode):
        G = Guarded(dev, seed + 50)
        g = {k: G.add(k, params[k].shape, "rand", 0.01) for k in _CPB_KEYS}
        gt = _cpb_t(g, nd, hid, H)
        scratch = torch.full((scratch_floats,), NAN, device=dev)
        sync()
        L.check(lib.probe_cpb_backward(C.byref(ct), C.byref(gt), _p(dbias), d3[0], d3[1], d3[2], _p(scratch),
                                       L.stream_ptr()), "probe_cpb_backward")
        sync()
        G.check(f"{name} ({mode})")
        out = {k: v.clone() for k, v in g.items()}
        out["_G"] = G
        return out

    det = (Un // 256 + 2) * (hid * max(H, nd, 64) + 64)
    for mode, out in _modes(lib, dev, det, run, sync):
        G = out.pop("_G")
        for k in _CPB_KEYS:
            pre = G.pre(k)
            # U = 1: the only delta is 0, whose input row is 0 and whose sign cannot slip
            al = {lab: a[k] + pre for lab, a in alts.items()} if k in ("w0", "b0", "w1", "b1") and Un > 1 else None
            _within(f"{name} ({mode}) d{k}", out[k], ref[k] + pre, bars[k] + U * pre.abs(), al)


# ---------------------------------------------------------------------------------------------------------------------
# J. head losses: ce_rows (mask_count_kernel, ce_rows_kernel), bce_rows, loss_reduce
# ---------------------------------------------------------------------------------------------------------------------
def check_ce(lib, dev, c, sync):
    """c: rows, V, mask ('partial' | 'all' | 'none'), scale, seed.  Logits spread +-80; row 0's target holds a logit 40
    above the rest (its probability rounds to 1 in fp32)."""
    rows, V, scale, seed = c["rows"], c["V"], c["scale"], c["seed"]
    gen = _g(seed)
    logits = (torch.rand((rows, V), generator=gen) * 160.0 - 80.0)
    targets = torch.randint(0, V, (rows,), generator=gen)
    logits[0, targets[0]] = logits[0].max() + 40.0
    mask = {"partial": torch.rand((rows,), generator=gen) < 0.4, "all": torch.ones(rows, dtype=torch.bool),
            "none": torch.zeros(rows, dtype=torch.bool)}[c["mask"]]
    if c["mask"] == "partial":
        mask[0] = True
        mask[-1] = False
    logits, targets, mask_u8 = logits.to(dev), targets.to(dev), mask.to(torch.uint8).to(dev)
    mask = mask.to(dev)
    name = f"ce {c['id']}"
    G = Guarded(dev, seed + 60)
    dl = G.add("dlogits", (rows, V), "nan")
    dl.copy_(logits)  # overwritten in place
    count = G.add("count", (1,), "nan")
    row_loss = G.add("row_loss", (rows,), "nan")
    loss = G.add("loss", (1,), "nan")
    sync()
    L.check(lib.probe_ce_rows(_p(dl), _p(targets), _p(mask_u8), _p(count), scale, _p(row_loss), rows, V,
                              L.stream_ptr()), "probe_ce_rows")
    L.check(lib.probe_loss_reduce(_p(row_loss), rows, _p(loss), L.stream_ptr()), "probe_loss_reduce")
    sync()
    G.check(name)
    nm = int(mask.sum())
    if nm == 0:  # all-false mask: the count clamps at 1, loss 0 and zero gradients (the reference would give NaN)
        assert float(count) == 1.0, f"{name}: count {float(count)}"
        assert _same_bits(dl, torch.zeros_like(dl)) and _same_bits(row_loss, torch.zeros_like(row_loss)), \
            f"{name}: an all-false mask left nonzero dlogits or row losses"
        assert float(loss) == 0.0, f"{name}: loss {float(loss)} for an all-false mask"
        print(f"[train-backward] {name}: all-false mask gives loss 0 and zero gradients")
        return
    assert float(count) == nm, f"{name}: count {float(count)} for {nm} masked rows"
    ld = logits.double().requires_grad_()
    ce = F.cross_entropy(ld[mask], targets[mask], reduction="none")
    (ce.mean() * scale).backward()
    ref_dl = ld.grad
    ref_rows = torch.zeros(rows, dtype=torch.float64, device=dev)
    ref_rows[mask] = ce.detach() / nm
    # bars
    lg = logits.double()
    mx = lg.max(-1, keepdim=True).values
    p = torch.softmax(lg, -1)
    depth = -(-V // 256) + 10
    wavg = (p * (lg - mx).abs()).sum(-1, keepdim=True)
    e_s = (2 + depth + wavg) * U  # relative error of the exp-sum
    onehot = F.one_hot(targets, V).double()
    k = abs(scale) / nm
    bar_dl = k * (p * ((lg - mx).abs() + 6 + depth + wavg) * U + 3 * U * (p - onehot).abs() + 2.0 ** -126)
    bar_dl = bar_dl * mask[:, None]
    ls = torch.log(torch.exp(lg - mx).sum(-1))
    tl = lg.gather(1, targets[:, None])[:, 0]
    lse = mx[:, 0] + ls
    bar_rows = (e_s[:, 0] + U * ls.abs() + U * lse.abs() + 2 * U * (lse - tl).abs()) / nm * mask
    _within(f"{name} dlogits", dl, ref_dl, bar_dl, {"divided by all rows": ref_dl * nm / rows} if nm < rows else None)
    _within(f"{name} row loss", row_loss, ref_rows, bar_rows)
    bar_loss = (-(-rows // 1024) + 10) * U * ref_rows.abs().sum() + bar_rows.sum()
    _within(f"{name} loss", loss, ce.detach().mean().reshape(1), bar_loss.reshape(1))


def check_bce(lib, dev, c, sync):
    """c: rows, D, scale, seed; scores spread to |score| ~ 100, labels 0 / 1"""
    rows, D, scale, seed = c["rows"], c["D"], c["scale"], c["seed"]
    gen = _g(seed)
    emb = torch.randn((rows, D), generator=gen)
    w = torch.randn((D,), generator=gen) * (1.0 / math.sqrt(D))
    target = torch.linspace(-100.0, 100.0, rows)  # each row moved along w so that its score is near its target
    emb = emb + ((target - emb @ w) / (w @ w))[:, None] * w
    b = torch.tensor([0.25])
    labels = (torch.rand((rows,), generator=gen) < 0.5).float()
    emb, w, b, labels = emb.to(dev), w.to(dev), b.to(dev), labels.to(dev)
    name = f"bce {c['id']}"
    G = Guarded(dev, seed + 70)
    row_loss = G.add("row_loss", (rows,), "nan")
    dscore = G.add("dscore", (rows,), "nan")
    loss = G.add("loss", (1,), "nan")
    sync()
    L.check(lib.probe_bce_rows(_p(emb), _p(w), _p(b), _p(labels), scale, _p(row_loss), _p(dscore), rows, D,
                               L.stream_ptr()), "probe_bce_rows")
    L.check(lib.probe_loss_reduce(_p(row_loss), rows, _p(loss), L.stream_ptr()), "probe_loss_reduce")
    sync()
    G.check(name)
    a = (emb.double() @ w.double() + b.double()).requires_grad_()
    y = labels.double()
    lrows = F.binary_cross_entropy_with_logits(a, y, reduction="none")
    (lrows.mean() * scale).backward()
    ref_ds = a.grad
    ad = a.detach()
    ea = (-(-D // 32) + 6) * U * (emb.double().abs() @ w.double().abs() + b.double().abs())
    sg = torch.sigmoid(ad)
    kk = abs(scale) / rows
    bar_ds = kk * (sg * (1 - sg) * ea + sg * ((1 - sg) * (2 + ad.abs()) + 3) * U + 3 * U * (sg - y).abs() + 2.0 ** -126)
    alt = (torch.sigmoid(-ad) - y) * scale / rows
    _within(f"{name} dscore", dscore, ref_ds, bar_ds, {"sigmoid(-a)": alt})
    ref_rows = lrows.detach() / rows
    e = torch.exp(-ad.abs())
    bar_rows = (ea + (2 + ad.abs()) * U * e + U * (ad.clamp_min(0) + (ad * y).abs() + 3 * lrows.detach())) / rows
    _within(f"{name} row loss", row_loss, ref_rows, bar_rows)
    bar_loss = (-(-rows // 1024) + 10) * U * ref_rows.abs().sum() + bar_rows.sum()
    _within(f"{name} loss", loss, lrows.detach().mean().reshape(1), bar_loss.reshape(1))
