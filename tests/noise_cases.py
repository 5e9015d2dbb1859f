"""Shared bodies of the in-kernel noise checks (CPU executor and GPU): phk_sample_tokens with u == NULL, the fused head and
the masked-rows tail against the fp64 gumbel-max reference of tests/noise_ref.py.

How a case is judged.  Every perturbed logit y = l / T + g the device computes differs from the fp64 reference by at most
    err = dl / T                (the error of l itself, per kernel: see each body)
        + 2^-22 |l / T|         (fp32 rounding of 1 / max(T, 1e-10) and of the final fma)
        + gumbel_err(u)         (lg2.approx, fp32 constants; noise_ref.gumbel_err)
and a row's argmax is DECIDED when the reference winner beats every other column by more than the two columns' bounds
(noise_ref.decided).  Decided rows must carry the reference id exactly; the undecided rows must stay a small fraction,
so a case cannot pass by being undecidable.  The fraction grows with V because lg2.approx's documented error near 1 is
absolute (2^-22): the winning draw of a V-wide row has 1 - u ~ 1 / V, hence an error up to ~V 2^-22 in g.
Scores: 1 - p with p = softmax(l)[pred]; |dp| <= p (2 max|dl| + (V / 8 + 64) 2^-24 + 1e-5) + 1e-6: the logits' error
enters p twice (numerator and the sum), the fp32 sum of exponentials is at most V / 8 + 64 additions deep in either
kernel, and the exp approximations (__expf / ex2.approx) add a few ulp."""
import numpy as np
import torch

from phenaki_pytorch_b200 import _lib as L
from tests import noise_ref as R

SENTINEL_ID, SENTINEL_SCORE = -77, 12345.0


def undecided_cap(V):
    """Largest tolerated fraction of undecided rows: 1 % up to V = 8192 (measured ~0.5 % there with the bound above),
    8 % at V = 65536 (~3.5 %); judge() always tolerates 2 rows, for the cases with few rows."""
    return 0.01 if V <= 8192 else 0.08


def judge(what, s, l, T, dl, pred, score=None, V=None):
    """Compares device ids (pred) / scores with the reference Sample s of logits l (fp64) under the error dl of l."""
    V = l.shape[1] if V is None else V
    Tc = max(float(T), 1e-10)
    err = dl / Tc + 2.0 ** -22 * np.abs(l / Tc) + R.gumbel_err(s.u)
    ok = R.decided(s.y, err, s.pred)
    frac = 1.0 - ok.mean()
    assert (~ok).sum() <= max(2, undecided_cap(V) * ok.size), f"{what}: {frac:.4f} of the rows are within the error bound of a tie"
    bad = np.nonzero(ok & (pred != s.pred))[0]
    assert bad.size == 0, (f"{what}: {bad.size} of {int(ok.sum())} decided rows differ, first row {bad[0]}: "
                           f"got {pred[bad[0]]}, reference {s.pred[bad[0]]} (gap {s.gap[bad[0]]:.3g})")
    if score is not None:
        same = pred == s.pred
        p = 1.0 - s.score
        dlm = np.max(np.broadcast_to(dl, l.shape), axis=1)
        tol = p * (2 * dlm + (V / 8 + 64) * 2.0 ** -24 + 1e-5) + 1e-6
        d = np.abs(score - s.score)
        worst = np.argmax(np.where(same, d - tol, -np.inf))
        assert not same.any() or d[worst] <= tol[worst], (f"{what}: score of row {worst} off by {d[worst]:.3g} "
                                                          f"(tolerance {tol[worst]:.3g})")
    return frac


def _np(t):
    return t.detach().cpu().double().numpy()


# ---- phk_sample_tokens with in-kernel noise -------------------------------------------------------------------------

def check_sample_tokens(lib, dev, *, rows, V, T, seed, offset, ld=None, scale=1.0, seg=None, data_seed=0,
                        sync=lambda: None):
    """rows token rows of V logits (leading dimension ld), optional CFG pair (scale != 1: l = null + (cond - null) s in
    fp64 from the fp32 inputs; the kernel's fp32 sub / mul / add is off by <= 2^-22 (|cond - null| |s| + |null| + |l|))
    and optional seg = (seg_len, seg_stride, seg_off) row map: token row r reads logits row
    (r / seg_len) seg_stride + seg_off + r % seg_len, while its noise counter row stays r."""
    ld = V if ld is None else ld
    g = torch.Generator().manual_seed(data_seed)
    seg_len, seg_stride, seg_off = seg or (0, 0, 0)
    r = np.arange(rows)
    lrow = (r // seg_len) * seg_stride + seg_off + r % seg_len if seg_len > 0 else r
    lrows = int(lrow.max()) + 1
    cond = torch.randn((lrows, ld), generator=g) * 2.0
    null = torch.randn((lrows, ld), generator=g) * 2.0 if scale != 1.0 else None
    cond[:, V:] = float("nan")  # the padding of each row is never read
    if null is not None:
        null[:, V:] = float("nan")
    c = _np(cond)[lrow, :V]
    if null is None:
        l, dl = c, np.zeros(1)
    else:
        n = _np(null)[lrow, :V]
        l = n + (c - n) * scale
        dl = 2.0 ** -22 * (np.abs(c - n) * abs(scale) + np.abs(n) + np.abs(l))
    mask = (torch.rand(rows, generator=g) < 0.7).to(torch.uint8)
    ids0 = torch.randint(0, max(V, 2), (rows,), generator=g)
    ids = torch.cat((ids0, torch.full((4,), SENTINEL_ID))).to(dev)
    pred = torch.full((rows + 4,), SENTINEL_ID, dtype=torch.int64, device=dev)
    score = torch.full((rows + 4,), SENTINEL_SCORE, device=dev)
    condd = cond.to(dev)
    nulld = null.to(dev) if null is not None else None
    L.check(lib.phk_sample_tokens(L.ptr(condd), L.ptr(nulld), ld, None, seed, offset, scale, T, L.ptr(mask.to(dev)),
                                  L.ptr(ids), L.ptr(pred), L.ptr(score), rows, V, seg_len, seg_stride, seg_off,
                                  L.stream_ptr()), "phk_sample_tokens")
    sync()
    ids, pred, score = ids.cpu(), pred.cpu(), score.cpu()
    assert bool((ids[rows:] == SENTINEL_ID).all() & (pred[rows:] == SENTINEL_ID).all() & (score[rows:] == SENTINEL_SCORE).all())
    s = R.gumbel_max(l, T, seed, offset)
    pr = pred[:rows].numpy()
    m = mask.bool().numpy()
    sc = score[:rows].double().numpy()
    assert np.array_equal(ids[:rows].numpy(), np.where(m, pr, ids0.numpy()))
    assert bool((sc[~m] == -1e4).all())
    # unmasked rows carry -1e4 (checked above), not a confidence
    return judge(f"sample_tokens V={V} T={T}", s, l, T, dl, pr, np.where(m, sc, s.score))


# ---- phk_head_sample / phk_head_sample_rng ------------------------------------------------------------------------

def head_inputs(n_tokens, V, dim, *, emb_rows=None, ld_emb=None, ldw=None, data_seed=0):
    """bf16 emb [emb_rows, ld_emb] / W [V, ldw] with NaN in every element the head must not read (rows past n_tokens,
    padding columns), fp32 bias; the fp64 logits and their error bound: the device sums dim exact bf16 products in fp32
    (wgmma), off by <= dim 2^-23 sum_k |e_k w_k| (twice the round-to-nearest bound, so a truncating accumulator is
    covered too), plus 2^-24 |l| for the bias add."""
    emb_rows = n_tokens if emb_rows is None else emb_rows
    ld_emb = dim if ld_emb is None else ld_emb
    ldw = dim if ldw is None else ldw
    g = torch.Generator().manual_seed(data_seed)
    emb = torch.full((emb_rows, ld_emb), float("nan"))
    emb[:n_tokens, :dim] = torch.randn((n_tokens, dim), generator=g)
    W = torch.full((V, ldw), float("nan"))
    W[:, :dim] = torch.randn((V, dim), generator=g) / dim ** 0.5
    emb, W = emb.bfloat16(), W.bfloat16()
    bias = torch.randn((V,), generator=g) * 0.5
    e, w = _np(emb[:n_tokens, :dim].float()), _np(W[:, :dim].float())
    l = e @ w.T + _np(bias)[None, :]
    dl = dim * 2.0 ** -23 * (np.abs(e) @ np.abs(w).T) + 2.0 ** -24 * np.abs(l)
    return emb, W, bias, l, dl


def run_head(lib, dev, emb, W, bias, *, n_tokens, V, dim, T, seed, offset, mask=None, ids0=None, rng=None,
             drop=(), sync=lambda: None):
    """One phk_head_sample(_rng) call with outputs that extend 5 sentinel entries past n_tokens; `drop` names the optional
    pointers passed as NULL (bias, mask, ids, pred, score).  Returns the outputs (CPU), sentinels checked."""
    pad = 5
    ids = torch.full((n_tokens + pad,), SENTINEL_ID, dtype=torch.int64)
    if ids0 is not None:
        ids[:n_tokens] = ids0
    ids = ids.to(dev)
    pred = torch.full((n_tokens + pad,), SENTINEL_ID, dtype=torch.int64, device=dev)
    score = torch.full((n_tokens + pad,), SENTINEL_SCORE, device=dev)
    embd, Wd = emb.to(dev), W.to(dev)
    biasd = None if "bias" in drop else bias.to(dev)
    maskd = None if ("mask" in drop or mask is None) else mask.to(dev)
    nb = int(lib.phk_head_sample_scratch_bytes(n_tokens))
    scratch = torch.full((nb,), 0xFF, dtype=torch.uint8, device=dev)
    args = (L.ptr(embd), emb.shape[1], emb.shape[0], L.ptr(Wd), W.shape[1], L.ptr(biasd), n_tokens, V, dim, T, seed, offset)
    outs = (None if "ids" in drop else L.ptr(ids), None if "pred" in drop else L.ptr(pred),
            None if "score" in drop else L.ptr(score), L.ptr(scratch), nb, L.stream_ptr())
    if rng is None:
        L.check(lib.phk_head_sample(*args, L.ptr(maskd), *outs), "phk_head_sample")
    else:
        L.check(lib.phk_head_sample_rng(*args, L.ptr(rng), L.ptr(maskd), *outs), "phk_head_sample_rng")
    sync()
    ids, pred, score = ids.cpu(), pred.cpu(), score.cpu()
    assert bool((ids[n_tokens:] == SENTINEL_ID).all()), "ids written past n_tokens"
    assert bool((pred[n_tokens:] == SENTINEL_ID).all()), "pred_out written past n_tokens"
    assert bool((score[n_tokens:] == SENTINEL_SCORE).all()), "score_out written past n_tokens"
    return ids[:n_tokens].numpy(), pred[:n_tokens].numpy(), score[:n_tokens].double().numpy()


def check_head(lib, dev, *, n_tokens, V, dim, T, seed, offset, emb_rows=None, ld_emb=None, ldw=None, drop=(),
               data_seed=0, sync=lambda: None):
    emb, W, bias, l, dl = head_inputs(n_tokens, V, dim, emb_rows=emb_rows, ld_emb=ld_emb, ldw=ldw, data_seed=data_seed)
    if "bias" in drop:
        l = l - _np(bias)[None, :]
    g = torch.Generator().manual_seed(data_seed + 1)
    mask = (torch.rand(n_tokens, generator=g) < 0.6).to(torch.uint8)
    ids0 = torch.randint(0, V, (n_tokens,), generator=g)
    ids, pred, score = run_head(lib, dev, emb, W, bias, n_tokens=n_tokens, V=V, dim=dim, T=T, seed=seed, offset=offset,
                                mask=mask, ids0=ids0, drop=drop, sync=sync)
    s = R.gumbel_max(l, T, seed, offset)
    m = np.ones(n_tokens, dtype=bool) if "mask" in drop else mask.bool().numpy()
    what = f"head n={n_tokens} V={V} dim={dim} T={T} NULL={drop}"
    if "pred" in drop:
        pred = np.where(m, ids, s.pred)  # the ids of the masked rows are the only prediction left to check
    if "ids" not in drop:
        assert np.array_equal(ids, np.where(m, pred, ids0.numpy())), f"{what}: ids != where(mask, pred, ids)"
    if "score" in drop:
        return judge(what, s, l, T, dl, pred)
    assert bool((score[~m] == -1e4).all())
    return judge(what, s, l, T, dl, pred, np.where(m, score, s.score))


# ---- phk_sample_tail(_rows) at T > 0 -------------------------------------------------------------------------------

def check_tail(lib, dev, *, b, n, k, V, dim, T, seed, offset, counts=None, plen=0, data_seed=0, sync=lambda: None):
    """b sequences of n sampled tokens (behind a prime prefix of plen rows of the residual stream), counts[i] <= k masked
    positions each (default k).  Reference: the masked positions of sequence i in increasing order are compact rows
    i k + j, whose noise counter row is that compact index; padding rows (j >= counts[i]) use up counters and scatter
    nothing.  The embedding e = s norm(x_cond) + (1 - s) norm(x_null) is taken in fp64 without the device's bf16
    rounding, which moves a logit by <= 2^-8 sum_k |e_k w_k| (one bf16 rounding, 2^-9 relative, doubled for the fp32
    LayerNorm), on top of the fp32 accumulation bound of head_inputs; W is scaled so that the noise decides most rows."""
    counts = [k] * b if counts is None else counts
    g = torch.Generator().manual_seed(data_seed)
    src = plen + n
    xc = torch.randn((b * src, dim), generator=g) * 2 + 0.3
    xn = torch.randn((b * src, dim), generator=g) * 2 - 0.1
    gamma, beta = torch.randn((dim,), generator=g), torch.randn((dim,), generator=g) * 0.1
    W = (torch.randn((V, dim), generator=g) * (0.03 / dim ** 0.5)).bfloat16()
    bias = torch.randn((V,), generator=g) * 0.3
    mask = torch.zeros((b, n), dtype=torch.uint8)
    for i in range(b):
        mask[i, torch.randperm(n, generator=g)[:counts[i]]] = 1
    ids0 = torch.randint(0, V, (b, n), generator=g)
    scale = 3.0
    x64c, x64n = xc.double(), xn.double()
    ln = lambda x: torch.nn.functional.layer_norm(x, (dim,), gamma.double(), beta.double(), eps=1e-5)
    e = (scale * ln(x64c) + (1 - scale) * ln(x64n)).numpy()
    w = _np(W.float())
    # compact rows: (sequence, rank among its masked positions) -> residual row, padding rows -> -1
    comp = np.full(b * k, -1)
    tok = np.full(b * k, -1)
    for i in range(b):
        pos = np.nonzero(mask[i].numpy())[0]
        comp[i * k:i * k + len(pos)] = i * src + plen + pos
        tok[i * k:i * k + len(pos)] = i * n + pos
    live = comp >= 0
    er = e[comp[live]]
    l = er @ w.T + _np(bias)[None, :]
    dl = (2.0 ** -8 + dim * 2.0 ** -23) * (np.abs(er) @ np.abs(w).T) + 2.0 ** -24 * np.abs(l)
    s = R.gumbel_max(l, T, seed, offset, row_ids=np.nonzero(live)[0])
    ids = ids0.clone().to(dev)
    pred = torch.empty((b, n), dtype=torch.int64, device=dev)
    score = torch.empty((b, n), device=dev)
    nb = int(lib.phk_sample_tail_scratch_bytes(b, k, dim))
    scratch = torch.full((nb,), 0xFF, dtype=torch.uint8, device=dev)
    t = [x.to(dev) for x in (xc, xn, gamma, beta, W, bias, mask)]
    L.check(lib.phk_sample_tail_rows(L.ptr(t[0]), L.ptr(t[1]), L.ptr(t[2]), L.ptr(t[3]), scale, L.ptr(t[4]), dim,
                                     L.ptr(t[5]), b, n, k, V, dim, T, seed, offset, None, L.ptr(t[6]), L.ptr(ids),
                                     L.ptr(pred), L.ptr(score), src, plen, L.ptr(scratch), nb, L.stream_ptr()),
            "phk_sample_tail_rows")
    sync()
    ids, pred, score = ids.cpu().reshape(-1).numpy(), pred.cpu().reshape(-1).numpy(), score.cpu().reshape(-1).numpy()
    m = mask.reshape(-1).bool().numpy()
    assert np.array_equal(ids[~m], ids0.reshape(-1).numpy()[~m]) and bool((score[~m] == -1e4).all())
    assert np.array_equal(pred[m], ids[m])
    t_live = tok[live]
    return judge(f"tail b={b} n={n} k={k} counts={counts} plen={plen} T={T}", s, l, T, dl, ids[t_live],
                 score[t_live].astype(np.float64))


# ---- chi-square helpers of the distribution tests --------------------------------------------------------------------

P_FLOOR = 1e-6


def chi2_pvalue(counts, probs):
    from scipy.stats import chi2
    counts, probs = np.asarray(counts, dtype=np.float64), np.asarray(probs, dtype=np.float64)
    exp = counts.sum() * probs
    return float(chi2.sf(((counts - exp) ** 2 / exp).sum(), len(probs) - 1))


def chi2_power(N, probs, rel=0.05):
    """Smallest probability, over the cells, that the test at P_FLOOR rejects when that one cell's probability is
    scaled by (1 + rel) (the others renormalised): noncentral chi-square with lambda = N sum (p' - p)^2 / p."""
    from scipy.stats import chi2, ncx2
    probs = np.asarray(probs, dtype=np.float64)
    df = len(probs) - 1
    crit = chi2.isf(P_FLOOR, df)
    worst = 1.0
    for i in range(len(probs)):
        q = probs * (1 - rel * probs[i] / (1 - probs[i]))
        q[i] = probs[i] * (1 + rel)
        lam = N * float(((q - probs) ** 2 / probs).sum())
        worst = min(worst, float(ncx2.sf(crit, df, lam)))
    return worst
