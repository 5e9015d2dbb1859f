"""Independent fp64 reference of the in-kernel sampling noise (include/phk.h, phk_sample_tokens with u == NULL).

Philox4x32-R is written from the published algorithm (Salmon, Moraes, Dror, Shaw: "Parallel random numbers: as easy as
1, 2, 3", SC'11; the Random123 library), not from the CUDA source: one round maps the counter (c0, c1, c2, c3) with the
round key (k0, k1) to

    (hi(M1 c2) ^ c1 ^ k0,  lo(M1 c2),  hi(M0 c0) ^ c3 ^ k1,  lo(M0 c0)),    M0 = 0xD2511F53, M1 = 0xCD9E8D57,

and the key is bumped by (0x9E3779B9, 0xBB67AE85) between rounds.  Everything here is vectorised numpy over uint64
arrays holding 32-bit words, so a 32 x 32 -> 64-bit product is exact.

The noise contract on top of it: draw v of token row r under (seed, offset) is word v % 4 of
Philox4x32-7(key = (seed lo, seed hi), counter = (c lo, c hi, 0, 0)), c = offset + r * ceil(V / 4) + v / 4 (mod 2^64);
u = (2 (draw >> 9) + 1) / 2^24 and g = -ln(-ln u), here in fp64.
"""
import math

import numpy as np

NOISE_ROUNDS = 7
M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
LO32 = np.uint64(0xFFFFFFFF)
S32 = np.uint64(32)


def philox4x32(ctr, key, rounds=NOISE_ROUNDS):
    """ctr: four arrays (or ints) of 32-bit words, key: two 32-bit words -> four uint64 arrays of 32-bit words."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) for c in ctr)
    c0, c1, c2, c3 = np.broadcast_arrays(c0, c1, c2, c3)
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    for r in range(rounds):
        if r:
            k0, k1 = (k0 + W0) & LO32, (k1 + W1) & LO32
        p0, p1 = M0 * c0, M1 * c2
        c0, c1, c2, c3 = (p1 >> S32) ^ c1 ^ k0, p1 & LO32, (p0 >> S32) ^ c3 ^ k1, p0 & LO32
    return c0, c1, c2, c3


def counters(seed, offset, row_ids, V):
    """64-bit Philox counters [rows, ceil(V / 4)] of the noise contract (wrapping mod 2^64)."""
    nb = (V + 3) // 4
    rows = np.asarray(row_ids, dtype=np.uint64).reshape(-1, 1)
    with np.errstate(over="ignore"):
        return np.uint64(offset % 2 ** 64) + rows * np.uint64(nb) + np.arange(nb, dtype=np.uint64)[None, :]


def draws(seed, offset, row_ids, V):
    """The raw 32-bit draws [rows, V]: column v is word v % 4 of the block of counter offset + row * ceil(V/4) + v/4."""
    seed %= 2 ** 64
    c = counters(seed, offset, row_ids, V)
    words = philox4x32((c & LO32, c >> S32, 0, 0), (seed & 0xFFFFFFFF, seed >> 32))
    return np.stack(words, axis=-1).reshape(c.shape[0], -1)[:, :V]


def uniforms(seed, offset, row_ids, V):
    """u = (2 k + 1) / 2^24 for the top 23 bits k of each draw: strictly inside (0, 1)."""
    return (2.0 * (draws(seed, offset, row_ids, V) >> np.uint64(9)).astype(np.float64) + 1.0) / 2.0 ** 24


def gumbel(u):
    return -np.log(-np.log(u))


class Sample:
    """pred: argmax of l / max(T, 1e-10) + g (first index on ties); gap: fp64 top-two gap of that perturbed logit
    (inf for V = 1); score: 1 - softmax(l)[pred]; y, u: the perturbed logits and the uniforms."""

    def __init__(self, pred, gap, score, y, u):
        self.pred, self.gap, self.score, self.y, self.u = pred, gap, score, y, u


def gumbel_max(l, T, seed, offset, row_ids=None):
    """Gumbel-max sampling of the fp64 logits l [rows, V] with the in-kernel noise of (seed, offset); row_ids: the
    counter row of each logits row (default 0 .. rows-1)."""
    l = np.asarray(l, dtype=np.float64)
    rows, V = l.shape
    row_ids = np.arange(rows) if row_ids is None else np.asarray(row_ids)
    u = uniforms(seed, offset, row_ids, V)
    y = l / max(float(T), 1e-10) + gumbel(u)
    pred = np.argmax(y, axis=1)
    r = np.arange(rows)
    if V > 1:
        top2 = np.partition(y, V - 2, axis=1)[:, V - 2:]
        gap = top2[:, 1] - top2[:, 0]
    else:
        gap = np.full(rows, np.inf)
    m = l.max(axis=1, keepdims=True)
    p = np.exp(l - m)
    p = p[r, pred] / p.sum(axis=1)
    return Sample(pred, gap, 1.0 - p, y, u)


# ---- device error model ----------------------------------------------------------------------------------------------
# lg2.approx.f32 (the instruction behind __log2f): absolute error <= 2^-22 for x in [0.5, 2], else <= 2 ulp
# (CUDA C++ Programming Guide, intrinsic functions).  The device computes g = -ln2 * lg2(-lg2(u)) + ln(ln 2) in fp32.
LG2_ABS = 2.0 ** -22
LG2_REL = 2.0 ** -22  # 2 ulp of an fp32 result is at most 2^-22 of its magnitude
LN2 = math.log(2.0)


def _lg2_err(x, lx):
    return np.where((x >= 0.5) & (x <= 2.0), LG2_ABS, LG2_REL * np.abs(lx))


def gumbel_err(u):
    """Bound of |g_device - g| for the uniforms u: the first lg2's error propagated through the second (first order,
    with the perturbed argument as the denominator, inf where the error could reach zero), the second lg2's own error,
    the fp32 constants -ln 2 and ln(ln 2) (2e-9 |lg2 e| + 3e-8) and the rounding of the final fma (2^-24 |g|)."""
    e = -np.log2(u)
    de = _lg2_err(u, e)
    lo = e - de
    with np.errstate(divide="ignore"):
        dle = np.where(lo > 0, de / np.maximum(lo, 1e-300) / LN2, np.inf)
    le = np.log2(e)
    dle = dle + _lg2_err(e, le)
    return LN2 * dle + 2e-9 * np.abs(le) + 3e-8 + 2.0 ** -24 * np.abs(gumbel(u))


def decided(y, err, pred):
    """Rows whose argmax cannot move when every perturbed logit moves by up to `err`: the reference winner beats every
    other column by more than the sum of the two bounds."""
    rows = np.arange(y.shape[0])
    if y.shape[1] == 1:
        return np.ones(y.shape[0], dtype=bool)
    top, etop = y[rows, pred], err[rows, pred]
    slack = top[:, None] - y - err
    slack[rows, pred] = np.inf
    return slack.min(axis=1) > etop
