"""Case lists of the rest of the training backward (tests/train_backward_cases.py), shared by the GPU file (production
shapes plus the edges) and the CPU executor's file (reduced shapes plus the same edges)."""


def ln(rows, dim, dx="write", dbeta=True):
    return dict(id=f"{rows}x{dim}-dx_{dx}-{'dbeta' if dbeta else 'nobeta'}", rows=rows, dim=dim, dx=dx, dbeta=dbeta,
                seed=rows + 3 * dim)


# E: rows {1, 7, 257, 4097} x dim {33, 512, 768, 1536}; dx written / accumulated / NULL; dbeta NULL and present;
# 4097 rows: the default path's 64-chunk cap bites and the fixed path's last 256-row block holds one row
LN_EDGES = [ln(1, 33), ln(7, 512, "acc"), ln(257, 33, None, False), ln(257, 768, "acc", False), ln(4097, 33, "acc"),
            ln(7, 1536, None), ln(1, 768, "acc", False), ln(257, 1536)]
LN_EDGES_GPU = LN_EDGES + [ln(4097, 512), ln(4097, 1536, "acc", False)]


def geglu(rows, inner, p):
    return dict(id=f"{rows}x{inner}-p{p}", rows=rows, inner=inner, p=p, seed=rows + inner + int(100 * p))


GEGLU_EDGES = [geglu(9, inner, p) for inner in (1365, 77) for p in (0.0, 0.1, 1.0)]


def peg(B, T, H, W, D, causal):
    return dict(id=f"{B}x{T}x{H}x{W}-D{D}-{'causal' if causal else 'plain'}", B=B, T=T, H=H, W=W, D=D, causal=causal,
                seed=B + T * 7 + H * 11 + W * 13 + D)


# G: causal and not; a unit axis (every tap across it out of range); D 96 / 512 / 1024; fewer than 16 positions
PEG_EDGES = [peg(2, 3, 4, 5, 96, True), peg(1, 4, 1, 3, 96, False), peg(1, 1, 3, 3, 96, True),
             peg(1, 2, 2, 3, 512, True), peg(1, 3, 2, 1, 1024, False), peg(2, 2, 3, 3, 1024, True)]


def embed(b, n, D, vocab, ids, alpha=0.1):
    return dict(id=f"{b}x{n}-D{D}-V{vocab}-{ids}", b=b, n=n, D=D, vocab=vocab, ids=ids, alpha=alpha,
                seed=b * n + D + vocab)


# H: random ids; every row the mask id over more than two 128-row leader tiles; ids -1 and >= vocab; dim 33 / 512 / 768
EMBED_EDGES = [embed(3, 100, 33, 50, "random"), embed(3, 100, 768, 50, "mask"), embed(2, 37, 512, 20, "clamp"),
               embed(4, 70, 768, 300, "random")]


def cpb(dims, hidden, heads):
    return dict(id="x".join(map(str, dims)) + f"-h{hidden}", dims=dims, hidden=hidden, heads=heads,
                seed=sum(dims) + hidden)


CPB_EDGES = [cpb((1, 1, 1), 32, 4), cpb((3, 4), 32, 4), cpb((2, 3, 3), 48, 8)]


def ce(rows, V, mask, scale=1.0):
    return dict(id=f"{rows}x{V}-{mask}-s{scale}", rows=rows, V=V, mask=mask, scale=scale, seed=rows + V)


# J: V 65536 / 1000 / 257, logits +-80, a row whose target probability rounds to 1, partial / all-true / all-false masks
CE_EDGES = [ce(6, 1000, "partial", 0.5), ce(5, 257, "all"), ce(4, 257, "none"), ce(3, 65536, "partial")]


def bce(rows, D, scale):
    return dict(id=f"{rows}x{D}-s{scale}", rows=rows, D=D, scale=scale, seed=rows + D)


BCE_EDGES = [bce(41, 64, 0.5), bce(9, 512, 2.0)]
