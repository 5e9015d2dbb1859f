"""GPU: the statistical-mode sampling of the demasking loop -- in-kernel Philox noise in phk_sample_tokens (u == NULL), the
fused wgmma logits head (phk_head_sample / _rng) and the masked-rows tail (phk_sample_tail_rows) -- against the independent
fp64 gumbel-max reference of tests/noise_ref.py, and the sampling distribution itself.

Exact tests: ids must equal the reference on every row whose argmax is decided under the stated error bound, the
undecided rows must stay a small fraction, scores must agree within the stated tolerance (tests/noise_cases.py):
  * phk_sample_tokens: l is the fp32 input (error 0) or the CFG combination (2^-22 of the operands);
  * phk_head_sample: fp32 accumulation of dim exact bf16 products, dim 2^-23 sum_k |e_k w_k|, plus the bias add;
  * the tail: the head's bound plus one bf16 rounding of the guided embedding, 2^-8 sum_k |e_k w_k|;
  * every kernel: 2^-22 |l / T| for 1 / T and the fma, and the documented lg2.approx error propagated through g.
Distribution tests: chi-square goodness of fit with a p-value floor of 1e-6 and fixed seeds; each test asserts that its N
and cell layout reject a 5 % relative change of any one cell's probability with probability > 0.99
(noncentral chi-square, noise_cases.chi2_power)."""
import numpy as np
import pytest
import torch

from phenaki_pytorch_b200 import _lib as L
from phenaki_pytorch_b200 import phenaki as PH
from tests import noise_cases as NC
from tests import noise_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
HI_SEED = (0x9E3779B97F4A7C15 ^ 0x5DEECE66D) & (2 ** 64 - 1)  # both 32-bit key words non-zero
WRAP = 2 ** 32 - 3  # counters carry into the high word inside one call


def sync():
    torch.cuda.synchronize()


# ---- phk_sample_tokens, u == NULL ----------------------------------------------------------------------------------
# V = 1..65536: block sizes 64 (V < 1024), 256 (1024 <= V < 8192) and 512 threads, several passes per block from V = 257 on

@pytest.mark.parametrize("V,T", [(1, 1.0), (3, 0.45), (4, 3.0), (5, 0.05), (257, 1.0), (1023, 0.0), (1024, 1e-12),
                                 (8191, 0.45), (8192, 3.0), (65536, 1.0), (65536, 0.05)])
def test_sample_tokens_in_kernel_noise_matches_reference(V, T):
    rows = 512 if V <= 1024 else 256
    NC.check_sample_tokens(L.lib(), DEV, rows=rows, V=V, T=T, seed=HI_SEED, offset=WRAP, data_seed=V, sync=sync)


@pytest.mark.parametrize("V,ld,scale,seg,T", [(257, 263, 2.5, (5, 9, 4), 0.7), (1024, 1030, 3.0, None, 1.0),
                                              (8192, 8197, 1.0, (64, 80, 16), 0.45), (100, 100, 3.0, (7, 7, 0), 0.0)])
def test_sample_tokens_scalar_path_cfg_and_row_map(V, ld, scale, seg, T):
    """ld % 4 != 0 (scalar loads), CFG pairs with scale != 1, the seg_* map of a primed sample (logits from the mapped row,
    noise from the token row)."""
    NC.check_sample_tokens(L.lib(), DEV, rows=320, V=V, T=T, seed=HI_SEED, offset=WRAP, ld=ld, scale=scale, seg=seg,
                           data_seed=ld, sync=sync)


# ---- phk_head_sample -----------------------------------------------------------------------------------------------
# vocabulary splits: n_splits = 132 / ceil(n / 128) capped by the tile count and re-balanced (head_sample.cu)

@pytest.mark.parametrize("n,V,dim,T", [
    (300, 1, 64, 1.0), (300, 2, 64, 0.45), (300, 3, 72, 1.0), (129, 5, 8, 3.0), (127, 63, 96, 1.0), (128, 64, 200, 0.45),
    (129, 65, 512, 1.0), (1, 127, 64, 1.0), (300, 128, 96, 0.05), (129, 129, 72, 1.0), (300, 1000, 512, 0.45),
    (128, 4097, 200, 1.0), (127, 16896, 64, 1.0),       # 1 token tile: 132 vocabulary splits of one tile each
    (300, 65536, 512, 1.0),                             # 3 token tiles: 43 splits of 12 tiles, the last with 8
    (16896, 1000, 64, 0.45), (16897, 1000, 64, 1.0),    # 132 / 133 token tiles: one split
    (40000, 129, 72, 1.0)])
def test_head_sample_matches_reference(n, V, dim, T):
    NC.check_head(L.lib(), DEV, n_tokens=n, V=V, dim=dim, T=T, seed=HI_SEED, offset=WRAP, data_seed=n + V + dim, sync=sync)


@pytest.mark.parametrize("n,V,dim,emb_rows,ld_emb,ldw", [(300, 1000, 200, 337, 216, 264), (129, 65, 72, 260, 80, 136),
                                                         (1, 5, 8, 128, 16, 8)])
def test_head_sample_never_reads_padding(n, V, dim, emb_rows, ld_emb, ldw):
    """NaN in the emb rows past n_tokens and in the padding columns of emb and W: nothing of it may reach a result."""
    NC.check_head(L.lib(), DEV, n_tokens=n, V=V, dim=dim, T=0.7, seed=HI_SEED, offset=WRAP, emb_rows=emb_rows,
                  ld_emb=ld_emb, ldw=ldw, data_seed=7, sync=sync)


@pytest.mark.parametrize("drop", ["bias", "mask", "ids", "pred", "score"])
def test_head_sample_optional_pointers(drop):
    NC.check_head(L.lib(), DEV, n_tokens=300, V=1000, dim=64, T=1.0, seed=HI_SEED, offset=WRAP, drop=(drop,), data_seed=3,
                  sync=sync)


def test_head_sample_rng_device_key_and_advance():
    """phk_head_sample_rng with the key in device memory draws what the by-value call draws; after
    phk_rng_advance(stride) the next call draws the reference's noise at offset + stride."""
    lib = L.lib()
    n, V, dim, T = 300, 1000, 128, 1.0
    emb, W, bias, l, dl = NC.head_inputs(n, V, dim, data_seed=5)
    offset = WRAP - 2
    as_i64 = lambda v: v - 2 ** 64 if v >= 2 ** 63 else v
    rng = torch.tensor([as_i64(HI_SEED), as_i64(offset)], dtype=torch.int64, device=DEV)
    _, by_value, _ = NC.run_head(lib, DEV, emb, W, bias, n_tokens=n, V=V, dim=dim, T=T, seed=HI_SEED, offset=offset,
                                 sync=sync)
    _, by_key, sc = NC.run_head(lib, DEV, emb, W, bias, n_tokens=n, V=V, dim=dim, T=T, seed=1, offset=2, rng=rng, sync=sync)
    assert np.array_equal(by_value, by_key)
    NC.judge("head rng", R.gumbel_max(l, T, HI_SEED, offset), l, T, dl, by_key, sc)
    stride = PH._noise_stride(n, V)
    L.check(lib.phk_rng_advance(L.ptr(rng), stride, L.stream_ptr()), "phk_rng_advance")
    _, nxt, sc = NC.run_head(lib, DEV, emb, W, bias, n_tokens=n, V=V, dim=dim, T=T, seed=1, offset=2, rng=rng, sync=sync)
    assert int(rng[1].item()) % 2 ** 64 == offset + stride
    NC.judge("head rng after advance", R.gumbel_max(l, T, HI_SEED, offset + stride), l, T, dl, nxt, sc)


# ---- the masked-rows tail ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("b,n,k,V,dim,counts,plen", [(3, 20, 9, 70, 128, None, 0), (3, 20, 9, 70, 128, [9, 4, 0], 0),
                                                     (2, 100, 40, 1000, 256, [40, 33], 24),
                                                     (4, 576, 100, 4096, 512, None, 0)])
def test_sample_tail_noise_uses_the_compact_row(b, n, k, V, dim, counts, plen):
    NC.check_tail(L.lib(), DEV, b=b, n=n, k=k, V=V, dim=dim, T=0.8, seed=HI_SEED, offset=WRAP, counts=counts, plen=plen,
                  data_seed=n, sync=sync)


# ---- counter ranges of the demasking loop --------------------------------------------------------------------------

def test_demask_iterations_reserve_disjoint_counter_ranges():
    """Phenaki.sample on the iteration path (one phk_maskgit_demask_iteration per step): the device counter
    rng_state[1] ends exactly steps * stride past the first reserved counter, stride = round_up(b n ceil(V/4) + 1, 4)
    (include/phk.h) = _noise_stride >= b n ceil(V/4), and torch's generator offset -- where the next sample's range
    starts -- is at or past that end."""
    import phenaki_pytorch_b200 as P
    from tests import cases as C
    torch.manual_seed(4)
    cv = P.CViViT(**C.SAMPLE_CVIVIT).to(DEV)
    mg = P.MaskGit(dim=128, num_tokens=256, max_seq_len=64, heads=2, dim_head=64, depth=1, dim_context=48).to(DEV)
    mg.precision = L.PREC_BF16
    steps = 4
    ph = P.Phenaki(cvivit=cv, maskgit=mg, steps=steps, text_embed_dim=48)
    ph.iteration_call = True
    ctx = C.synthetic_text_embeds(2, 6, 48, (6, 3), 3).to(DEV)
    gen = torch.cuda.default_generators[torch.cuda.current_device()]
    b, n, V = 2, 18, 256
    stride = (b * n * ((V + 3) // 4) + 1 + 3) // 4 * 4
    assert PH._noise_stride(b * n, V) == stride and stride >= b * n * ((V + 3) // 4)
    for _ in range(2):
        first = int(gen.get_offset())
        ph.sample(num_frames=7, text_embeds=ctx, return_token_ids=True)
        sync()
        (bufs,) = ph._iter_bufs.values()
        end = int(bufs["rng"][1].item()) % 2 ** 64
        assert end - first == steps * stride
        assert int(gen.get_offset()) >= end


# ---- distributions -------------------------------------------------------------------------------------------------

def _sample_rows(V, logits, rows, T, seed, offset):
    """`rows` token rows that all read the same logits row (seg_len 1, seg_stride 0): the sampled ids."""
    lg = torch.tensor(logits, dtype=torch.float32, device=DEV).reshape(1, V)
    pred = torch.empty(rows, dtype=torch.int64, device=DEV)
    L.check(L.lib().phk_sample_tokens(L.ptr(lg), None, V, None, seed, offset, 1.0, T, None, None, L.ptr(pred), None, rows,
                                      V, 1, 0, 0, L.stream_ptr()), "phk_sample_tokens")
    return pred


@pytest.mark.parametrize("T", [0.5, 1.0, 2.0])
def test_sample_tokens_samples_softmax_of_l_over_T(T):
    """N = 2^21 rows of the same 12 logits (spread 0.6 around 0); 12 cells, the smallest holding >= 4.5 % at T = 0.5."""
    V, N = 12, 2 ** 21
    l = np.linspace(-0.3, 0.3, V)[np.random.default_rng(0).permutation(V)]
    p = np.exp(l / T) / np.exp(l / T).sum()
    assert NC.chi2_power(N, p) > 0.99
    counts = torch.bincount(_sample_rows(V, l, N, T, HI_SEED, WRAP), minlength=V).cpu().numpy()
    assert counts.size == V
    pv = NC.chi2_pvalue(counts, p)
    assert pv > NC.P_FLOOR, f"T={T}: p-value {pv:.3g}, counts {counts.tolist()}"


@pytest.mark.parametrize("n_tokens,calls", [(32768, 32), (256, 4096)])
def test_head_sample_samples_softmax_of_l_over_T(n_tokens, calls):
    """Exactly known logits through the wgmma head: emb rows one-hot in column 0 (bf16), W[:, 0] bf16-exact, fp32 bias, so
    l_v = W[v, 0] + bias[v] exactly.  V = 8192 (64 tiles): the mass sits on columns 0, 63 (tile 0, first column quadrant),
    64, 127 (second quadrant), 128 (tile 1), 700 (tile 5) and 8191 (last tile), plus the 'other' cell.  32768 tokens are
    256 token tiles (one vocabulary split); 256 tokens are 2 tiles (64 splits of one tile each, every marked column in
    its own split but 0 / 63 / 64 / 127).  N = 2^20 draws over `calls` calls at disjoint offsets."""
    lib = L.lib()
    V, dim, T = 8192, 64, 1.0
    cols = [0, 63, 64, 127, 128, 700, V - 1]
    a = np.full(V, -5.5)
    a[cols] = 2.0
    b = np.zeros(V)
    b[cols] = [0.0, 0.25, -0.25, 0.5, -0.5, 0.125, -0.375]
    l = a + b
    p_all = np.exp(l / T) / np.exp(l / T).sum()
    p = np.append(p_all[cols], 1.0 - p_all[cols].sum())
    N = n_tokens * calls
    assert N == 2 ** 20 and NC.chi2_power(N, p) > 0.99
    emb = torch.zeros((n_tokens, dim), dtype=torch.bfloat16, device=DEV)
    emb[:, 0] = 1.0
    W = torch.zeros((V, dim), dtype=torch.bfloat16)
    W[:, 0] = torch.tensor(a, dtype=torch.float32).bfloat16()
    W = W.to(DEV)
    bias = torch.tensor(b, dtype=torch.float32, device=DEV)
    pred = torch.empty((calls, n_tokens), dtype=torch.int64, device=DEV)
    nb = int(lib.phk_head_sample_scratch_bytes(n_tokens))
    scratch = torch.empty(nb, dtype=torch.uint8, device=DEV)
    stride = PH._noise_stride(n_tokens, V)
    for c in range(calls):
        L.check(lib.phk_head_sample(L.ptr(emb), dim, n_tokens, L.ptr(W), dim, L.ptr(bias), n_tokens, V, dim, T, HI_SEED,
                                    WRAP + c * stride, None, None, L.ptr(pred[c]), None, L.ptr(scratch), nb,
                                    L.stream_ptr()), "phk_head_sample")
    cell = torch.full((V,), len(cols), dtype=torch.int64, device=DEV)
    cell[cols] = torch.arange(len(cols), device=DEV)
    counts = torch.bincount(cell[pred.reshape(-1)], minlength=len(p)).cpu().numpy()
    pv = NC.chi2_pvalue(counts, p)
    assert pv > NC.P_FLOOR, f"{n_tokens} tokens: p-value {pv:.3g}, counts {counts.tolist()} expected {(N * p).round().tolist()}"


def _independent_pairs(a, b, what):
    """Joint counts of (a, b) over the 16 x 16 = 256 cells against the uniform product distribution: N = 2^25 pairs
    (each cell expects 131072), enough to reject a 5 % change of any one cell."""
    N, p = a.numel(), np.full(256, 1 / 256)
    assert N == 2 ** 25 and NC.chi2_power(N, p) > 0.99
    counts = torch.bincount(a * 16 + b, minlength=256).cpu().numpy()
    pv = NC.chi2_pvalue(counts, p)
    assert pv > NC.P_FLOOR, f"{what}: p-value {pv:.3g}"


def test_noise_of_neighbouring_tokens_and_iterations_is_independent():
    """Uniform logits, V = 16 (uniform ids): token pairs (t, t + 1), (t, t + 1024), and the same token at offset o and at
    o + stride (two consecutive demasking iterations)."""
    V, rows, n = 16, 2 ** 26, 1024
    zero = np.zeros(V)
    ids = _sample_rows(V, zero, rows, 1.0, HI_SEED, WRAP)
    _independent_pairs(ids[0::2], ids[1::2], "(t, t + 1)")
    blocks = ids.reshape(-1, 2, n)
    _independent_pairs(blocks[:, 0].reshape(-1), blocks[:, 1].reshape(-1), f"(t, t + {n})")
    half = rows // 2
    stride = PH._noise_stride(half, V)
    first = ids[:half]
    second = _sample_rows(V, zero, half, 1.0, HI_SEED, WRAP + stride)
    _independent_pairs(first, second, "(offset o, offset o + stride)")
