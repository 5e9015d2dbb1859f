"""CPU (tests/cuda_emu): the in-kernel sampling noise against the independent fp64 gumbel-max reference of
tests/noise_ref.py.  The real sample_tokens_kernel (csrc/rowops.cu, u == NULL) and the real compaction / gather / scatter of
csrc/sample_tail.cu run from the shipped source; this pins their counter layout, CFG combination, seg_* row map and the
compact counter rows of the tail, and checks that the executor's copy of the generator agrees with the published
algorithm.  Judging rules (error bounds, undecided rows, score tolerance): tests/noise_cases.py."""
import numpy as np
import pytest
import torch

from phenaki_pytorch_b200 import _lib as L
from phenaki_pytorch_b200 import phenaki as PH
from tests import emu_runtime
from tests import noise_cases as NC
from tests import noise_ref as R

CPU = torch.device("cpu")
HI_SEED = (0x9E3779B97F4A7C15 ^ 0x5DEECE66D) & (2 ** 64 - 1)  # both 32-bit key words non-zero
WRAP = 2 ** 32 - 3  # counters carry into the high word inside one call


@pytest.fixture(scope="module")
def lib():
    return emu_runtime.build_emu()


@pytest.fixture(autouse=True)
def _cpu(lib, monkeypatch):
    monkeypatch.setattr(L, "stream_ptr", lambda: None)
    monkeypatch.setattr(L, "lib", lambda: lib)


def test_philox_reference_reproduces_the_published_known_answers():
    """Random123's known-answer vectors of Philox4x32-10 (kat_vectors): the reference is the published generator."""
    kat = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
           ((0xFFFFFFFF,) * 4, (0xFFFFFFFF, 0xFFFFFFFF), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
           ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
            (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for ctr, key, want in kat:
        assert tuple(int(w) for w in R.philox4x32(ctr, key, rounds=10)) == want


def test_noise_contract_layout():
    """Counter = offset + row ceil(V/4) + v/4 in 64 bits, draw = word v % 4: a V = 7 row spans two blocks, the second
    row starts at the next block, and the 64-bit counter wraps."""
    seed = HI_SEED
    d = R.draws(seed, WRAP, [0, 1], 7)
    for row in range(2):
        for v in range(7):
            c = (WRAP + row * 2 + v // 4) % 2 ** 64
            words = R.philox4x32((c & 0xFFFFFFFF, c >> 32, 0, 0), (seed & 0xFFFFFFFF, seed >> 32))
            assert int(d[row, v]) == int(words[v % 4])
    top = R.draws(seed, 2 ** 64 - 1, [0], 8)
    assert np.array_equal(top[0, 4:], R.draws(seed, 0, [0], 4)[0])


@pytest.mark.parametrize("V,T", [(1, 1.0), (3, 0.45), (5, 3.0), (257, 1.0), (1024, 0.05), (1023, 1e-12), (8192, 0.45)])
def test_sample_tokens_in_kernel_noise_matches_reference(lib, V, T):
    NC.check_sample_tokens(lib, CPU, rows=12, V=V, T=T, seed=HI_SEED, offset=WRAP, data_seed=V)


def test_sample_tokens_scalar_path_cfg_and_row_map_match_reference(lib):
    """ld > V with ld % 4 != 0 (scalar loads), a CFG pair with scale 2.5, and the seg_* map of a primed sample
    (3 sequences of 5 sampled tokens behind 4 prime rows): logits from the mapped row, noise from the token row."""
    NC.check_sample_tokens(lib, CPU, rows=15, V=257, T=0.7, seed=HI_SEED, offset=WRAP, ld=263, scale=2.5, seg=(5, 9, 4),
                           data_seed=3)
    NC.check_sample_tokens(lib, CPU, rows=10, V=64, T=0.0, seed=7, offset=5, ld=66, scale=3.0, data_seed=4)


@pytest.mark.parametrize("counts,plen", [(None, 0), ([9, 4, 0], 0), ([9, 7, 3], 6)])
def test_sample_tail_rows_noise_uses_the_compact_row(lib, counts, plen):
    """The tail at T = 0.8 (phk_sample_tail_rows; the head is the executor's contract of phk_head_sample): counter row
    of a masked position = sequence * k + its rank among the sequence's masked positions; with fewer than k masked the
    padding rows keep their counters and scatter nothing; a prime prefix (src_stride / src_off) moves only the rows read."""
    NC.check_tail(lib, CPU, b=3, n=20, k=9, V=70, dim=128, T=0.8, seed=HI_SEED, offset=WRAP, counts=counts, plen=plen,
                  data_seed=11)


def test_noise_stride_covers_one_draw_and_matches_the_library_advance(lib, monkeypatch):
    """Phenaki.sample on the iteration path (phk_maskgit_demask_iteration per step, executed from csrc/api.cu): the
    device counter ends exactly steps * _noise_stride(b n, V) past the first reserved counter, _noise_stride is the
    documented round_up(b n ceil(V/4) + 1, 4) >= b n ceil(V/4), and the next sample's range starts at or after it."""
    import phenaki_pytorch_b200 as P
    from tests import cases as C
    emu_runtime.route_product_to_emulator(lib, monkeypatch)
    torch.manual_seed(4)
    cv = P.CViViT(**C.SAMPLE_CVIVIT)
    mg = P.MaskGit(dim=128, num_tokens=256, max_seq_len=64, heads=2, dim_head=64, depth=1, dim_context=48)
    mg.precision = L.PREC_BF16
    steps = 3
    ph = P.Phenaki(cvivit=cv, maskgit=mg, steps=steps, text_embed_dim=48)
    ph.iteration_call = True
    ctx = C.synthetic_text_embeds(2, 6, 48, (6, 3), 3)
    taken = []
    real_take = PH._rng_take
    monkeypatch.setattr(PH, "_rng_take", lambda dev, seed, count: taken.append(real_take(dev, seed, count)) or taken[-1])
    ends = []
    for _ in range(2):
        ph.sample(num_frames=7, text_embeds=ctx, return_token_ids=True)
        (bufs,) = [v for k, v in ph._iter_bufs.items()]
        ends.append(int(bufs["rng"][1]) % 2 ** 64)
    b, n, V = 2, 18, 256
    stride = (b * n * ((V + 3) // 4) + 1 + 3) // 4 * 4
    assert PH._noise_stride(b * n, V) == stride and stride >= b * n * ((V + 3) // 4)
    assert ends[0] - taken[0] == steps * stride
    assert ends[1] - taken[1] == steps * stride
    assert taken[1] >= ends[0]
