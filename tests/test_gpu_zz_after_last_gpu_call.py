"""GPU: tests of the code written AFTER round 1's last GPU call (DESIGN sections 4.3, 8, 9): the masked-rows tail of the
demasking step, the shared first layer of a CFG pair, the cosine-sim VectorQuantize tokenizer.  All of it passes on the
CPU executor (tests/test_*_emulated_cpu.py run these same bodies); this file sorts after the validated suites so that,
under `pytest -x`, a surprise here cannot hide their results."""
import pytest
import torch

import phenaki_pytorch_b200 as P
from phenaki_pytorch_b200 import _lib as L
from tests import cases as C
from tests import test_gpu_decode as D
from tests import test_gpu_models as G

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.mark.parametrize("b,n,k,dim,V", [(4, 576, 100, 512, 4096), (2, 48, 17, 128, 300), (3, 30, 1, 256, 130),
                                         (4, 576, 441, 512, 1024)])
def test_sample_tail_on_the_masked_rows_only(b, n, k, dim, V):
    """phk_sample_tail (csrc/sample_tail.cu + the wgmma head on the compact rows) against plain torch arithmetic; the
    same body runs on the CPU executor in tests/test_sample_tail_emulated_cpu.py."""
    from tests import tail_cases
    tail_cases.check_exact_k(L.lib(), torch.device(DEV), b, n, k, dim, V, sync=torch.cuda.synchronize)


def test_fused_sample_step_on_masked_rows_equals_the_all_rows_step():
    """Model level, temperature 0 (pure argmax): telling phk_maskgit_sample_step how many tokens per sequence are masked
    (head on those rows only) must give the ids of the all-rows step at every masked position, the same confidences,
    and leave the other positions alone."""
    torch.manual_seed(8)
    cfg = dict(dim=128, num_tokens=1000, max_seq_len=256, heads=2, dim_head=64, depth=2, dim_context=96)
    mg = P.MaskGit(**cfg).to(DEV).eval()
    mg.precision = L.PREC_BF16
    b, shape, n, k = 3, (3, 6, 8), 144, 37
    g = torch.Generator().manual_seed(2)
    ids0 = torch.randint(0, cfg["num_tokens"] + 1, (b, n), generator=g).to(DEV)
    ctx = C.synthetic_text_embeds(b, 5, 96, (5, 2, 4), 2).to(DEV)
    tmask = torch.any(ctx != 0, dim=-1)
    mask = torch.zeros((b, n), dtype=torch.uint8)
    for i in range(b):
        mask[i, torch.randperm(n, generator=g)[:k]] = 1
    mask = mask.to(DEV)
    kv = mg.context_kv(ctx)
    outs = []
    for count in (0, k):
        ids, pred, sc = ids0.clone(), torch.empty_like(ids0), torch.empty((b, n), device=DEV)
        mg._sample_step(ids0, shape, ctx_kv=kv, ctx_len=5, text_mask=tmask, cond_scale=3.0, temperature=0.0, seed=1, offset=0,
                        mask=mask, ids=ids, pred=pred, scores=sc, masked_per_seq=count)
        torch.cuda.synchronize()
        outs.append((ids.cpu(), sc.cpu()))
    m = mask.cpu().bool()
    (ids_a, sc_a), (ids_b, sc_b) = outs
    same = ids_a == ids_b  # (a near-tie of two logits may resolve differently if the two LayerNorm kernels round apart)
    assert int((~same).sum()) <= max(1, int(0.01 * m.sum())), f"{int((~same).sum())} ids differ"
    torch.testing.assert_close(sc_a[m & same], sc_b[m & same], rtol=1e-3, atol=1e-4)
    assert bool((sc_b[~m] == -1e4).all()) and torch.equal(ids_b[~m], ids0.cpu()[~m])


def test_cosine_vq_ids_in_bf16_mode_against_fp32_reference_golden(golden):
    """lookup_free_quantization=False in bf16 mode: the nearest-code search runs on the fused wgmma head at temperature 0
    (phk_vq_cosine_ids).  An id may differ from the fp32 reference's only where the reference's similarities of the two
    candidates are within bf16 noise (0.03 in cosine units), and at least 85 % of the ids agree."""
    case, g = C.CVIVIT_CASES["cosine_vq"], golden("cvivit_cosine_vq")
    torch.manual_seed(case["seed"])
    model = P.CViViT(**case["ctor"]).to(DEV).eval()
    model.precision = L.PREC_BF16
    video = C.seeded_randn(case["video"], case["video_seed"]).to(DEV)
    got = model(video, return_only_codebook_ids=True).cpu().reshape(-1)
    want, sims = g["ids"].reshape(-1), g["proj"].reshape(-1, g["proj"].shape[-1])
    assert bool(((got >= 0) & (got < case["ctor"]["codebook_size"])).all())
    differ = torch.nonzero(got != want).flatten().tolist()
    for r in differ:
        assert abs(float(sims[r, got[r]] - sims[r, want[r]])) < 0.03, f"token {r}: a clearly worse code was chosen"
    assert len(differ) <= 0.15 * want.numel(), f"{len(differ)} of {want.numel()} ids differ"


def test_cosine_vq_token_ids_match_reference_golden(golden):
    """lookup_free_quantization=False, fp32 parity mode: ids identical to the reference's (stage taps as for LFQ)."""
    G.test_cvivit_token_ids_match_reference_golden(golden, "cosine_vq")


def test_cosine_vq_decode_matches_reference_golden(golden):
    D.test_decode_from_codebook_indices_matches_reference_golden(golden, "cosine_vq")


@pytest.mark.parametrize("k", [574, 288, 50])
def test_cfg3_masked_rows_step_equals_all_rows_step_at_full_size(k):
    """BASELINE configs[2] sizes (b=4, N=576, V=65536, depth 6, 16 text tokens): the demasking step with the head on the
    b*k masked rows (18, 9 and 2 token tiles -> 8, 16 and 74 vocabulary splits of the fused head) against the all-rows
    step, temperature 0: same ids at the masked positions, same confidences, nothing else touched."""
    torch.manual_seed(3)
    mg = P.MaskGit(dim=512, num_tokens=65536, max_seq_len=1024, dim_context=768, depth=6).to(DEV).eval()
    mg.precision = L.PREC_BF16
    b, shape, n = 4, (9, 8, 8), 576
    g = torch.Generator().manual_seed(k)
    ids0 = torch.randint(0, 65537, (b, n), generator=g).to(DEV)
    ctx = torch.randn((b, 16, 768), generator=g).to(DEV)
    tmask = torch.ones((b, 16), dtype=torch.bool, device=DEV)
    mask = torch.zeros((b, n), dtype=torch.uint8)
    for i in range(b):
        mask[i, torch.randperm(n, generator=g)[:k]] = 1
    mask = mask.to(DEV)
    kv = mg.context_kv(ctx)
    outs = []
    for count in (0, k):
        ids, pred, sc = ids0.clone(), torch.empty_like(ids0), torch.empty((b, n), device=DEV)
        mg._sample_step(ids0, shape, ctx_kv=kv, ctx_len=16, text_mask=tmask, cond_scale=3.0, temperature=0.0, seed=1, offset=0,
                        mask=mask, ids=ids, pred=pred, scores=sc, masked_per_seq=count)
        torch.cuda.synchronize()
        outs.append((ids.cpu(), sc.cpu()))
    m = mask.cpu().bool()
    (ids_a, sc_a), (ids_b, sc_b) = outs
    same = ids_a == ids_b
    assert int((~same).sum()) <= max(1, int(0.01 * m.sum())), f"{int((~same).sum())} ids differ"
    torch.testing.assert_close(sc_a[m & same], sc_b[m & same], rtol=1e-3, atol=1e-4)
    assert bool((sc_b[~m] == -1e4).all()) and torch.equal(ids_b[~m], ids0.cpu()[~m])
    assert bool(((ids_b[m] >= 0) & (ids_b[m] < 65536)).all())


def test_primed_fused_sample_step_equals_the_unprimed_step_on_the_same_rows():
    """phk_maskgit_sample_step_primed (scene chains of make_video, phenaki_pytorch.py:493, 503-504): with a prime prefix of
    `plen` ids the head runs on the masked rows of the sampled tokens only.  The step sees the same network input whether
    the prefix is declared as prime or the whole sequence is treated as sampled with the prefix unmasked, so at temperature
    0 both calls must produce the same ids / confidences on the sampled tokens."""
    torch.manual_seed(9)
    cfg = dict(dim=128, num_tokens=1000, max_seq_len=256, heads=2, dim_head=64, depth=2, dim_context=96)
    mg = P.MaskGit(**cfg).to(DEV).eval()
    mg.precision = L.PREC_BF16
    b, shape, n_total, plen = 2, (4, 4, 6), 96, 24
    n = n_total - plen
    g = torch.Generator().manual_seed(4)
    full = torch.randint(0, cfg["num_tokens"], (b, n_total), generator=g)
    k = 40
    mask_new = torch.zeros((b, n), dtype=torch.uint8)
    for i in range(b):
        mask_new[i, torch.randperm(n, generator=g)[:k]] = 1
    full[:, plen:][mask_new.bool()] = cfg["num_tokens"]  # masked positions carry the mask id
    ctx = C.synthetic_text_embeds(b, 5, 96, (5, 3), 6).to(DEV)
    tmask = torch.any(ctx != 0, dim=-1)
    kv = mg.context_kv(ctx)
    full_d, mask_new_d = full.to(DEV), mask_new.to(DEV)
    # (a) primed: mask / ids / pred / scores cover the n sampled tokens
    ids_a, pred_a, sc_a = full_d[:, plen:].clone(), torch.empty((b, n), dtype=torch.int64, device=DEV), torch.empty((b, n), device=DEV)
    mg._sample_step(full_d, shape, ctx_kv=kv, ctx_len=5, text_mask=tmask, cond_scale=3.0, temperature=0.0, seed=5, offset=0,
                    mask=mask_new_d, ids=ids_a, pred=pred_a, scores=sc_a, masked_per_seq=k, prime_len=plen)
    # (b) unprimed: the whole sequence, prefix unmasked
    mask_full = torch.cat((torch.zeros((b, plen), dtype=torch.uint8), mask_new), dim=1).to(DEV)
    ids_b, pred_b, sc_b = full_d.clone(), torch.empty_like(full_d), torch.empty((b, n_total), device=DEV)
    mg._sample_step(full_d, shape, ctx_kv=kv, ctx_len=5, text_mask=tmask, cond_scale=3.0, temperature=0.0, seed=5, offset=0,
                    mask=mask_full, ids=ids_b, pred=pred_b, scores=sc_b, masked_per_seq=k)
    if DEV == "cuda":
        torch.cuda.synchronize()
    assert torch.equal(ids_a.cpu(), ids_b[:, plen:].cpu())
    torch.testing.assert_close(sc_a.cpu(), sc_b[:, plen:].cpu(), rtol=1e-5, atol=1e-6)
    assert torch.equal(ids_b[:, :plen].cpu(), full[:, :plen])
