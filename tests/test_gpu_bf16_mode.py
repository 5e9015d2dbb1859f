"""GPU: PHK_PREC_BF16 (wgmma GEMMs, bf16 operands, fp32 accumulation / residual / LayerNorm / softmax)
against the fp32 reference goldens.  This is the dtype flow of the reference under
torch.autocast(bfloat16) (SURVEY.md H2), so the comparison is reference-fp32 vs bf16 contraction noise.

Stated tolerances (normalised activations are O(1); bf16 has 8 mantissa bits, error grows ~sqrt(layers)):
  * activations after patch-embed / each transformer:  |err| <= 0.06 + 0.03*|ref|
  * MaskGit logits / embeds:                           |err| <= 0.08 + 0.03*|ref|
  * LFQ token ids: a bit may flip only where the reference pre-sign margin is below 0.12
    (the bf16 noise floor on the 16 projections); bits with larger margins must agree, and
    overall bit agreement must exceed 97 %.
"""
import pytest
import torch

import phenaki_pytorch_b200 as P
from phenaki_pytorch_b200 import _lib as L
from tests import cases as C

pytestmark = pytest.mark.gpu
DEV = "cuda"


def close(a, b, atol, rtol, what):
    err = (a - b).abs()
    bound = atol + rtol * b.abs()
    worst = float((err - bound).max())
    assert worst <= 0, f"{what}: max |err| {float(err.max()):.4f} exceeds {atol} + {rtol}*|ref| by {worst:.4f}"
    return float(err.max())


@pytest.mark.parametrize("name", ["cfg1", "rect"])
def test_cvivit_bf16_mode_against_fp32_reference_golden(golden, name):
    case, g = C.CVIVIT_CASES[name], golden(f"cvivit_{name}")
    torch.manual_seed(case["seed"])
    model = P.CViViT(**case["ctor"]).to(DEV).eval()
    model.precision = L.PREC_BF16
    video = C.seeded_randn(case["video"], case["video_seed"]).to(DEV)
    taps = {}
    ids = model.encode_ids(video, taps=taps)
    b, t, h, w, d = g["patch"].shape
    close(taps["patch"].cpu(), g["patch"], 0.06, 0.03, "patch embed")
    close(taps["spatial"].cpu().reshape(b * t, h * w, d), g["spatial"], 0.06, 0.03, "spatial transformer")
    close(taps["temporal"].cpu().permute(0, 2, 3, 1, 4).reshape(b * h * w, t, d), g["temporal"], 0.06, 0.03,
          "temporal transformer")
    bits = model.vq.codebook_dim
    proj = g["proj"].reshape(-1, bits)
    diff = (ids.cpu().reshape(-1) ^ g["ids"].reshape(-1))
    flipped = 0
    for r in range(diff.numel()):
        for dbit in range(bits):
            if (int(diff[r]) >> (bits - 1 - dbit)) & 1:
                flipped += 1
                assert abs(float(proj[r, dbit])) < 0.12, f"bit flipped with reference margin {float(proj[r, dbit]):.3f}"
    assert flipped <= 0.03 * diff.numel() * bits, f"{flipped} of {diff.numel() * bits} LFQ bits differ"


def test_maskgit_bf16_mode_against_fp32_reference_golden(golden):
    case, g = C.MASKGIT_CASES["wide"], golden("maskgit_wide")
    torch.manual_seed(case["seed"])
    model = P.MaskGit(**case["ctor"]).to(DEV).eval()
    model.precision = L.PREC_BF16
    ids, ctx = C.token_inputs(case, case["ctor"]["num_tokens"])
    ids, ctx = ids.to(DEV), ctx.to(DEV)
    kw = dict(text_mask=torch.any(ctx != 0, dim=-1), video_patch_shape=case["patch_shape"], context=ctx)
    close(model(ids, return_embeds=True, **kw).cpu(), g["embeds"], 0.08, 0.03, "embeds")
    close(model(ids, **kw).cpu(), g["cond"], 0.08, 0.03, "logits (cond)")
    close(model(ids, cond_drop_prob=1.0, **kw).cpu(), g["null"], 0.08, 0.03, "logits (null)")


def test_sampling_runs_in_bf16_mode_and_is_deterministic():
    case = C.SAMPLE_CASES["critic_primed"]
    torch.manual_seed(case["seed"])
    cv, mg, cr = P.CViViT(**C.SAMPLE_CVIVIT), P.MaskGit(**C.SAMPLE_MASKGIT), P.TokenCritic(**C.SAMPLE_CRITIC)
    for m in (cv, mg, cr):
        m.precision = L.PREC_BF16
    ph = P.Phenaki(cvivit=cv.to(DEV), maskgit=mg.to(DEV), critic=cr.to(DEV), steps=4,
                   text_embed_dim=C.SAMPLE_MASKGIT["dim_context"])
    ph.cvivit.precision = L.PREC_BF16
    ctx = C.synthetic_text_embeds(2, 6, C.SAMPLE_MASKGIT["dim_context"], (6, 3), 3).to(DEV)
    outs = []
    for _ in range(2):
        tape = C.NoiseTape(8)
        outs.append(ph.sample(num_frames=7, text_embeds=ctx, return_token_ids=True,
                              noise_fn=lambda s, t: tape(s, t).to(DEV)).cpu())
    assert torch.equal(outs[0], outs[1])
    assert (outs[0] < C.SAMPLE_MASKGIT["num_tokens"]).all()


def test_layernorm_cfg_combination():
    """e_cfg = LN(x_null) + s*(LN(x_cond) - LN(x_null)) (guidance folded before the linear logits head)."""
    rows, dim, scale = 70, 512, 3.0
    xc, xn = C.seeded_randn((rows, dim), 300) * 2 + 0.3, C.seeded_randn((rows, dim), 301)
    g, b = C.seeded_randn((dim,), 302), C.seeded_randn((dim,), 303)
    ln = lambda t: torch.nn.functional.layer_norm(t, (dim,), g, b)
    ref = ln(xn) + (ln(xc) - ln(xn)) * scale
    xcd, xnd, gd, bd = xc.to(DEV), xn.to(DEV), g.to(DEV), b.to(DEV)
    out = torch.empty((rows, dim), dtype=torch.bfloat16, device=DEV)
    L.check(L.lib().phk_layernorm_cfg(L.ptr(xcd), L.ptr(xnd), L.ptr(gd), L.ptr(bd), scale, L.ptr(out), rows, dim,
                                      L.stream_ptr()))
    torch.testing.assert_close(out.cpu().float(), ref, rtol=1e-2, atol=3e-2)  # one bf16 rounding


@pytest.mark.parametrize("n_tokens,V,dim", [(300, 1000, 128), (2304, 4096, 512), (64, 130, 256)])
def test_fused_head_kernel_matches_gemm_plus_sample_tokens(n_tokens, V, dim):
    """phk_head_sample (logits only ever in registers) vs phk_gemm_bf16 -> logits -> phk_sample_tokens with the same
    Philox counters: identical sampled ids (same MMA arithmetic), confidence within 1e-4 (softmax summation order)."""
    lib = L.lib()
    emb = (C.seeded_randn((n_tokens, dim), 310)).bfloat16().to(DEV)
    W = (C.seeded_randn((V, dim), 311) / dim ** 0.5).bfloat16().to(DEV)
    bias = C.seeded_randn((V,), 312).to(DEV)
    g = torch.Generator().manual_seed(5)
    mask = (torch.rand(n_tokens, generator=g) < 0.6).to(torch.uint8).to(DEV)
    ids0 = torch.randint(0, V, (n_tokens,), generator=g).to(DEV)
    seed, offset, temp = 99, 1234567, 0.55
    logits = torch.empty((n_tokens, V), device=DEV)
    L.check(lib.phk_gemm_bf16(L.ptr(emb), dim, L.ptr(W), dim, L.ptr(logits), V, n_tokens, V, dim, L.ptr(bias), None,
                              0, 0, 0, 0, L.stream_ptr()))
    ids_a, pred_a, sc_a = ids0.clone(), torch.empty_like(ids0), torch.empty(n_tokens, device=DEV)
    L.check(lib.phk_sample_tokens(L.ptr(logits), None, V, None, seed, offset, 1.0, temp, L.ptr(mask), L.ptr(ids_a),
                                  L.ptr(pred_a), L.ptr(sc_a), n_tokens, V, 0, 0, 0, L.stream_ptr()))
    ids_b, pred_b, sc_b = ids0.clone(), torch.empty_like(ids0), torch.empty(n_tokens, device=DEV)
    nb = lib.phk_head_sample_scratch_bytes(n_tokens)
    scratch = torch.empty(nb, dtype=torch.uint8, device=DEV)
    L.check(lib.phk_head_sample(L.ptr(emb), dim, n_tokens, L.ptr(W), dim, L.ptr(bias), n_tokens, V, dim, temp, seed,
                                offset, L.ptr(mask), L.ptr(ids_b), L.ptr(pred_b), L.ptr(sc_b), L.ptr(scratch), nb,
                                L.stream_ptr()))
    torch.cuda.synchronize()
    assert torch.equal(pred_a, pred_b)
    assert torch.equal(ids_a, ids_b)
    torch.testing.assert_close(sc_a, sc_b, rtol=1e-4, atol=1e-4)


def test_fused_sample_step_agrees_with_unfused_path():
    """Model level: guidance folded into the embeddings (fused) vs combined on the logits (reference order).  Same
    noise counters; the two differ only by bf16 rounding of the guided embedding, so the sampled ids agree on the large
    majority of tokens and the confidences are close."""
    torch.manual_seed(7)
    cfg = dict(dim=128, num_tokens=1000, max_seq_len=256, heads=2, dim_head=64, depth=2, dim_context=96)
    mg = P.MaskGit(**cfg).to(DEV).eval()
    mg.precision = L.PREC_BF16
    b, shape, n = 3, (3, 6, 8), 144
    g = torch.Generator().manual_seed(1)
    ids0 = torch.randint(0, cfg["num_tokens"] + 1, (b, n), generator=g).to(DEV)
    ctx = C.synthetic_text_embeds(b, 5, 96, (5, 2, 4), 2).to(DEV)
    tmask = torch.any(ctx != 0, dim=-1)
    mask = (torch.rand(b, n, generator=g) < 0.7).to(torch.uint8).to(DEV)
    kv = mg.context_kv(ctx)
    lib = L.lib()
    seed, offset, scale, temp = 1234, 77, 3.0, 0.6
    logits = mg._run(ids0, shape, ctx_kv=kv, ctx_len=5, text_mask=tmask, cfg_pair=True)
    ids_a, pred_a, sc_a = ids0.clone(), torch.empty_like(ids0), torch.empty((b, n), device=DEV)
    L.check(lib.phk_sample_tokens(L.ptr(logits[:b]), L.ptr(logits[b:]), 1000, None, seed, offset, scale, temp,
                                  L.ptr(mask), L.ptr(ids_a), L.ptr(pred_a), L.ptr(sc_a), b * n, 1000, 0, 0, 0,
                                  L.stream_ptr()))
    ids_b, pred_b, sc_b = ids0.clone(), torch.empty_like(ids0), torch.empty((b, n), device=DEV)
    mg._sample_step(ids_b, shape, ctx_kv=kv, ctx_len=5, text_mask=tmask, cond_scale=scale, temperature=temp, seed=seed,
                    offset=offset, mask=mask, ids=ids_b, pred=pred_b, scores=sc_b)
    torch.cuda.synchronize()
    agree = (pred_a == pred_b).float().mean().item()
    assert agree >= 0.9, f"only {agree:.3f} of the sampled ids agree"
    same = pred_a == pred_b
    torch.testing.assert_close(sc_a[same], sc_b[same], rtol=0.05, atol=2e-3)
    assert torch.equal(ids_b[mask == 0], ids0[mask == 0]) and torch.equal(ids_b[mask == 1], pred_b[mask == 1])


def test_bf16_sampling_with_fused_head_is_deterministic():
    case = C.SAMPLE_CASES["confidence"]
    torch.manual_seed(case["seed"])
    cv = P.CViViT(**C.SAMPLE_CVIVIT)
    mg = P.MaskGit(dim=128, num_tokens=256, max_seq_len=64, heads=2, dim_head=64, depth=2, dim_context=48)
    mg.precision = L.PREC_BF16
    ph = P.Phenaki(cvivit=cv.to(DEV), maskgit=mg.to(DEV), steps=6, text_embed_dim=48)
    ctx = C.synthetic_text_embeds(2, 6, 48, (6, 3), 3).to(DEV)
    outs = []
    for seed in (11, 11, 12):
        torch.manual_seed(seed)
        outs.append(ph.sample(num_frames=7, text_embeds=ctx, return_token_ids=True).cpu())
    assert torch.equal(outs[0], outs[1]) and not torch.equal(outs[0], outs[2])
    assert (outs[0] >= 0).all() and (outs[0] < 256).all()



@pytest.mark.parametrize("dim", [192, 768])
def test_bf16_sampling_falls_back_to_the_unfused_step_for_widths_the_fused_head_does_not_take(dim):
    """The fused demasking step keeps a token tile's whole embedding row in shared memory (dim <= 512, dim % 128 == 0);
    other widths must take phk_maskgit_forward + phk_sample_tokens instead of raising (ADVICE r01)."""
    torch.manual_seed(3)
    cv = P.CViViT(**C.SAMPLE_CVIVIT)
    mg = P.MaskGit(dim=dim, num_tokens=256, max_seq_len=64, heads=2, dim_head=64, depth=1, dim_context=48)
    mg.precision = L.PREC_BF16
    ph = P.Phenaki(cvivit=cv.to(DEV), maskgit=mg.to(DEV), steps=4, text_embed_dim=48)
    ctx = C.synthetic_text_embeds(2, 6, 48, (6, 3), 3).to(DEV)
    ids = ph.sample(num_frames=7, text_embeds=ctx, return_token_ids=True).cpu()
    assert tuple(ids.shape) == (2, 18) and bool(((ids >= 0) & (ids < 256)).all())


def test_one_graph_launch_per_iteration_equals_the_per_step_loop():
    """BASELINE north_star "one kernel launch per decode iteration": phk_maskgit_demask_iteration (default; eager on the
    first sample with a shape, captured on the second, ONE cudaGraphLaunch per iteration from the third on) against the
    per-step loop (PHK_STEP_GRAPH=0 path): same noise counters, so the ids of four consecutive samples are identical."""
    torch.manual_seed(2)
    cv = P.CViViT(**C.SAMPLE_CVIVIT)
    mg = P.MaskGit(dim=128, num_tokens=256, max_seq_len=64, heads=2, dim_head=64, depth=2, dim_context=48)
    mg.precision = L.PREC_BF16
    ph = P.Phenaki(cvivit=cv.to(DEV), maskgit=mg.to(DEV), steps=6, text_embed_dim=48)
    ctx = C.synthetic_text_embeds(2, 6, 48, (6, 3), 3).to(DEV)
    runs = {}
    for graph in (True, False):
        ph.iteration_call = graph
        torch.manual_seed(21)
        l0 = L.lib().phk_launch_count()
        runs[graph] = [ph.sample(num_frames=7, text_embeds=ctx, return_token_ids=True).cpu() for _ in range(4)]
        runs[graph, "launches"] = L.lib().phk_launch_count() - l0
    for a, b in zip(runs[True], runs[False]):
        assert torch.equal(a, b)
    assert not torch.equal(runs[True][0], runs[True][1])  # fresh noise per sample
    assert bool(((runs[True][3] >= 0) & (runs[True][3] < 256)).all())


@pytest.mark.parametrize("critic_kind,primed", [("token", True), ("self", False), (None, True)])
def test_critic_and_primed_iterations_equal_the_per_step_loop(critic_kind, primed):
    """phk_maskgit_demask_iteration (re-mask + MaskGit CFG pair + tail + critic CFG pair + scores in ONE launch
    sequence per iteration, replayed as a graph from the third sample on; make_video's primed scenes) against the per-step
    loop: same V-wide noise counters and the same torch generator draws for the critic noise -> identical ids, four
    consecutive samples."""
    torch.manual_seed(31)
    cv = P.CViViT(**C.SAMPLE_CVIVIT)
    mg = P.MaskGit(dim=128, num_tokens=256, max_seq_len=64, heads=2, dim_head=64, depth=2, dim_context=48)
    critic = None
    if critic_kind == "token":
        critic = P.TokenCritic(dim=128, num_tokens=256, max_seq_len=64, has_cross_attn=True, heads=2, dim_head=64, depth=1,
                               dim_context=48).to(DEV)
        critic.precision = L.PREC_BF16
    mg = mg.to(DEV)
    if critic_kind == "self":
        critic = P.SelfCritic(mg).to(DEV)
    mg.precision = L.PREC_BF16
    ph = P.Phenaki(cvivit=cv.to(DEV), maskgit=mg, critic=critic, steps=5, text_embed_dim=48)
    ctx = C.synthetic_text_embeds(2, 6, 48, (6, 3), 3).to(DEV)
    prime = torch.randint(0, 256, (2, 16), generator=torch.Generator().manual_seed(5)).to(DEV) if primed else None
    n = 32 if primed else 48
    runs = {}
    for graph in (True, False):
        ph.iteration_call = graph
        torch.manual_seed(12)
        runs[graph] = [ph.sample_token_ids(num_tokens=n, patch_shape=(3, 4, 4), batch_size=2, text_embeds=ctx,
                                           prime_token_ids=prime, cond_scale=3.0).cpu() for _ in range(4)]
    for a, b in zip(runs[True], runs[False]):
        assert torch.equal(a, b)
    assert not torch.equal(runs[True][0], runs[True][1])


def test_cvivit_with_36_token_frames_takes_the_mid_size_attention_and_tracks_fp32_mode():
    """Frames of 6 x 6 = 36 tokens: the spatial self-attention runs on attention_mid_mma_kernel (17..63 tokens) in bf16 mode.
    Against the same model in fp32 mode: LFQ bit agreement above the bf16 bar, and bf16 attention really ran on the mid-size
    kernel's path (the fp32 fallback for these lengths would give the same bar, so the launch count is checked too)."""
    torch.manual_seed(9)
    model = P.CViViT(dim=256, codebook_size=4096, image_size=48, patch_size=8, temporal_patch_size=2, spatial_depth=2,
                     temporal_depth=2, dim_head=64, heads=4, use_vgg_and_gan=False).to(DEV).eval()
    video = C.seeded_randn((3, 3, 5, 48, 48), 17).to(DEV)
    model.precision = L.PREC_F32
    ref = model(video, return_only_codebook_ids=True).cpu()
    model.precision = L.PREC_BF16
    ids = model(video, return_only_codebook_ids=True).cpu()
    assert ids.shape == ref.shape == (3, 3, 6, 6)
    x = (ids ^ ref).reshape(-1)
    flipped = sum(int(((x >> k) & 1).sum()) for k in range(12))
    assert flipped <= 0.03 * x.numel() * 12, f"{flipped} of {x.numel() * 12} LFQ bits differ from fp32 mode"
