"""GPU: PHK_PREC_BF16X3 -- fp32-grade nn.Linear products on the wgmma tensor cores (operands split into two bf16 terms,
one GEMM over K' = 3K) with the parity mode's fp32 LayerNorm / attention core / GEGLU around them.  Bars are the fp32
parity mode's: token ids identical to the reference goldens, activations / logits / pixels within 2e-4 (+ 2e-4 |ref|).
At configs[1] / configs[2] sizes: tests/test_gpu_parity_at_size.py."""
import pytest
import torch

import phenaki_pytorch_b200 as P
from phenaki_pytorch_b200 import _lib as L
from tests import cases as C

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.mark.parametrize("M,N,K", [(300, 200, 512), (129, 96, 77), (4608, 512, 1365)])
def test_split_gemm_matches_fp64_product_to_fp32_grade(M, N, K):
    """phk_split3 on both sides + one wgmma GEMM over 3 Kp == A W^T to ~1e-5 of the row scale (bf16 alone: ~4e-3)."""
    from phenaki_pytorch_b200.modules import split3_weight
    a, w = C.seeded_randn((M, K), 500), C.seeded_randn((N, K), 501) / K ** 0.5
    ref = (a.double() @ w.double().t()).float()
    lib = L.lib()
    kp = (K + 7) // 8 * 8
    ad, w3 = a.to(DEV), split3_weight(w.to(DEV))
    a3 = torch.empty((M, 3 * kp), dtype=torch.bfloat16, device=DEV)
    L.check(lib.phk_split3(L.ptr(ad), K, L.ptr(a3), M, K, 0, L.stream_ptr()), "phk_split3")
    w3k = torch.empty((N, 3 * kp), dtype=torch.bfloat16, device=DEV)
    wd = w.to(DEV)
    L.check(lib.phk_split3(L.ptr(wd), K, L.ptr(w3k), N, K, 1, L.stream_ptr()), "phk_split3")
    assert torch.equal(w3k, w3)  # the kernel's weight-side split == the host pack
    out = torch.empty((M, N), dtype=torch.float32, device=DEV)
    L.check(lib.phk_gemm_bf16(L.ptr(a3), 3 * kp, L.ptr(w3), 3 * kp, L.ptr(out), N, M, N, 3 * kp, None, None, 0, 0, 0, 0,
                              L.stream_ptr()), "phk_gemm_bf16")
    err = (out.cpu() - ref).abs().max().item()
    assert err <= 1.5e-4, err  # measured 5.7e-5 at K = 1365 on O(1) outputs (plain bf16 operands: ~4e-3)


@pytest.mark.parametrize("name", ["cfg1", "rect", "image"])
def test_cvivit_ids_and_reconstruction_in_split_bf16_mode(golden, name):
    case, g = C.CVIVIT_CASES[name], golden(f"cvivit_{name}")
    torch.manual_seed(case["seed"])
    model = P.CViViT(**case["ctor"]).to(DEV).eval()
    model.precision = L.PREC_BF16X3
    video = C.seeded_randn(case["video"], case["video_seed"]).to(DEV)
    ids = model(video, return_only_codebook_ids=True)
    assert torch.equal(ids.cpu(), g["ids"])
    rec = model.decode_from_codebook_indices(ids)
    model.precision = L.PREC_F32
    torch.testing.assert_close(rec, model.decode_from_codebook_indices(ids), rtol=2e-4, atol=2e-4)


@pytest.mark.parametrize("name", list(C.MASKGIT_CASES))
def test_maskgit_logits_in_split_bf16_mode(golden, name):
    case, g = C.MASKGIT_CASES[name], golden(f"maskgit_{name}")
    torch.manual_seed(case["seed"])
    model = P.MaskGit(**case["ctor"]).to(DEV).eval()
    model.precision = L.PREC_BF16X3
    ids, ctx = C.token_inputs(case, case["ctor"]["num_tokens"])
    ids, ctx = ids.to(DEV), ctx.to(DEV)
    kw = dict(text_mask=torch.any(ctx != 0, dim=-1), video_patch_shape=case["patch_shape"], context=ctx)
    torch.testing.assert_close(model(ids, **kw).cpu(), g["cond"], rtol=2e-4, atol=2e-4)
    torch.testing.assert_close(model.forward_with_cond_scale(ids, cond_scale=3.0, **kw).cpu(), g["cfg"], rtol=2e-4, atol=1e-3)


def test_sampling_loop_in_split_bf16_mode_equals_the_reference(golden):
    """The free-running demasking loop with the reference's noise replayed: every integer identical, as in fp32 mode."""
    case, g = C.SAMPLE_CASES["confidence"], golden("sample_confidence")
    torch.manual_seed(case["seed"])
    cv, mg = P.CViViT(**C.SAMPLE_CVIVIT), P.MaskGit(**C.SAMPLE_MASKGIT)
    mg.precision = cv.precision = L.PREC_BF16X3
    ph = P.Phenaki(cvivit=cv.to(DEV), maskgit=mg.to(DEV), steps=case["steps"], text_embed_dim=C.SAMPLE_MASKGIT["dim_context"])
    ph.cvivit.precision = L.PREC_BF16X3
    ctx = C.synthetic_text_embeds(case["batch"], case["ctx_len"], C.SAMPLE_MASKGIT["dim_context"], case["ctx_valid"],
                                  case["seed"] + 1000).to(DEV)
    tape = C.NoiseTape(case["noise_seed"])
    ids = ph.sample(num_frames=case["num_frames"], text_embeds=ctx, cond_scale=case["cond_scale"], return_token_ids=True,
                    noise_fn=lambda shape, tag: tape(shape, tag).to(DEV))
    assert torch.equal(ids.cpu(), g["final_ids"])
