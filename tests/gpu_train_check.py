"""Runs the CUDA training step (Phenaki.forward -> phk_maskgit_train_step) on cuda:0 against the reference's
autograd loss and gradients stored in tests/golden/train_*.pt and prints one line per case.

Importable (tests/test_gpu_train.py) and stand-alone: python tests/gpu_train_check.py [--bf16] [case ...].
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import phenaki_pytorch_b200 as P  # noqa: E402
from oracle import phenaki_oracle as O  # noqa: E402  (the checker)
from tests import cases as C  # noqa: E402


def check_case(name, verbose=True, bf16=False, device="cuda:0"):
    """bf16=True: wgmma products (PHK_PREC_BF16); the bar is then closeness to the fp32 reference (5 % of each
    gradient tensor's largest entry), not parity."""
    case = C.TRAIN_CASES[name]
    g = torch.load(os.path.join(ROOT, "tests", "golden", f"train_{name}.pt"), weights_only=False)
    torch.manual_seed(case["seed"])
    cvivit = P.CViViT(**C.SAMPLE_CVIVIT)
    maskgit = P.MaskGit(**case["maskgit"])
    critic = P.TokenCritic(**case["critic"]) if case["critic"] else None
    assert C.state_digest(maskgit.state_dict()) == g["maskgit_digest"]
    dev = torch.device(device)
    phenaki = P.Phenaki(cvivit=cvivit, maskgit=maskgit, critic=critic, steps=case["steps"],
                        self_token_critic=case.get("self_critic", False),
                        text_embed_dim=case["maskgit"]["dim_context"]).to(dev).train()
    if bf16:
        from phenaki_pytorch_b200 import _lib as L
        phenaki.maskgit.precision = L.PREC_BF16
        if critic is not None:
            critic.precision = L.PREC_BF16
    ids, ctx = C.train_inputs(case)
    b, n = ids.shape[0], ids[0].numel()
    vocab = case["maskgit"]["num_tokens"]
    # the reference's draws, in its order, from the CPU generator it used (tests/golden/make_golden.py::make_train)
    torch.manual_seed(case["noise_seed"])
    rand_step, u = O.train_draws(b, n, case["steps"])
    draws = {"rand_step": rand_step, "perm": u}
    if phenaki.critic is not None:
        draws["gumbel"] = torch.zeros((b, n, vocab)).uniform_(0, 1)
    loss = phenaki(video_codebook_ids=ids.to(dev), text_embeds=ctx.to(dev), draw_fn=lambda shape, tag: draws[tag])
    loss.backward()
    if dev.type == "cuda":
        torch.cuda.synchronize()
    worst = 0.0
    if bf16 and phenaki.critic is not None:
        # the sampled predictions (an argmax over noisy bf16-product logits) may differ from the fp32 run, and with them
        # the critic's inputs: only the generator half is comparable
        print("  (bf16: critic half not compared -- its inputs are sampled from the logits)")
    torch.testing.assert_close(loss.detach().cpu(), g["loss"], rtol=5e-2 if bf16 else 1e-4, atol=1e-5)

    def compare(module, ref_grads, who):
        nonlocal worst
        named = dict(module.named_parameters())
        for k, p in named.items():
            if k not in ref_grads:
                assert p.grad is None, f"{who}.{k}: the reference leaves this gradient unset"
                continue
            assert p.grad is not None, f"{who}.{k}: no gradient"
            ref = ref_grads[k]
            got = p.grad.detach().cpu()
            if ref.numel() == 0:
                assert got.shape == ref.shape
                continue
            scale = max(ref.abs().max().item(), 1e-12)
            err = (got - ref).abs().max().item() / scale
            if scale > 1e-7:  # (gradients that are zero in exact arithmetic, e.g. the softmax-invariant bias shift, are ~1e-9 noise)
                worst = max(worst, err)
            if verbose:
                print(f"  {who}.{k:60s} max|ref| {scale:.3e}  max err / max|ref| {err:.2e}")
            if bf16:
                assert scale < 1e-7 or err < 5e-2, f"{who}.{k}: max err / max|ref| = {err:.3e}"
            else:
                torch.testing.assert_close(got, ref, rtol=2e-3, atol=2e-4 * scale + 1e-7, msg=lambda m, k=k: f"{who}.{k}: {m}")

    if not (bf16 and case.get("self_critic")):
        compare(phenaki.maskgit, g["maskgit_grads"], "maskgit")
    if critic is not None and not bf16:
        compare(phenaki.critic, g["critic_grads"], "critic")
    if case.get("self_critic") and not bf16:
        compare(phenaki.critic.to_pred[0], g["to_pred_grads"], "to_pred")
    print(f"TRAIN_OK {name}{' bf16' if bf16 else ''} loss {loss.item():.6f} worst relative gradient error {worst:.2e}")


def check_frame_mask_case(device="cuda:0", verbose=False):
    """Phenaki.forward(videos, video_frame_mask=...) (phenaki_pytorch.py:587-612): raw videos tokenised live, frame
    mask -> token mask, CE + TokenCritic BCE; loss and every gradient against the reference's autograd
    (tests/golden/train_frame_mask.pt)."""
    case = C.FRAME_MASK_TRAIN_CASE
    g = torch.load(os.path.join(ROOT, "tests", "golden", "train_frame_mask.pt"), weights_only=False)
    torch.manual_seed(case["seed"])
    cvivit = P.CViViT(**C.SAMPLE_CVIVIT)
    maskgit = P.MaskGit(**case["maskgit"])
    critic = P.TokenCritic(**case["critic"])
    assert C.state_digest(maskgit.state_dict()) == g["maskgit_digest"]
    assert C.state_digest(critic.state_dict()) == g["critic_digest"]
    dev = torch.device(device)
    phenaki = P.Phenaki(cvivit=cvivit, maskgit=maskgit, critic=critic, steps=case["steps"],
                        text_embed_dim=case["maskgit"]["dim_context"]).to(dev).train()
    videos = C.seeded_randn(case["video"], case["input_seed"])
    ctx = C.synthetic_text_embeds(case["batch"], case["ctx_len"], case["maskgit"]["dim_context"], case["ctx_valid"],
                                  case["input_seed"] + 1000)
    fmask = C.frame_mask_of(case["frames_valid"], case["video"][2])
    b, n = g["ids"].shape[0], g["ids"][0].numel()
    torch.manual_seed(case["noise_seed"])
    rand_step, u = O.train_draws(b, n, case["steps"])
    draws = {"rand_step": rand_step, "perm": u,
             "gumbel": torch.zeros((b, n, case["maskgit"]["num_tokens"])).uniform_(0, 1)}
    loss = phenaki(videos.to(dev), text_embeds=ctx.to(dev), video_frame_mask=fmask.to(dev),
                   draw_fn=lambda shape, tag: draws[tag])
    loss.backward()
    torch.testing.assert_close(loss.detach().cpu(), g["loss"], rtol=1e-4, atol=1e-5)
    worst = 0.0
    for who, module, ref_grads in (("maskgit", phenaki.maskgit, g["maskgit_grads"]), ("critic", phenaki.critic, g["critic_grads"])):
        for k, p in module.named_parameters():
            if k not in ref_grads:
                assert p.grad is None, f"{who}.{k}: the reference leaves this gradient unset"
                continue
            assert p.grad is not None, f"{who}.{k}: no gradient"
            ref, got = ref_grads[k], p.grad.detach().cpu()
            if ref.numel() == 0:
                continue
            scale = max(ref.abs().max().item(), 1e-12)
            if scale > 1e-7:
                worst = max(worst, (got - ref).abs().max().item() / scale)
            torch.testing.assert_close(got, ref, rtol=2e-3, atol=2e-4 * scale + 1e-7, msg=lambda m, k=k: f"{who}.{k}: {m}")
    print(f"TRAIN_OK frame_mask loss {loss.item():.6f} worst relative gradient error {worst:.2e}")


if __name__ == "__main__":
    args = [a for a in sys.argv[1:] if a != "--bf16"]
    for nm in args or list(C.TRAIN_CASES):
        check_case(nm, bf16="--bf16" in sys.argv)
