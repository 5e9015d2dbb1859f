"""Generates tests/golden/train_text_grad.pt: the training loss of the UNMODIFIED reference's ``Phenaki.forward``
(phenaki_pytorch.py:562-687) with ``text_embeds.requires_grad_()`` and what its autograd gives for ``text_embeds``.
Cases: MaskGit + a cross-attention TokenCritic, MaskGit + SelfCritic (the networks, inputs, padded text rows and noise
seeds of tests/cases.py TRAIN_CASES).  The reference draws from the global CPU generator;
tests/text_grad_cases.py::reference_draws replays them, and this script checks that it does.

The parameter gradients of the same run are those tests/golden/make_golden.py stored in train_with_critic.pt and
train_self_critic.pt (a gradient of the parameters does not depend on whether the embeddings require grad): this
script checks that they are bit for bit the same and does not store them again.

In the same pass the float32 run of the composition in tests/text_grad_cases.py is pinned against the reference (within
fp32 summation order, as tests/golden/make_golden.py does), otherwise this script aborts.

Run in the build container only:   python tests/golden/make_text_grad_golden.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import phenaki_oracle as O  # noqa: E402
from oracle.reference_loader import load_reference  # noqa: E402
from tests import cases as C  # noqa: E402
from tests import text_grad_cases as TG  # noqa: E402
from tests.golden.make_golden import same  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
GOLDEN_CASES = ("token_critic", "self_critic")


def named_grads(phenaki):
    """{name: gradient} of the reference modules, named as tests/text_grad_cases.py names them."""
    out = {f"maskgit.{k}": p.grad for k, p in phenaki.maskgit.named_parameters() if p.grad is not None}
    critic = phenaki.critic
    if critic is not None and hasattr(critic, "to_pred"):
        out.update({f"critic.to_pred.0.{k}": p.grad for k, p in critic.to_pred[0].named_parameters() if p.grad is not None})
    elif critic is not None:
        out.update({f"critic.{k}": p.grad for k, p in critic.named_parameters() if p.grad is not None})
    return {k: v.detach().clone() for k, v in out.items()}


def main():
    ref = load_reference()
    gold = {}
    for name in GOLDEN_CASES:
        case = TG.SMALL[name]
        print(f"[train_text_grad/{name}]")
        torch.manual_seed(case["seed"])
        cvivit = ref.CViViT(**C.SAMPLE_CVIVIT)
        maskgit = ref.MaskGit(**case["maskgit"])
        critic = ref.TokenCritic(**case["critic"]) if case["critic_kind"] == "token" else None
        phenaki = ref.Phenaki(cvivit=cvivit, maskgit=maskgit, critic=critic, steps=case["steps"],
                              self_token_critic=case["critic_kind"] == "self",
                              text_embed_dim=case["maskgit"]["dim_context"]).train()
        ids, ctx = C.train_inputs(case)
        b, n, V = ids.shape[0], ids[0].numel(), case["maskgit"]["num_tokens"]
        e = ctx.clone().requires_grad_()
        torch.manual_seed(case["noise_seed"])
        loss = phenaki(video_codebook_ids=ids, text_embeds=e)
        loss.backward()
        assert e.grad is not None, "the reference gave the text embeddings no gradient"
        # the draws it took, replayed in its order from the same generator state
        torch.manual_seed(case["noise_seed"])
        rand_step, perm = O.train_draws(b, n, case["steps"])
        draws = TG.reference_draws(case)
        same(draws["rand_step"], rand_step, "draw rand_step")
        same(draws["perm"], perm, "draw perm")
        if case["critic_kind"] is not None:
            same(draws["gumbel"], torch.zeros((b, n, V)).uniform_(0, 1), "draw gumbel")
        grads = named_grads(phenaki)
        tr = torch.load(os.path.join(OUT, f"train_{TG.GOLDEN_SOURCE[name]}.pt"), weights_only=False)
        stored = TG.golden_parameter_grads(tr)
        assert set(stored) == set(grads), set(stored) ^ set(grads)
        for k, g in grads.items():
            same(stored[k], g, f"stored d loss / d {k}")
        if case["critic_kind"] == "self":
            same(tr["to_pred_weight"], phenaki.critic.to_pred[0].weight.detach(), "stored to_pred.weight")
            same(tr["to_pred_bias"], phenaki.critic.to_pred[0].bias.detach(), "stored to_pred.bias")

        # pin the composition (float32, same weights and draws)
        mine = TG.build(case)
        assert C.state_digest(mine.maskgit.state_dict()) == C.state_digest(maskgit.state_dict())
        if critic is not None:
            assert C.state_digest(mine.critic.state_dict()) == C.state_digest(critic.state_dict())
        if case["critic_kind"] == "self":
            mine.critic.to_pred.load_state_dict(phenaki.critic.to_pred.state_dict())
        r = TG.reference(mine, ids, ctx, draws, dtype=torch.float32)
        same(r["losses"]["loss"], loss.detach(), "training loss")
        assert set(r["grads"]) == set(grads) | {"text_embeds"}, set(r["grads"]) ^ (set(grads) | {"text_embeds"})
        for k, g in grads.items():
            same(r["grads"][k], g, f"d loss / d {k}")
        same(r["grads"]["text_embeds"], e.grad, "d loss / d text_embeds")
        gold[name] = dict(loss=loss.detach().clone(), text_embeds_grad=e.grad.detach().clone())
    torch.save(gold, os.path.join(OUT, "train_text_grad.pt"))
    print("wrote", os.path.join(OUT, "train_text_grad.pt"))


if __name__ == "__main__":
    main()
