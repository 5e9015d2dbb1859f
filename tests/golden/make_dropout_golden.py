"""Generates tests/golden/train_dropout.pt: the MaskGit training loss (phenaki_pytorch.py:620-640) and every gradient of
the UNMODIFIED reference in training mode with attention and FF dropout, each nn.Dropout replaced by a multiplication
with a stored mask (the masks of the training step's counter contract, include/phk.h phk_dropout_t, at a fixed seed and
offset).  In the same pass it pins the dropout-aware restatement (tests/dropout_ref.py) against the reference: loss and
gradients within fp32 summation order (<= 1e-5), otherwise this script aborts, as tests/golden/make_golden.py does.

Run in the build container only:   python tests/golden/make_dropout_golden.py
"""
import math
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle.reference_loader import load_reference  # noqa: E402
from tests import dropout_ref as DR  # noqa: E402
from tests import train_at_size_cases as T  # noqa: E402
from tests import train_dropout_cases as TD  # noqa: E402
from tests.golden.make_golden import same  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
SEED, OFFSET = 20251015, 4096  # the (seed, first counter) whose masks the fixture stores


class _MaskMul(torch.nn.Module):
    """Stands in for one nn.Dropout: multiplies by the next stored mask (the calls come in the contract's site order)."""

    def __init__(self, feed):
        super().__init__()
        self.feed = feed

    def forward(self, x):
        m = next(self.feed)
        assert m.shape == x.shape, (m.shape, x.shape)
        return x * m


def main():
    ref = load_reference()
    c = TD.case("tiny")
    torch.manual_seed(c["seed"])
    maskgit = ref.MaskGit(**c["ctor"]).train()
    x = T.inputs(c)
    b, n = x["ids"].shape
    masks = DR.step_masks(T.build_module(c), b, n, c["ctx_len"], SEED, OFFSET, TD.ATTN_P, TD.FF_P, torch.float32)
    order = [m for layer in masks for m in (layer["self"], layer["cross"], layer["ff"]) if m is not None]
    feed = iter(order)
    for parent in list(maskgit.modules()):
        for name, child in list(parent.named_children()):
            if isinstance(child, torch.nn.Dropout):
                setattr(parent, name, _MaskMul(feed))
    masked = torch.where(x["token_mask"], maskgit.mask_id, x["ids"])
    logits = maskgit(masked, video_patch_shape=c["patch_shape"], text_mask=x["text_mask"], context=x["context"])
    loss = F.cross_entropy(logits[x["token_mask"]], x["ids"][x["token_mask"]])
    loss.backward()
    assert next(feed, None) is None, "the reference used fewer masks than the contract has sites"
    grads = {k: p.grad.detach().clone() for k, p in maskgit.named_parameters() if p.grad is not None}
    sd = {k: v.detach().clone() for k, v in maskgit.state_dict().items()}

    # pin the restatement: same weights, same masks
    leaf = {k: (v.clone().requires_grad_(True) if k in grads else v.clone()) for k, v in sd.items()}
    o_loss = DR.maskgit_train_loss(x["ids"], leaf, x["token_mask"], video_patch_shape=c["patch_shape"],
                                   heads=c["ctor"]["heads"], context=x["context"], text_mask=x["text_mask"],
                                   masks=masks)
    o_loss.backward()
    same(o_loss.detach(), loss.detach(), "training loss with dropout")
    for k, g in grads.items():
        same(leaf[k].grad, g, f"d loss / d {k}")
    torch.save(dict(case="tiny", seed=SEED, offset=OFFSET, attn_p=TD.ATTN_P, ff_p=TD.FF_P, state_dict=sd,
                    masks=masks, loss=loss.detach().clone(), grads=grads, n=n, patch=math.prod(c["patch_shape"])),
               os.path.join(OUT, "train_dropout.pt"))
    print("wrote", os.path.join(OUT, "train_dropout.pt"))


if __name__ == "__main__":
    main()
