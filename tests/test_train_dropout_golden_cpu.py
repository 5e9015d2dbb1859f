"""CPU: the dropout-aware training loss of tests/dropout_ref.py against the reference's autograd with dropout
(tests/golden/train_dropout.pt, written by tests/golden/make_dropout_golden.py from the unmodified reference with each
nn.Dropout replaced by the stored masks): loss and every gradient within fp32 summation order.  The stored masks are the
ones the counter contract gives for the stored (seed, offset)."""
import torch

from tests import dropout_ref as DR
from tests import train_at_size_cases as T
from tests import train_dropout_cases as TD


def _fixture(golden):
    return golden("train_dropout")


def test_stored_masks_are_the_contract_masks(golden):
    g = _fixture(golden)
    c = TD.case(g["case"], g["attn_p"], g["ff_p"])
    x = T.inputs(c)
    b, n = x["ids"].shape
    rebuilt = DR.step_masks(T.build_module(c), b, n, c["ctx_len"], g["seed"], g["offset"], g["attn_p"], g["ff_p"],
                            torch.float32)
    for want, got in zip(g["masks"], rebuilt):
        for site in ("self", "cross", "ff"):
            assert torch.equal(want[site], got[site]), site


def test_restatement_with_masks_matches_the_reference_loss_and_gradients(golden):
    g = _fixture(golden)
    c = TD.case(g["case"], g["attn_p"], g["ff_p"])
    x = T.inputs(c)
    sd = {k: (v.clone().requires_grad_(True) if k in g["grads"] else v.clone()) for k, v in g["state_dict"].items()}
    loss = DR.maskgit_train_loss(x["ids"], sd, x["token_mask"], video_patch_shape=c["patch_shape"],
                                 heads=c["ctor"]["heads"], context=x["context"], text_mask=x["text_mask"],
                                 masks=g["masks"])
    loss.backward()
    torch.testing.assert_close(loss.detach(), g["loss"], rtol=1e-5, atol=1e-5)
    for k, want in g["grads"].items():
        torch.testing.assert_close(sd[k].grad, want, rtol=1e-5, atol=1e-5, msg=lambda m, k=k: f"{k}: {m}")
    # the masks matter: without them the same weights give another loss
    plain = DR.maskgit_train_loss(x["ids"], sd, x["token_mask"], video_patch_shape=c["patch_shape"],
                                  heads=c["ctor"]["heads"], context=x["context"], text_mask=x["text_mask"])
    assert not torch.allclose(plain.detach(), g["loss"], rtol=1e-5, atol=1e-5)
