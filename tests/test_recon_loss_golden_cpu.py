"""CPU: the oracle composition of the reconstruction loss (tests/recon_loss_cases.py::cvivit_recon_loss, the float64
reference of the GPU and emulated tests) against tests/golden/cvivit_recon_loss.pt, which the UNMODIFIED reference wrote
in training and eval mode (tests/golden/make_recon_golden.py).  This pins the composition's rearranges, the frame-mask
indexing, the straight-through estimator, the set of parameters left without a gradient and the CPU random draw against
the real reference.  The composition runs in float32 here, as the reference did, with q = sign(x) of its own."""
import os

import pytest
import torch

from tests import recon_loss_cases as RL
from tests.golden.make_recon_golden import fingerprint

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cvivit_recon_loss.pt")
KEYS = ["cfg1/train", "cfg1/eval", "image/train", "image/eval", "rect_mask/train", "rect_mask/eval"]


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN, weights_only=False)


def _close(got, want, what):
    """Fingerprints within 1e-4 of the gradient's norm (fp32 summation order)."""
    assert (got is None) == (want is None), f"{what}: None {got is None}, reference None {want is None}"
    if want is None:
        return
    assert got[0] == want[0], what
    norm = want[1] ** 0.5
    assert abs(got[1] - want[1]) <= 2e-4 * want[1] + 1e-30, f"{what}: sum of squares {got[1]} vs {want[1]}"
    for a, b in zip(got[2], want[2]):
        assert abs(a - b) <= 1e-4 * norm + 1e-30, f"{what}: projection {a} vs {b} (norm {norm})"


@pytest.mark.parametrize("key", KEYS)
def test_oracle_recon_loss_matches_the_reference(golden, key):
    g = golden[key]
    training = key.endswith("/train")
    torch.manual_seed(g["seed"])
    module = RL.P.CViViT(**g["ctor"])
    params = dict(module.named_parameters())
    sd = {k: (v.detach().requires_grad_(True) if k in params else v) for k, v in module.state_dict().items()}
    video = torch.randn(g["shape"], generator=torch.Generator().manual_seed(g["video_seed"])).requires_grad_(True)
    mask = None if g["mask"] is None else torch.tensor(g["mask"], dtype=torch.bool)
    torch.manual_seed(77)
    loss, _ = RL.cvivit_recon_loss(video, sd, module.image_size, module.patch_size, mask, training)
    torch.randn(video.shape[0], 1 if video.ndim == 4 else video.shape[2])  # the reference's pick_frame_logits draw
    assert torch.equal(torch.randn(4), g["randn_after"]), "the reference draws torch.randn(b, f) once before it returns"
    assert abs(float(loss.detach()) - g["loss"]) <= 1e-5 * g["loss"], (float(loss.detach()), g["loss"])
    loss.backward()
    names = sorted(params)
    t = 1 if video.ndim == 4 else 1 + (video.shape[2] - 1) // module.temporal_patch_size
    for k, n in enumerate(names):
        grad = sd[n].grad
        if grad is None and t == 1 and (n.startswith("to_pixels.") or (training and n.startswith("to_patch_emb."))):
            grad = torch.zeros_like(sd[n])  # the reference runs these on empty batches, the oracle returns before them
        if grad is None and sd[n].numel() == 0 and (training or not n.startswith(RL.ENCODER_PREFIXES)):
            grad = torch.zeros_like(sd[n])  # (heads, 0, dim_head) null_kv: autograd hands it an empty gradient
        _close(fingerprint(grad, k), g["grads"][n], f"{key} {n}")
    _close(fingerprint(video.grad, len(names)), g["video_grad"], f"{key} video")
