"""Generates tests/golden/cvivit_recon_loss.pt by running the UNMODIFIED reference (imported from /root/reference with
the stubs of oracle/reference_loader.py) through ``loss = CViViT(video, mask); loss.backward()`` with
use_vgg_and_gan=False, in training mode and in eval mode, on the CPU in float32 (the reference builds float32 tensors
internally, so it does not run in float64).

The stub's LFQ (oracle/lfq.py) restates upstream's eval-mode arithmetic only; here it is extended by upstream's
training-mode straight-through estimator, ``quantized = x + (quantized - x).detach()``, which is what the reference's
CViViT calls in training mode.

Per case and mode the file records the loss, the CPU generator's next torch.randn(4) after the call (the reference draws
pick_frame_logits before it returns), and a fingerprint of every parameter gradient and of video.grad: None, or (shape,
sum of squares, the dot products with 4 seeded random vectors, see ``fingerprint``).  Fingerprints keep the fixture small
while pinning every entry.  tests/test_recon_loss_golden_cpu.py checks the oracle composition against it.

Run in the build container only:   python tests/golden/make_recon_golden.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import lfq  # noqa: E402
from oracle.reference_loader import load_reference  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cvivit_recon_loss.pt")

# name -> (module seed, ctor, video shape, video seed, frame mask rows or None)
CASES = {
    "cfg1": (0, dict(dim=256, codebook_size=65536, image_size=64, patch_size=16, temporal_patch_size=2, spatial_depth=2,
                     temporal_depth=2, use_vgg_and_gan=False), (1, 3, 5, 64, 64), 1, None),
    "image": (5, dict(dim=64, codebook_size=256, image_size=32, patch_size=8, temporal_patch_size=2, spatial_depth=1,
                      temporal_depth=1, dim_head=32, heads=2, channels=1, use_vgg_and_gan=False), (3, 1, 32, 32), 6, None),
    "rect_mask": (3, dict(dim=128, codebook_size=1024, image_size=(32, 48), patch_size=(8, 16), temporal_patch_size=3,
                          spatial_depth=1, temporal_depth=2, dim_head=32, heads=4, use_vgg_and_gan=False),
                  (2, 3, 7, 32, 48), 4, [[1, 1, 1, 1, 0, 0, 0], [1] * 7]),
}
RNG_SEED = 77


def fingerprint(g, key):
    """None, or (shape, sum of squares, dot products with 4 standard-normal vectors drawn from seed `key`) in float64."""
    if g is None:
        return None
    flat = g.detach().double().flatten()
    r = torch.randn((4, flat.numel()), generator=torch.Generator().manual_seed(key), dtype=torch.float64)
    return tuple(g.shape), float(flat.square().sum()), (r @ flat).tolist()


class TrainingLFQ(lfq.LFQ):
    """Upstream LFQ's forward with its straight-through estimator in training mode (no entropy aux loss: the
    use_vgg_and_gan=False loss does not include it)."""

    def forward(self, x, **unused):
        x = self.project_in(x)
        positive = x > 0
        quantized = torch.where(positive, self.codebook_scale, -self.codebook_scale).to(x.dtype)
        indices = (positive.int() * self.mask.int()).sum(dim=-1)
        if self.training:
            quantized = x + (quantized - x).detach()
        return self.project_out(quantized), indices, torch.zeros((), device=x.device)


def main():
    load_reference()
    import phenaki_pytorch.cvivit as RC
    RC.LFQ = TrainingLFQ
    out = {}
    for name, (seed, ctor, shape, vseed, mask) in CASES.items():
        for training in (True, False):
            torch.manual_seed(seed)
            model = RC.CViViT(**ctor).train(training)
            video = torch.randn(shape, generator=torch.Generator().manual_seed(vseed)).requires_grad_(True)
            m = None if mask is None else torch.tensor(mask, dtype=torch.bool)
            torch.manual_seed(RNG_SEED)
            loss = model(video, mask=m)
            after = torch.randn(4)
            loss.backward()
            names = sorted(n for n, _ in model.named_parameters())
            params = dict(model.named_parameters())
            grads = {n: fingerprint(params[n].grad, k) for k, n in enumerate(names)}
            out[f"{name}/{'train' if training else 'eval'}"] = dict(
                seed=seed, ctor=ctor, shape=shape, video_seed=vseed, mask=mask, loss=float(loss), randn_after=after,
                grads=grads, video_grad=fingerprint(video.grad, len(names)))
            print(name, "train" if training else "eval", float(loss), sum(g is None for g in grads.values()), "None")
    torch.save(out, OUT)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
