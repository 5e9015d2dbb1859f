"""Data-parallel C-ViViT training on two gloo ranks: each rank runs ``loss = cvivit(shard); loss.backward()`` on its
contiguous video shard with the whole product path on the CPU executor of tests/cuda_emu, in fp32 mode.

With ``sync_gradients = True`` every parameter gradient must be the mean over the ranks of the float64 oracle gradients of
each rank's own objective (``recon_loss_cases.cvivit_recon_loss`` on that rank's shard and frame mask, q from that rank's
ids), at the bars of tests/recon_loss_cases.py ``check_fp32``; ``video.grad`` must be the rank's own gradient.  With
``sync_gradients = False`` each rank's gradients must be bit-identical to a single-process run on the same shard."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests import recon_loss_cases as RL
from tests.decode_grad_cases import ANALYTICALLY_ZERO

WORLD = 2


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _global_batch(name):
    """(video, mask or None) of two videos: the case's own when it has two, else the case's video and a second one."""
    video, mask = RL.inputs(name)
    if video.shape[0] == 1:
        video = torch.cat([video, -video.flip(-1)])
    return video, mask


def _upstream(name, shape):
    return RL.upstream_weights(name, shape).to(torch.float32)


def _run(module, video, mask, training, with_recon, sync, name, rank):
    """({parameter name: gradient or None}, video.grad, ids) of the rank's objective."""
    module.train(training)
    module.sync_gradients = sync
    module.zero_grad(set_to_none=True)
    ids = module(video, return_only_codebook_ids=True)
    vid = video.clone().requires_grad_(True)
    if with_recon:
        loss, recon = module(vid, mask=mask, return_recons=True)
        g = _upstream(name, (WORLD * recon.shape[0], *recon.shape[1:]))
        lo = rank * recon.shape[0]
        RL._objective(loss, recon, g[lo:lo + recon.shape[0]]).backward()
    else:
        module(vid, mask=mask).backward()
    grads = {k: None if p.grad is None else p.grad.detach().clone() for k, p in module.named_parameters()}
    module.zero_grad(set_to_none=True)
    return grads, vid.grad.detach().clone(), ids


def _worker(rank, port, name, runs, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=WORLD)
    results = {}
    try:
        torch.set_num_threads(2)
        from phenaki_pytorch_b200 import sharding as S
        from tests import emu_runtime
        emu_runtime.route_product_to_emulator(emu_runtime.build_emu())
        module = RL.build_module(name)  # the same seeded weights on every rank
        video, mask = _global_batch(name)
        mine, my_mask = S.shard_batch(video), None if mask is None else S.shard_batch(mask)
        for run in runs:
            training, with_recon, sync = run
            results[run] = _run(module, mine, my_mask, training, with_recon, sync, name, rank)
        dist.barrier()
    finally:
        dist.destroy_process_group()
    # the same shard in a single process (no process group): what sync_gradients=False must reproduce bit for bit
    for run in runs:
        training, with_recon, sync = run
        if not sync:
            results[("single",) + run] = _run(module, mine, my_mask, training, with_recon, False, name, rank)
    torch.save(results, f"{out}.{rank}")


def _reference(name, rank, training, with_recon, ids):
    """{parameter name | "video": float64 oracle gradient} of rank's objective (absent: the reference leaves None)."""
    from phenaki_pytorch_b200 import sharding as S
    module = RL.build_module(name)
    video, mask = _global_batch(name)
    lo, hi = S.shard_range(video.shape[0], rank, WORLD)
    video, mask = video[lo:hi], None if mask is None else mask[lo:hi]
    params = dict(module.named_parameters())
    sd = {}
    for k, v in module.state_dict().items():
        v = v.detach().to(torch.float64) if v.is_floating_point() else v.detach()
        sd[k] = v.requires_grad_(True) if k in params else v
    vid = video.to(torch.float64).requires_grad_(True)
    loss, recon = RL.cvivit_recon_loss(vid, sd, module.image_size, module.patch_size, mask, training, codes_from_ids=ids)
    g = None
    if with_recon:
        g = _upstream(name, (WORLD * recon.shape[0], *recon.shape[1:]))[lo:hi].double()
    RL._objective(loss, recon, g).backward()
    grads = {k: sd[k].grad for k in params if sd[k].grad is not None}
    for k, p in params.items():  # self-attention null_kv (heads, 0, dim_head): autograd hands it an empty gradient
        if p.numel() == 0 and (training or not k.startswith(RL.ENCODER_PREFIXES)):
            grads[k] = torch.zeros_like(sd[k])
    grads["video"] = vid.grad
    return grads


def _assert_close(label, got, want, top):
    """check_fp32's bars: 1e-4 of the tensor's largest entry and 2e-5 relative Frobenius error; the analytically zero
    gradient within 1e-6 of the largest gradient."""
    if want.numel() == 0:
        return
    assert got.shape == want.shape, label
    err = (got.double() - want).abs().max().item()
    if label.split(" ")[-1] in ANALYTICALLY_ZERO:
        assert err <= 1e-6 * top, f"{label}: {err:.3e} above 1e-6 x the largest gradient {top:.3e}"
        return
    scale = want.abs().max().item()
    if scale == 0.0:
        assert err == 0.0, f"{label}: {err:.3e} where the reference is exactly zero"
        return
    fro = ((got.double() - want).norm() / want.norm()).item()
    assert err <= 1e-4 * scale and fro <= 2e-5, f"{label}: max err / max|ref| {err / scale:.3e}, Frobenius {fro:.3e}"


# name -> runs (training, with_recon, sync_gradients)
CASES = {
    "cfg1": [(True, False, True)],
    "rect": [(True, False, True), (True, True, True), (True, False, False)],
    "rect_mask": [(True, False, True), (False, False, True), (False, False, False)],
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_two_rank_gloo_recon_loss_gradients(tmp_path, name):
    runs = CASES[name]
    out = str(tmp_path / "r")
    mp.spawn(_worker, args=(_free_port(), name, runs, out), nprocs=WORLD, join=True)
    res = [torch.load(f"{out}.{r}") for r in range(WORLD)]
    for run in runs:
        training, with_recon, sync = run
        what = f"{name} training={training} return_recons={with_recon} sync_gradients={sync}"
        refs = [_reference(name, r, training, with_recon, res[r][run][2]) for r in range(WORLD)] if sync else None
        for r in range(WORLD):
            grads, vgrad, _ = res[r][run]
            if not sync:  # each rank on its own: bit for bit what one process computes on that shard
                single, single_v, _ = res[r][("single",) + run]
                assert grads.keys() == single.keys()
                for k, g in grads.items():
                    assert (g is None) == (single[k] is None) and (g is None or torch.equal(g, single[k])), \
                        f"{what} rank {r}: {k} differs from the single-process run"
                assert torch.equal(vgrad, single_v), f"{what} rank {r}: video.grad differs from the single-process run"
                continue
            want_none = {k for k in grads if k not in refs[0]}
            assert {k for k, g in grads.items() if g is None} == want_none, f"{what}: None set"
            if not training:
                assert all(grads[k] is None for k in grads if k.startswith(RL.ENCODER_PREFIXES)), what
            mean = {k: sum(ref[k] for ref in refs) / WORLD for k in refs[0] if k != "video"}
            top = max(float(g.abs().max()) for g in mean.values() if g.numel())
            for k, g in grads.items():
                if g is not None:
                    _assert_close(f"{what} rank {r} {k}", g, mean[k], top)
            _assert_close(f"{what} rank {r} video.grad", vgrad, refs[r]["video"], float(refs[r]["video"].abs().max()))
            # every rank holds the same averaged gradients
            other = res[1 - r][run][0]
            assert all(g is None or torch.equal(g, other[k]) for k, g in grads.items()), f"{what}: ranks disagree"
