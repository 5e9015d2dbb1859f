"""GPU: ``Phenaki.forward(video_codebook_ids=ids, text_embeds=e).backward()`` fills ``e.grad``
(phk_maskgit_train_step's d_context).

``e.grad`` and every parameter gradient are held to the float64 reference of tests/text_grad_cases.py -- fp32 mode at
the parity bars of tests/test_gpu_train_at_size.py, bf16 mode within 5 % of each tensor's largest entry -- for MaskGit
alone, with a cross-attention TokenCritic, with a SelfCritic, for ``only_train_generator`` / ``only_train_critic``, with
``video_frame_mask``, with attention and FF dropout (masks rebuilt from the counters the steps drew), and at the
configs[3] shape.  The fp32 product also matches the unmodified reference's golden.  Asking for ``e.grad`` leaves the
loss bit for bit as it was, the parameter gradients up to the order of their atomic adds, and issues the same library
launches; the gradient is deterministic,
accumulates over steps, is not all-reduced, and ``create_graph=True`` is refused.

The file sorts after the files that compare in-process ``torch.profiler`` traces (see tests/test_gpu_zz_encode_backward.py);
its own trace is taken in a child process."""
import json
import os
import subprocess
import sys

import pytest
import torch

from phenaki_pytorch_b200 import _lib as L
from phenaki_pytorch_b200 import sharding
from tests import cases as C
from tests import text_grad_cases as TG

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _set_precision(phenaki, precision):
    phenaki.maskgit.precision = precision
    if isinstance(phenaki.critic, TG.P.TokenCritic):
        phenaki.critic.precision = precision


@pytest.mark.parametrize("precision", [L.PREC_F32, L.PREC_BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("name,dropout,mode", [
    ("generator", 0.0, None), ("token_critic", 0.0, None), ("self_critic", 0.0, None),
    ("token_critic", 0.0, "only_train_generator"), ("token_critic", 0.0, "only_train_critic"),
    ("self_critic", 0.0, "only_train_critic"), ("generator", 0.2, None), ("token_critic", 0.2, None),
    ("self_critic", 0.2, None)])
def test_text_grad_matches_fp64_autograd(name, dropout, mode, precision):
    case = TG.SMALL[name]
    phenaki = TG.build(case, dropout=dropout, device=DEV)
    _set_precision(phenaki, precision)
    kw = {mode: True} if mode else {}
    loss, grads, e_grad, ref = TG.run_and_reference(case, phenaki, TG.decisive_draws(case), **kw)
    worst = TG.check(name, loss, grads, e_grad, ref, bf16=precision == L.PREC_BF16)
    assert TG.padded_rows_are_zero(e_grad, C.train_inputs(case)[1])
    print(f"\nTEXT_GRAD {name} dropout {dropout} {mode} prec {precision}: worst {worst:.3e}")


@pytest.mark.parametrize("precision", [L.PREC_F32, L.PREC_BF16], ids=["f32", "bf16"])
def test_text_grad_at_the_configs3_shape(precision):
    case = TG.AT_SIZE_CASE
    phenaki = TG.build(case, device=DEV)
    _set_precision(phenaki, precision)
    loss, grads, e_grad, ref = TG.run_and_reference(case, phenaki, TG.decisive_draws(case), ref_device=DEV)
    worst = TG.check("configs3", loss, grads, e_grad, ref, bf16=precision == L.PREC_BF16)
    assert TG.padded_rows_are_zero(e_grad, C.train_inputs(case)[1])
    print(f"\nTEXT_GRAD configs[3] prec {precision}: worst {worst:.3e}")


@pytest.mark.parametrize("precision", [L.PREC_F32, L.PREC_BF16], ids=["f32", "bf16"])
def test_text_grad_with_a_video_frame_mask(precision):
    case = dict(C.FRAME_MASK_TRAIN_CASE, critic_kind="token")
    phenaki = TG.build(case, device=DEV)
    _set_precision(phenaki, precision)
    videos = C.seeded_randn(case["video"], case["input_seed"]).to(DEV)
    fmask = C.frame_mask_of(case["frames_valid"], case["video"][2]).to(DEV)
    ctx = C.train_inputs(case)[1]
    with torch.no_grad():
        ids = phenaki.cvivit(videos, return_only_codebook_ids=True)
        vmask = phenaki.cvivit.calculate_video_token_mask(videos, video_frame_mask=fmask)
    assert not bool(vmask.all())
    draws = TG.decisive_draws(case)
    e = ctx.to(DEV).requires_grad_()
    loss = phenaki(videos, text_embeds=e, video_frame_mask=fmask, draw_fn=lambda shape, tag: draws[tag].to(DEV))
    loss.backward()
    ref = TG.reference(phenaki, ids.cpu(), ctx, draws, video_mask=vmask.cpu())
    TG.check("frame_mask", loss.detach().cpu(), TG.product_grads(phenaki), e.grad.cpu(), ref,
             bf16=precision == L.PREC_BF16)


@pytest.mark.parametrize("name", ["token_critic", "self_critic"])
def test_text_grad_matches_the_reference_golden(golden, name):
    g = TG.golden_case(golden, name)
    phenaki = TG.build(TG.SMALL[name], device=DEV)
    if g["to_pred"] is not None:
        phenaki.critic.to_pred.load_state_dict(g["to_pred"])
    loss, grads, e_grad = TG.product(phenaki, g["ids"], g["text_embeds"], g["draws"])
    torch.testing.assert_close(loss, g["loss"], rtol=1e-4, atol=1e-5)
    for k, want in dict(g["grads"], text_embeds=g["text_embeds_grad"]).items():
        got = e_grad if k == "text_embeds" else grads[k]
        if want.numel():
            torch.testing.assert_close(got, want, rtol=2e-3, atol=2e-4 * float(want.abs().max()) + 1e-7,
                                       msg=lambda m, k=k: f"{k}: {m}")
    assert TG.padded_rows_are_zero(e_grad, g["text_embeds"])


@pytest.mark.parametrize("precision", [L.PREC_F32, L.PREC_BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("name", ["token_critic", "self_critic"])
def test_loss_and_parameter_gradients_do_not_depend_on_the_text_grad(name, precision):
    """The loss is bit-identical with and without ``e.grad``.  Several parameter gradients (LayerNorm gammas, q/k scales,
    null keys, embeddings, PEG) are reduced with atomic adds, so two identical steps repeat them only up to the order of
    those adds, with or without ``e.grad``: each gradient is held to 1e-6 of the largest, the bar of
    tests/test_gpu_train_dropout.py.  ``e.grad`` itself is reduced without atomics and repeats bit for bit."""
    case = TG.SMALL[name]
    phenaki = TG.build(case, device=DEV)
    _set_precision(phenaki, precision)
    ids, ctx = C.train_inputs(case)
    draws = TG.decisive_draws(case)
    l0, g0, e0 = TG.product(phenaki, ids, ctx, draws, requires_grad=False)
    l1, g1, e1 = TG.product(phenaki, ids, ctx, draws)
    l2, g2, e2 = TG.product(phenaki, ids, ctx, draws)
    assert e0 is None and e1 is not None
    assert torch.equal(l0, l1) and torch.equal(l1, l2)
    top = max(float(g.abs().max()) for g in g0.values() if g is not None and g.numel())
    for k, g in g0.items():
        assert (g is None) == (g1[k] is None), k
        if g is not None and g.numel():
            assert float((g - g1[k]).abs().max()) <= 1e-6 * top, k
    assert torch.equal(e1, e2), "e.grad differs between two identical steps"


def test_text_grad_accumulates_over_two_steps():
    case = TG.SMALL["token_critic"]
    phenaki = TG.build(case, device=DEV)
    ids, ctx = C.train_inputs(case)
    draws = TG.decisive_draws(case)
    _, _, once = TG.product(phenaki, ids, ctx, draws)
    e = ctx.to(DEV).requires_grad_()
    for _ in range(2):
        phenaki(video_codebook_ids=ids.to(DEV), text_embeds=e, draw_fn=lambda shape, tag: draws[tag].to(DEV)).backward()
    assert torch.equal(e.grad.cpu(), once + once)


def test_create_graph_is_refused():
    case = TG.SMALL["token_critic"]
    phenaki = TG.build(case, device=DEV)
    ids, ctx = C.train_inputs(case)
    draws = TG.decisive_draws(case)
    e = ctx.to(DEV).requires_grad_()
    loss = phenaki(video_codebook_ids=ids.to(DEV), text_embeds=e, draw_fn=lambda shape, tag: draws[tag].to(DEV))
    with pytest.raises(RuntimeError, match="create_graph"):
        torch.autograd.grad(loss, [e], create_graph=True)


# ---------------------------------------------------------------- child processes
def launches_and_kernels():
    """{precision: {requires_grad: (phk_launch_count delta, device op names)}} of one MaskGit + TokenCritic training
    step (forward + backward) at the configs[3] shape, after a warm-up step of each."""
    from torch.profiler import ProfilerActivity, profile
    lib = L.lib()
    case = TG.AT_SIZE_CASE
    phenaki = TG.build(case, device=DEV)
    ids, ctx = C.train_inputs(case)
    draws = {k: v.to(DEV) for k, v in TG.decisive_draws(case).items()}
    ids, ctx = ids.to(DEV), ctx.to(DEV)

    def step(requires_grad):
        e = ctx.clone().requires_grad_(requires_grad)
        phenaki.zero_grad(set_to_none=True)
        phenaki(video_codebook_ids=ids, text_embeds=e, draw_fn=lambda shape, tag: draws[tag]).backward()
        torch.cuda.synchronize()

    out = {}
    for prec in (L.PREC_F32, L.PREC_BF16):
        _set_precision(phenaki, prec)
        res = {}
        for rg in (False, True):
            step(rg)
            before = lib.phk_launch_count()
            step(rg)
            count = lib.phk_launch_count() - before
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                step(rg)
            ops = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
            res[str(rg)] = (count, [e.name for e in sorted(ops, key=lambda e: e.time_range.start)])
        out[str(prec)] = res
    return out


def _child(fn):
    code = (f"import json, sys; sys.path.insert(0, {ROOT!r}); from tests import test_gpu_zz_train_text_grad as T; "
            f"print(json.dumps(T.{fn}()))")
    flags = ["-s"] if sys.flags.no_user_site else []
    run = subprocess.run([sys.executable, *flags, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert run.returncode == 0, run.stderr[-4000:]
    return json.loads(run.stdout.strip().splitlines()[-1])


def test_launches_and_kernel_sequence_do_not_depend_on_the_text_grad():
    """The train step issues the same launches whether or not it writes d_context; the rest of the step (the added
    gradient scaling is one elementwise op per input that wants a gradient) is torch's.  The comparison is of the
    library's launch count and of the library's kernels in the trace."""
    res = _child("launches_and_kernels")
    for prec, r in res.items():
        (c0, ops0), (c1, ops1) = r["False"], r["True"]
        assert c0 == c1 and c0 > 0, f"prec {prec}: {c0} launches without e.grad, {c1} with"
        lib0 = [o for o in ops0 if "phk::" in o]
        lib1 = [o for o in ops1 if "phk::" in o]
        assert lib0, f"prec {prec}: no library kernel in the trace"
        # the profiler may drop a trace's first record
        assert lib1 == lib0 or lib1[1:] == lib0 or lib1 == lib0[1:], f"prec {prec}: the library kernels differ"


def sync_one_rank():
    """One-rank NCCL group with the overlapped all-reduce: (overlap ran, e.grad equal to the unsynced run's,
    parameter gradients' largest difference over the largest gradient)."""
    import torch.distributed as dist
    port = 29000 + os.getpid() % 2000
    dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1,
                            device_id=torch.device(DEV))
    sharding.OVERLAP_AT_WORLD_SIZE_1 = True
    real, seen = sharding.launch_overlapped_all_reduce, []

    def launch(flat, plan, groups):
        seen.append(flat.numel())
        return real(flat, plan, groups)

    sharding.launch_overlapped_all_reduce = launch
    try:
        case = TG.SMALL["token_critic"]
        phenaki = TG.build(case, device=DEV)
        ids, ctx = C.train_inputs(case)
        draws = TG.decisive_draws(case)
        runs = {}
        for sync in (False, True):
            phenaki.sync_gradients = sync
            runs[sync] = TG.product(phenaki, ids, ctx, draws)
        g0, g1 = runs[False][1], runs[True][1]
        top = max(float(g.abs().max()) for g in g0.values() if g is not None and g.numel())
        diff = max(float((g1[k] - g).abs().max()) for k, g in g0.items() if g is not None and g.numel())
        return dict(ran=len(seen) == 2, e_equal=torch.equal(runs[False][2], runs[True][2]), rel_diff=diff / top)
    finally:
        dist.destroy_process_group()


def test_sync_gradients_in_a_one_rank_nccl_group_leaves_the_text_grad_per_rank():
    res = _child("sync_one_rank")
    assert res["ran"], "the overlapped all-reduce did not run for both steps"
    assert res["e_equal"], "e.grad changed under sync_gradients"
    assert res["rel_diff"] <= 1e-6, res
