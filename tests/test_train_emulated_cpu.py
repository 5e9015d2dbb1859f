"""CPU: the CUDA sources of the training step -- csrc/train.cu and the validated fp32 kernels it launches (rowops.cu,
gemm_simt.cu, attention.cu) -- compiled by g++ against tests/cuda_emu (every CUDA thread a fiber, __syncthreads / warp
shuffles as barriers) and EXECUTED on the CPU through the product's own Python path (MaskGit.train_step -> ctypes
tables -> phk_maskgit_train_step), against the reference's autograd loss and gradients (tests/golden/train_*.pt).
Every kernel of the fp32 step is the shipped source; the one stand-in is the wgmma GEMM of the bf16 mode (its
include/phk.h contract stated on the CPU).  That the GPU-validated forward kernels give the reference's numbers here
too is the evidence that the executor is faithful."""
import pytest
import torch

import phenaki_pytorch_b200 as P
from tests import cases as C

from tests import emu_runtime


@pytest.fixture(scope="module")
def emu():
    return emu_runtime.build_emu()


@pytest.fixture
def on_cpu(emu, monkeypatch):
    """Routes the product's host path to the emulated library with CPU tensors (test only)."""
    emu_runtime.route_product_to_emulator(emu, monkeypatch)


def _modules(case):
    torch.manual_seed(case["seed"])
    cvivit = P.CViViT(**C.SAMPLE_CVIVIT)
    maskgit = P.MaskGit(**case["maskgit"])
    critic = P.TokenCritic(**case["critic"]) if case["critic"] else None
    if case.get("self_critic"):  # built inside Phenaki's constructor, after the networks (same order as the reference)
        critic = P.Phenaki(cvivit=cvivit, maskgit=maskgit, self_token_critic=True,
                           text_embed_dim=case["maskgit"]["dim_context"]).critic
    return maskgit, critic


def _compare(module, gk, ref, who):
    for k, p in module.named_parameters():
        got = gk.grad_of(p)
        if k not in ref:
            assert got is None, f"{who}.{k}"
            continue
        if ref[k].numel() == 0:
            assert got.shape == ref[k].shape
            continue
        scale = max(ref[k].abs().max().item(), 1e-12)
        torch.testing.assert_close(got, ref[k], rtol=1e-3, atol=1e-4 * scale + 1e-7, msg=lambda m, k=k: f"{who}.{k}: {m}")


@pytest.fixture(params=[0, 1], ids=["in-order", "shuffled"])
def schedule(emu, request):
    """In-order schedule, then a random block / thread order: a missing __syncthreads() or a dependence on block
    order passes the first and fails the second."""
    emu.phk_emu_set_shuffle(request.param)
    yield request.param
    emu.phk_emu_set_shuffle(0)


@pytest.mark.parametrize("name", list(C.TRAIN_CASES))
def test_cuda_training_step_executed_on_the_cpu_matches_reference_autograd(golden, on_cpu, schedule, name):
    case, g = C.TRAIN_CASES[name], golden(f"train_{name}")
    maskgit, critic = _modules(case)
    ids, ctx = C.train_inputs(case)
    b, n = ids.shape[0], ids[0].numel()
    flat = ids.reshape(b, n)
    token_mask = g["token_mask"]
    tmask = torch.any(ctx != 0, dim=-1)
    vmask = torch.ones((b, n), dtype=torch.bool)
    mask_id = case["maskgit"]["num_tokens"]
    loss, gk, logits = maskgit.train_step(torch.where(token_mask, mask_id, flat), case["patch_shape"], targets=flat,
                                          token_mask=token_mask, context=ctx, text_mask=tmask, video_mask=vmask,
                                          keep_logits=critic is not None)
    ref_loss = g["ce"] if critic is not None else g["loss"]
    torch.testing.assert_close(loss, ref_loss, rtol=1e-5, atol=1e-6)
    if case.get("self_critic"):
        # SelfCritic (phenaki_pytorch.py:307-336): the MaskGit body with to_pred as head; MaskGit's gradient is the sum
        # of both passes, the bucket follows SelfCritic.parameters() (MaskGit's parameters, then to_pred)
        assert torch.equal(critic.to_pred[0].weight.detach(), g["to_pred_weight"])
        pred = g["pred_ids"]
        closs, cgk, _ = critic.train_step(torch.where(token_mask, pred, flat), case["patch_shape"],
                                          labels=(flat != pred).float(), context=ctx, text_mask=tmask, video_mask=vmask)
        torch.testing.assert_close(closs, g["bce"], rtol=1e-5, atol=1e-6)
        lin = critic.to_pred[0]
        torch.testing.assert_close(cgk.grad_of(lin.weight), g["to_pred_grads"]["weight"], rtol=1e-3, atol=1e-7)
        torch.testing.assert_close(cgk.grad_of(lin.bias), g["to_pred_grads"]["bias"], rtol=1e-3, atol=1e-7)
        assert cgk.flat.numel() == gk.flat.numel() + 128  # to_pred.weight and .bias, each on its own 256-byte line
        gk.flat += cgk.flat[:gk.flat.numel()]
        _compare(maskgit, gk, g["maskgit_grads"], "maskgit")
        return
    _compare(maskgit, gk, g["maskgit_grads"], "maskgit")
    if critic is not None:
        # the logits handed back for the critic's sampling are the forward logits, not their gradient
        from oracle import phenaki_oracle as O
        with torch.no_grad():
            ref_logits = O.maskgit_forward(torch.where(token_mask, mask_id, flat), maskgit.state_dict(),
                                           video_patch_shape=case["patch_shape"], heads=case["maskgit"]["heads"],
                                           context=ctx, text_mask=tmask, video_mask=vmask)
        torch.testing.assert_close(logits, ref_logits, rtol=1e-4, atol=1e-4)
        pred = g["pred_ids"]
        closs, cgk, _ = critic.train_step(torch.where(token_mask, pred, flat), case["patch_shape"],
                                          labels=(flat != pred).float(), context=ctx, text_mask=tmask, video_mask=vmask,
                                          loss_scale=1.0)
        torch.testing.assert_close(closs, g["bce"], rtol=1e-5, atol=1e-6)
        _compare(critic, cgk, g["critic_grads"], "critic")


def test_emulated_step_with_a_gradient_scale_and_without_text(golden, on_cpu):
    """loss_scale scales every gradient but not the reported loss; without context the cross-attention is skipped
    (attention.py:327) and its parameters get no gradient."""
    case = C.TRAIN_CASES["with_critic"]
    g = golden("train_with_critic")
    maskgit, _ = _modules(case)
    ids, ctx = C.train_inputs(case)
    b, n = ids.shape[0], ids[0].numel()
    flat, token_mask = ids.reshape(b, n), g["token_mask"]
    inp = torch.where(token_mask, case["maskgit"]["num_tokens"], flat)
    kw = dict(targets=flat, token_mask=token_mask, context=ctx, text_mask=torch.any(ctx != 0, dim=-1))
    l1, g1, _ = maskgit.train_step(inp, case["patch_shape"], **kw)
    l2, g2, _ = maskgit.train_step(inp, case["patch_shape"], loss_scale=0.25, **kw)
    torch.testing.assert_close(l1, l2, rtol=0, atol=0)
    torch.testing.assert_close(g2.flat, 0.25 * g1.flat, rtol=1e-5, atol=1e-9)
    l3, g3, _ = maskgit.train_step(inp, case["patch_shape"], targets=flat, token_mask=token_mask)
    cross = maskgit.transformer.layers[0][2]
    assert g3.grad_of(cross.to_q.weight) is None and g3.grad_of(maskgit.to_logits.weight) is not None
    from oracle import phenaki_oracle as O
    sd = {k: (v.clone().requires_grad_(True) if v.is_floating_point() else v) for k, v in maskgit.state_dict().items()}
    ref = O.maskgit_train_loss(flat, sd, token_mask, video_patch_shape=case["patch_shape"], heads=case["maskgit"]["heads"])
    ref.backward()
    torch.testing.assert_close(l3, ref.detach(), rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(g3.grad_of(maskgit.to_logits.weight), sd["to_logits.weight"].grad, rtol=1e-3, atol=1e-7)
    torch.testing.assert_close(g3.grad_of(maskgit.token_emb.weight), sd["token_emb.weight"].grad, rtol=1e-3, atol=1e-7)


@pytest.mark.parametrize("name", ["generator", "with_critic"])
def test_emulated_bf16_mode_step_tracks_the_fp32_reference(golden, on_cpu, name):
    """PHK_PREC_BF16: forward / dgrad / wgrad products through the wgmma GEMM contract (here its CPU stand-in: bf16
    operands, fp32 accumulation) with operands cast / transposed on the fly by the shipped kernels.  The dtype flow is
    torch.autocast's, so the bar is closeness to the fp32 reference: loss within 2 %, every gradient tensor within 5 % of
    its largest entry and at a cosine similarity above 0.995."""
    from phenaki_pytorch_b200 import _lib as L
    case, g = C.TRAIN_CASES[name], golden(f"train_{name}")
    maskgit, critic = _modules(case)
    maskgit.precision = L.PREC_BF16
    ids, ctx = C.train_inputs(case)
    b, n = ids.shape[0], ids[0].numel()
    flat, token_mask = ids.reshape(b, n), g["token_mask"]
    inp = torch.where(token_mask, case["maskgit"]["num_tokens"], flat)
    loss, gk, _ = maskgit.train_step(inp, case["patch_shape"], targets=flat, token_mask=token_mask, context=ctx,
                                     text_mask=torch.any(ctx != 0, dim=-1))
    ref_loss = g["ce"] if critic is not None else g["loss"]
    torch.testing.assert_close(loss, ref_loss, rtol=2e-2, atol=0)
    worst = 0.0
    for k, p in maskgit.named_parameters():
        ref = g["maskgit_grads"].get(k)
        if ref is None or ref.numel() == 0:
            continue
        got = gk.grad_of(p)
        scale = ref.abs().max().item()
        if scale < 1e-7:
            continue  # analytically zero gradients (e.g. the bias of the last position-bias layer): rounding noise
        err = (got - ref).abs().max().item() / scale
        cos = torch.nn.functional.cosine_similarity(got.flatten(), ref.flatten(), dim=0).item()
        worst = max(worst, err)
        assert err < 5e-2 and cos > 0.995, f"{k}: max err / max|ref| {err:.3e}, cosine {cos:.5f}"
    assert worst > 1e-5, "bf16 mode produced fp32-exact gradients: the tensor-core path was not taken"


def test_emulated_step_default_head_width_and_ragged_sizes(on_cpu, schedule):
    """dim_head 64 (two values per lane in the warp-per-row attention kernels), a vocabulary, context width and token
    count that are not multiples of the GEMM / warp tile sizes, a masked-out text tail: the emulated CUDA step against
    autograd through the oracle (itself pinned against the reference on the golden cases)."""
    from oracle import phenaki_oracle as O
    torch.manual_seed(123)
    ctor = dict(dim=128, num_tokens=300, max_seq_len=64, heads=2, dim_head=64, depth=1, dim_context=40)
    maskgit = P.MaskGit(**ctor)
    b, shape, L_ = 2, (2, 3, 5), 11
    n = 30
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(0, 300, (b, n), generator=g)
    token_mask = torch.rand((b, n), generator=g) < 0.4
    token_mask[0, 0] = True
    ctx = torch.randn((b, L_, 40), generator=g)
    ctx[1, 6:] = 0.0
    tmask = torch.any(ctx != 0, dim=-1)
    inp = torch.where(token_mask, 300, ids)
    loss, gk, _ = maskgit.train_step(inp, shape, targets=ids, token_mask=token_mask, context=ctx, text_mask=tmask)
    sd = {k: (v.clone().requires_grad_(True) if v.is_floating_point() else v) for k, v in maskgit.state_dict().items()}
    ref = O.maskgit_train_loss(ids, sd, token_mask, video_patch_shape=shape, heads=2, context=ctx, text_mask=tmask)
    ref.backward()
    torch.testing.assert_close(loss, ref.detach(), rtol=1e-5, atol=1e-6)
    for k, p in maskgit.named_parameters():
        got, want = gk.grad_of(p), sd[k].grad
        if got is None:
            assert want is None or float(want.abs().max()) == 0.0, k
            continue
        if want.numel() == 0:
            continue
        scale = max(want.abs().max().item(), 1e-12)
        torch.testing.assert_close(got, want, rtol=1e-3, atol=1e-4 * scale + 1e-7, msg=lambda m, k=k: f"{k}: {m}")


@pytest.mark.parametrize("name", list(C.TRAIN_CASES))
def test_phenaki_forward_end_to_end_on_the_emulator(on_cpu, monkeypatch, name):
    """The exact check the first GPU run will perform (tests/gpu_train_check.py): Phenaki.forward with the reference's
    draws injected -> MaskGit step -> gumbel sampling of the critic's input (phk_sample_tokens) -> TokenCritic /
    SelfCritic step -> loss.backward() through the autograd bridge -> loss and every p.grad against the reference."""
    from tests import gpu_train_check
    gpu_train_check.check_case(name, verbose=False, device="cpu")
