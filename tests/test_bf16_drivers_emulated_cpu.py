"""CPU: the bf16-mode parity tests of tests/test_gpu_bf16_mode.py with the DRIVERS executed from the shipped source
(csrc/api.cu, sample_tail.cu and every plain kernel they launch) and the wgmma / TMA kernels represented by their
include/phk.h contracts (tests/cuda_emu/cuda_emu.cpp: bf16 operands, fp32 accumulation).  What this covers is the host
logic of bf16 mode -- bf16 weight packing (GEGLU row interleave, padding), buffer wiring, the CFG-pair sharing of the
first layer, the masked-rows tail of the demasking step -- not the tensor-core kernels themselves, which only the H100
run exercises."""
import ctypes

import pytest
import torch

from tests import emu_runtime
from tests import test_gpu_bf16_mode as G
from tests import test_gpu_zz_after_last_gpu_call as Z

_NAMES = ["test_cvivit_bf16_mode_against_fp32_reference_golden", "test_maskgit_bf16_mode_against_fp32_reference_golden",
          "test_layernorm_cfg_combination",
          "test_fused_sample_step_agrees_with_unfused_path", "test_bf16_sampling_with_fused_head_is_deterministic",
          "test_fused_sample_step_on_masked_rows_equals_the_all_rows_step",
          "test_cosine_vq_ids_in_bf16_mode_against_fp32_reference_golden",
          "test_primed_fused_sample_step_equals_the_unprimed_step_on_the_same_rows"]
for _n in _NAMES:
    globals()[_n] = getattr(G, _n) if hasattr(G, _n) else getattr(Z, _n)


@pytest.fixture(scope="module")
def _emu_lib():
    return emu_runtime.build_emu()


@pytest.fixture(autouse=True)
def _product_on_the_cpu(_emu_lib, monkeypatch):
    emu_runtime.route_product_to_emulator(_emu_lib, monkeypatch)
    monkeypatch.setattr(G, "DEV", "cpu")
    monkeypatch.setattr(Z, "DEV", "cpu")
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    monkeypatch.setattr(torch.cuda, "manual_seed_all", lambda *a, **k: None, raising=False)


def test_demasking_iterations_as_replayed_graphs_equal_the_default_loop(_emu_lib):
    """phk_maskgit_demask_iteration (one call per iteration, all state in device memory) -- eager, and captured /
    replayed as a graph (the executor records the operations submitted between BeginCapture and EndCapture with their
    arguments BY VALUE, i.e. it bakes in exactly what a CUDA graph bakes in) -- must produce the ids of the default loop
    for three consecutive sample() calls: the second call captures, the third replays, and each call draws fresh noise,
    so a value wrongly baked into the graph (noise key, k, temperature, a stale pointer) shows up as a difference."""
    from phenaki_pytorch_b200 import _lib as L
    from tests import cases as C
    import phenaki_pytorch_b200 as P
    case = C.SAMPLE_CASES["confidence"]

    def run(iteration_call, graph):
        torch.manual_seed(case["seed"])
        cv = P.CViViT(**C.SAMPLE_CVIVIT)
        mg = P.MaskGit(dim=128, num_tokens=256, max_seq_len=64, heads=2, dim_head=64, depth=2, dim_context=48)
        mg.precision = L.PREC_BF16
        ph = P.Phenaki(cvivit=cv, maskgit=mg, steps=5, text_embed_dim=48)
        ph.iteration_call = iteration_call
        _emu_lib.phk_debug_step_graph(graph)
        ctx = C.synthetic_text_embeds(2, 6, 48, (6, 3), 3)
        torch.manual_seed(11)
        outs = [ph.sample(num_frames=7, text_embeds=ctx, return_token_ids=True).clone() for _ in range(3)]
        _emu_lib.phk_debug_step_graph(-1)
        return outs

    base = run(False, 0)
    assert not torch.equal(base[0], base[1]) and not torch.equal(base[1], base[2])  # fresh noise per call
    _emu_lib.phk_emu_graph_launches.restype = ctypes.c_long
    for graph in (0, 1):
        before = _emu_lib.phk_emu_graph_launches()
        got = run(True, graph)
        replays = _emu_lib.phk_emu_graph_launches() - before
        assert replays == (10 if graph else 0)  # 5 iterations each: captured + launched in call 2, replayed in call 3
        for i in range(3):
            assert torch.equal(got[i], base[i]), f"graph={graph}, call {i}"


@pytest.mark.parametrize("critic_kind,primed", [("token", True), ("self", False), (None, True), ("token", False)])
def test_critic_and_primed_iterations_as_replayed_graphs_equal_the_per_step_loop(_emu_lib, critic_kind, primed):
    """phk_maskgit_demask_iteration_critic (re-mask + MaskGit CFG pair + tail + critic CFG pair + scores per call; prime ids
    ahead of the sampled tokens) against the per-step Python loop: three consecutive samples (eager, captured, replayed),
    fresh V-wide noise and fresh critic noise per call -- a value wrongly baked into a graph shows up as a difference."""
    from phenaki_pytorch_b200 import _lib as L
    from tests import cases as C
    import phenaki_pytorch_b200 as P

    def run(iteration_call, graph):
        torch.manual_seed(31)
        cv = P.CViViT(**C.SAMPLE_CVIVIT)
        mg = P.MaskGit(dim=128, num_tokens=256, max_seq_len=64, heads=2, dim_head=64, depth=2, dim_context=48)
        critic = None
        if critic_kind == "token":
            critic = P.TokenCritic(dim=128, num_tokens=256, max_seq_len=64, has_cross_attn=True, heads=2, dim_head=64, depth=1,
                                   dim_context=48)
            critic.precision = L.PREC_BF16
        elif critic_kind == "self":
            critic = P.SelfCritic(mg)
        mg.precision = L.PREC_BF16
        ph = P.Phenaki(cvivit=cv, maskgit=mg, critic=critic, steps=5, text_embed_dim=48, critic_noise_anneal_schedule="decay")
        ph.iteration_call = iteration_call
        _emu_lib.phk_debug_step_graph(graph)
        ctx = C.synthetic_text_embeds(2, 6, 48, (6, 3), 3)
        prime = torch.randint(0, 256, (2, 16), generator=torch.Generator().manual_seed(5)) if primed else None
        n = 32 if primed else 48
        torch.manual_seed(12)
        outs = [ph.sample_token_ids(num_tokens=n, patch_shape=(3, 4, 4), batch_size=2, text_embeds=ctx, prime_token_ids=prime,
                                    cond_scale=3.0).clone() for _ in range(3)]
        _emu_lib.phk_debug_step_graph(-1)
        return outs

    base = run(False, 0)
    assert not torch.equal(base[0], base[1])
    _emu_lib.phk_emu_graph_launches.restype = ctypes.c_long
    for graph in (0, 1):
        before = _emu_lib.phk_emu_graph_launches()
        got = run(True, graph)
        replays = _emu_lib.phk_emu_graph_launches() - before
        assert replays == (10 if graph else 0)
        for i in range(3):
            assert torch.equal(got[i], base[i]), f"graph={graph}, call {i}"
