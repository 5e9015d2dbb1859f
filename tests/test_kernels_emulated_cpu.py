"""CPU: the kernel-granularity parity tests of tests/test_gpu_kernels.py (the ones whose kernels are plain CUDA: rowops.cu,
gemm_simt.cu, attention.cu) run a second time with the kernels EXECUTED ON THE CPU by tests/cuda_emu.  Same test
bodies, same oracle comparisons, same tolerances -- only the device string and the library handle are swapped.

Two purposes: (1) these kernels are validated on the H100 by the -m gpu suite, so their passing here is the check of the
executor itself (the training-step tests rely on it); (2) the CPU-only container gets kernel-level coverage of the
shipped sources (indexing, barriers, edge tiles) before any GPU time is spent."""
import pytest
import torch

from phenaki_pytorch_b200 import _lib as L
from tests import emu_runtime
from tests import test_gpu_kernels as G

_NAMES = ["test_layernorm", "test_layernorm_row_map_and_bf16", "test_patchify_ln", "test_gemm_f32", "test_gemm_f32_row_map",
          "test_geglu", "test_attention_self_bias_mask", "test_attention_causal_alibi",
          "test_attention_cross_null_kv_mask_and_cfg_half", "test_attention_strided_sequences",
          "test_peg3d_against_reference_golden_semantics", "test_peg3d_matches_reference_module_golden",
          "test_continuous_position_bias", "test_lfq_ids_bit_exact_where_margin_allows", "test_token_embed_bit_exact",
          "test_sample_tokens_matches_reference_ops", "test_topk_mask_matches_torch_topk_scatter",
          "test_critic_scores_and_cfg_combine", "test_attention_short_sequence_warp_kernel",
          "test_layernorm_lfq_fused_matches_separate_kernels"]
for _n in _NAMES:  # collected here without the module-level gpu mark of test_gpu_kernels.py; parametrisations carry over
    globals()[_n] = getattr(G, _n)


@pytest.fixture(scope="module")
def _emu_lib():
    return emu_runtime.build_emu()


@pytest.fixture(autouse=True)
def _kernels_on_the_cpu(_emu_lib, monkeypatch):
    monkeypatch.setattr(G, "DEV", "cpu")
    monkeypatch.setattr(L, "lib", lambda: _emu_lib)
    monkeypatch.setattr(L, "stream_ptr", lambda: None)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    yield
    G._HOLD.clear()
