"""CPU: the module-granularity parity tests of tests/test_gpu_models.py and tests/test_gpu_decode.py (fp32 parity mode)
run a second time with the WHOLE product path executed on the CPU: the reference-facing classes, the ctypes tables, the
drivers of csrc/api.cu and every kernel they launch (rowops.cu, gemm_simt.cu, attention.cu), compiled by g++ against
tests/cuda_emu.  Same test bodies and bars as on the H100: C-ViViT token ids identical to the reference's, logits /
critic scores / reconstructions within 2e-4, the full demasking loop (with the reference's noise replayed) identical.

What only the GPU run covers: bf16 mode (wgmma / TMA kernels), pinned-memory pipelines, CUDA-graph replay, speed."""
import pytest
import torch

from tests import emu_runtime
from tests import test_gpu_decode as D
from tests import test_gpu_models as G

_MODELS = ["test_cvivit_token_ids_match_reference_golden", "test_cvivit_state_dict_roundtrip_changes_nothing",
           "test_cvivit_shape_contract_errors", "test_maskgit_logits_match_reference_golden",
           "test_maskgit_sequence_length_contract", "test_token_critic_scores_match_reference_golden",
           "test_sampling_loop_token_ids_match_reference_golden"]
for _n in _MODELS:
    globals()[_n] = getattr(G, _n)
from tests import test_gpu_zz_after_last_gpu_call as Z  # noqa: E402
test_cosine_vq_token_ids_match_reference_golden = Z.test_cosine_vq_token_ids_match_reference_golden
test_cosine_vq_decode_matches_reference_golden = Z.test_cosine_vq_decode_matches_reference_golden
# not repeated here: the refusal of CPU tensors (meaningless under the executor) and, to keep the CPU suite short, the
# sampled-video / make_video chains (their pieces -- sampling loops with priming, decode -- are covered above and below)
_SKIP = {"test_decode_token_count_contract", "test_sampled_video_matches_reference_golden",
         "test_make_video_scene_chain_matches_reference_golden"}
_DECODE = [n for n in dir(D) if n.startswith("test_") and "bf16" not in n and n not in _SKIP]
for _n in _DECODE:
    globals()["decode_" + _n if _n in globals() else _n] = getattr(D, _n)


@pytest.fixture(scope="module")
def _emu_lib():
    return emu_runtime.build_emu()


@pytest.fixture(autouse=True)
def _product_on_the_cpu(_emu_lib, monkeypatch):
    emu_runtime.route_product_to_emulator(_emu_lib, monkeypatch)
    monkeypatch.setattr(G, "DEV", "cpu")
    monkeypatch.setattr(D, "DEV", "cpu", raising=False)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
