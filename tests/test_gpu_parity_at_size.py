"""GPU: parity of every precision mode at BASELINE configs[1] / configs[2] SIZES against the reference's own CUDA paths
(tools/parity_report.py: the functional oracle -- bit-identical to the unmodified reference, tests/golden/make_golden.py
-- executed on CUDA in eager fp32 and under torch.autocast(bfloat16), the reference's only bf16 path, SURVEY H2).

Bars (the measured values in parentheses are from an earlier build; the report is also written to
gpurun_out/parity_at_size.json by this test):
  * fp32 parity mode: all 8 cfg2 videos -- LFQ ids identical (a flipped bit tolerated only below a 2e-5 reference margin;
    measured 0 of 73 728); cfg3 logits within 2e-5, identical arg-max; the whole 18-step demasking loop with injected
    noise identical to the reference at EVERY step.
  * bf16 mode (the benchmarked one): at least as close to the fp32 reference as the reference's own autocast-bf16 path
    (flipped LFQ bits <= 1.25 x the reference's own + 20; measured 84 vs 136), bit agreement >= 99.8 % (99.886 %), no
    flipped bit above a 0.02 reference margin (0.0043); bit agreement with the reference's autocast path >= 99.7 %
    (99.818 %); cfg3 logits max |err| <= 0.03 and mean <= 0.003 against fp32 (0.0089 / 0.0012; the reference's own
    autocast path: 0.0177 / 0.0023).
"""
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

pytestmark = pytest.mark.gpu
_REPORT = {}


def _save():
    try:
        os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
        with open(os.path.join(ROOT, "gpurun_out", "parity_at_size.json"), "w") as f:
            json.dump(_REPORT, f, indent=1)
    except OSError:
        pass


def test_cfg2_token_ids_of_all_8_videos_against_both_reference_dtypes():
    import parity_report as R
    rep = _REPORT["cfg2_encode_ids"] = R.cfg2_report(batch=8)
    _save()
    print(json.dumps(rep, indent=1))
    f32 = rep["ours_fp32_vs_reference_fp32"]
    assert f32["flipped_bits"] <= 2 and f32["max_margin"] < 2e-5, f32
    ref16 = rep["reference_autocast_bf16_vs_reference_fp32"]
    b16 = rep["ours_bf16_vs_reference_fp32"]
    assert b16["bit_agreement"] >= 0.998 and b16["max_margin"] <= 0.02, b16
    assert b16["flipped_bits"] <= 1.25 * ref16["flipped_bits"] + 20, (b16, ref16)
    assert rep["ours_bf16_vs_reference_autocast_bf16"]["bit_agreement"] >= 0.997
    if "ours_bf16x3_vs_reference_fp32" in rep:  # split-bf16 tensor-core mode: fp32-grade products
        x3 = rep["ours_bf16x3_vs_reference_fp32"]
        assert x3["bit_agreement"] >= 0.99995 and x3["max_margin"] <= 5e-4, x3


def test_cfg2_cosine_vq_tokenizer_at_full_codebook_size():
    """SURVEY 8f-3 at size: configs[1] encoder + cosine-sim VectorQuantize with K = 65536 codes (309 GFLOP nearest-code
    search, fused wgmma head in bf16 mode), all 8 videos against the oracle on CUDA."""
    import parity_report as R
    rep = _REPORT["cfg2_cosine_vq_K65536"] = R.cfg2_cosine_vq_report(batch=8)
    _save()
    print(json.dumps(rep, indent=1))
    f32 = rep["ours_fp32"]
    # ids of the fp32 mode equal the reference's except where two codes tie to fp32 summation order
    assert f32["id_agreement_vs_reference_fp32"] >= 0.999 and f32["worst_similarity_loss_of_a_differing_id"] <= 1e-5, f32
    b16 = rep["ours_bf16"]
    ref16 = rep["reference_autocast_bf16_vs_reference_fp32"]["id_agreement"]
    assert b16["worst_similarity_loss_of_a_differing_id"] <= 0.03, b16       # never a clearly worse code
    assert b16["id_agreement_vs_reference_fp32"] >= min(0.85, ref16 - 0.05), (b16, ref16)


def test_cfg3_logits_against_both_reference_dtypes():
    import parity_report as R
    rep = _REPORT["cfg3_logits"] = R.cfg3_logits_report(batch=4)
    _save()
    print(json.dumps(rep, indent=1))
    f32 = rep["ours_fp32_vs_reference_fp32"]
    assert f32["max_abs"] <= 2e-5 and f32["argmax_agreement"] == 1.0, f32
    b16, ref16 = rep["ours_bf16_vs_reference_fp32"], rep["reference_autocast_bf16_vs_reference_fp32"]
    assert b16["max_abs"] <= 0.03 and b16["mean_abs"] <= 0.003, b16
    assert b16["mean_abs"] <= 1.25 * ref16["mean_abs"], (b16, ref16)
    if "ours_bf16x3_vs_reference_fp32" in rep:
        x3 = rep["ours_bf16x3_vs_reference_fp32"]
        assert x3["max_abs"] <= 5e-4 and x3["argmax_agreement"] >= 0.9995, x3


def test_cfg3_full_demasking_loop_equals_the_reference_step_by_step():
    import parity_report as R
    rep = _REPORT["cfg3_demask_loop"] = R.cfg3_loop_report(batch=1, steps=18)
    _save()
    print(json.dumps(rep, indent=1))
    loop = rep["fp32_unfused_vs_reference_fp32_injected_noise"]
    assert loop["first_step_with_any_difference"] is None and loop["final_id_agreement"] == 1.0, loop
    t0 = rep["temperature0_ours_fp32"]
    assert t0["final_id_agreement_vs_reference_fp32"] == 1.0 and t0["step0_pred_agreement_vs_reference_fp32"] == 1.0, t0
    # temperature-0 decoding in bf16 is a chaotic map of the logits' last bits (the reference's own autocast path ends at
    # ~44 % of its fp32 ids): the fused bf16 loop must simply be in that regime, not closer to noise
    ours, ref = rep["temperature0_ours_bf16"], rep["temperature0_reference_autocast_bf16_vs_reference_fp32"]
    assert ours["final_id_agreement_vs_reference_fp32"] >= 0.5 * ref["final_id_agreement"], (ours, ref)
