"""CPU: PHK_PREC_BF16X3 (split-bf16 tensor-core mode) through the product path on the CPU executor: weight packs
[hi | lo | hi], the activation split kernel [hi | hi | lo] (rowops.cu, executed) and the drivers' wiring; the wgmma
GEMM itself is represented by its contract (bf16 operands, fp32 accumulation).  Bars: the fp32 parity mode's -- token ids
identical to the reference's, logits within 2e-4 -- because hi + lo carries 16 mantissa bits of every operand."""
import pytest
import torch

import phenaki_pytorch_b200 as P
from phenaki_pytorch_b200 import _lib as L
from phenaki_pytorch_b200.modules import split3_weight
from tests import cases as C
from tests import emu_runtime


@pytest.fixture(scope="module")
def _emu_lib():
    return emu_runtime.build_emu()


@pytest.fixture(autouse=True)
def _product_on_the_cpu(_emu_lib, monkeypatch):
    emu_runtime.route_product_to_emulator(_emu_lib, monkeypatch)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)


def test_split_pack_reconstructs_the_operand_to_16_mantissa_bits():
    w = C.seeded_randn((5, 13), 1) * 3
    pk = split3_weight(w).float()
    kp = 16
    assert pk.shape == (5, 3 * kp)
    hi, lo = pk[:, :13], pk[:, kp:kp + 13]
    assert torch.equal(pk[:, 2 * kp:2 * kp + 13], hi) and (pk[:, 13:kp] == 0).all()
    assert ((w - hi - lo).abs() <= w.abs() * 2.0 ** -16).all()


@pytest.mark.parametrize("name", ["cfg1", "rect"])
def test_cvivit_ids_in_split_bf16_mode_equal_the_reference(golden, name):
    case, g = C.CVIVIT_CASES[name], golden(f"cvivit_{name}")
    torch.manual_seed(case["seed"])
    model = P.CViViT(**case["ctor"]).eval()
    model.precision = L.PREC_BF16X3
    video = C.seeded_randn(case["video"], case["video_seed"])
    ids = model(video, return_only_codebook_ids=True)
    assert torch.equal(ids, g["ids"])
    rec = model.decode_from_codebook_indices(ids)
    model.precision = L.PREC_F32
    torch.testing.assert_close(rec, model.decode_from_codebook_indices(ids), rtol=2e-4, atol=2e-4)


def test_maskgit_logits_in_split_bf16_mode_match_the_reference(golden):
    case, g = C.MASKGIT_CASES["small"], golden("maskgit_small")
    torch.manual_seed(case["seed"])
    model = P.MaskGit(**case["ctor"]).eval()
    model.precision = L.PREC_BF16X3
    ids, ctx = C.token_inputs(case, case["ctor"]["num_tokens"])
    kw = dict(text_mask=torch.any(ctx != 0, dim=-1), video_patch_shape=case["patch_shape"], context=ctx)
    torch.testing.assert_close(model(ids, **kw), g["cond"], rtol=2e-4, atol=2e-4)
    torch.testing.assert_close(model.forward_with_cond_scale(ids, cond_scale=3.0, **kw), g["cfg"], rtol=2e-4, atol=1e-3)
