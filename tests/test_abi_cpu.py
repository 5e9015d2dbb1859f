"""CPU suite: the C-ABI shared library loads and exports every symbol include/phk.h declares; argument
validation (no device work) follows the documented error convention."""
import ctypes
import os
import re

import pytest

from phenaki_pytorch_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    text = open(os.path.join(ROOT, "include", "phk.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(phk_[a-z0-9_]+)\s*\(", text)))


def test_library_is_built_and_exports_every_declared_symbol():
    assert os.path.exists(L.LIB_PATH), "build libphk.so first: python -m phenaki_pytorch_b200.build"
    raw = ctypes.CDLL(L.LIB_PATH)
    syms = header_symbols()
    assert len(syms) >= 20
    missing = [s for s in syms if not hasattr(raw, s)]
    # phk_gemm_bf16 (wgmma) lands with the tensor-core path; everything else must already resolve
    assert missing == []


def test_bindings_cover_the_header():
    syms = set(header_symbols())
    bound = set(L.PROTOTYPES)
    assert bound <= syms, f"bindings without a declaration: {bound - syms}"
    assert syms == bound, f"declared but unbound: {syms - bound}"


def test_error_convention_without_a_gpu():
    lib = L.lib()
    assert lib.phk_version() >= 100
    # null pointers -> PHK_E_ARG (-1) and a message, never a crash
    rc = lib.phk_layernorm(None, None, None, None, None, 4, 8, 0, 0, 0, 0, None)
    assert rc == -1 and b"null" in lib.phk_last_error()
    with pytest.raises(L.PhkError):
        L.check(rc, "phk_layernorm")
    rc = lib.phk_topk_mask(ctypes.c_void_p(256), 1, 10, 11, ctypes.c_void_p(256), ctypes.c_void_p(256), 0, None)
    assert rc == -2  # k > n: shape contract (torch.topk would raise) -> AssertionError on the python side
    with pytest.raises(AssertionError):
        L.check(rc, "phk_topk_mask")


def test_struct_sizes_match_the_c_side():
    """ctypes mirrors must have the C layout (checked through the sizes the compiler reports)."""
    import subprocess
    import tempfile
    src = r'''
#include <stdio.h>
#include "phk.h"
int main(){printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(phk_attn_t), sizeof(phk_ff_t), sizeof(phk_peg_t),
 sizeof(phk_layer_t), sizeof(phk_transformer_t), sizeof(phk_cpb_t), sizeof(phk_cvivit_t), sizeof(phk_maskgit_t),
 sizeof(phk_attn_geom_t), sizeof(phk_cvivit_dec_t));return 0;}'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "s.c")
        open(c, "w").write(src)
        exe = os.path.join(d, "s")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        sizes = [int(v) for v in subprocess.check_output([exe]).split()]
    mine = [ctypes.sizeof(t) for t in (L.AttnT, L.FFT, L.PegT, L.LayerT, L.TransformerT, L.CpbT, L.CvivitT,
                                       L.MaskgitT, L.AttnGeomT, L.CvivitDecT)]
    assert mine == sizes
