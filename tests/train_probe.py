"""TEST INFRASTRUCTURE: the probe library of tests/train_probe.cu -- csrc/train.cu unchanged plus extern "C" wrappers
around its internal functions (the products sgemm_batched, linear_fwd / dgrad_p / wgrad_p, attention_backward, colsum;
the rest of the backward ln_backward, geglu_dropout_fwd / geglu_backward, peg_backward, embed_backward, cpb_backward,
ce_rows / bce_rows / loss_reduce; the deterministic-mode scratch t_det), so that tests can drive each one on its own.
libphk.so does not export them.

On the GPU the probe is compiled with the product's nvcc flags and linked with the other csrc objects that
phenaki_pytorch_b200.build leaves behind; on the CPU executor the same wrappers are appended to the emulated train.cu."""
import ctypes as C
import os
import subprocess

from phenaki_pytorch_b200 import _lib as L
from phenaki_pytorch_b200 import build as B
from tests import emu_runtime

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "train_probe.cu")
LIB = os.path.join(HERE, "train_probe", "_build", "libphk_train_probe.so")
EMU_LIB = os.path.join(emu_runtime.EMU_DIR, "_build", "libphk_train_probe_emu.so")
INCLUDE_TRAIN = '#include "../phenaki_pytorch_b200/csrc/train.cu"'

i64, i32, vp = C.c_int64, C.c_int32, C.c_void_p
f32, u32, u64 = C.c_float, C.c_uint32, C.c_uint64
PROTOTYPES = {
    "probe_sgemm_batched": [vp, i64, i64, vp, i64, i64, vp, i64, i64, i64, i64, i32, i32, i32, i64, i64, i64, i64, i64,
                            i64, i32, i32, vp],
    "probe_linear": [i32, i32, vp, i64, vp, vp, vp, i64, i64, i64, vp, vp, i32, vp],
    "probe_attention_backward": [vp, vp, C.POINTER(L.AttnT), C.POINTER(L.AttnT), vp, vp, vp, vp, vp, vp, i32, i32, i32,
                                 i32, i32, i32, vp, i32, vp],
    "probe_attn_bwd_layout": [i32, i32, i32, i32, i32, i32, C.POINTER(i64)],
    "probe_colsum": [vp, i64, i32, i64, vp, vp],
    "probe_set_det_scratch": [vp, i64],
    "probe_ln_backward": [vp, vp, vp, vp, i32, vp, vp, vp, i64, i32, vp],
    "probe_geglu_dropout_fwd": [vp, vp, i64, i32, f32, f32, u32, u32, u64, vp],
    "probe_geglu_backward": [vp, vp, vp, i64, i32, f32, f32, u32, u32, u64, vp],
    "probe_peg_backward": [vp, vp, vp, vp, vp, vp, i64, i32, i32, i32, i32, i32, vp],
    "probe_embed_backward": [vp, vp, vp, vp, i64, i32, i32, f32, i32, vp],
    "probe_cpb_backward": [C.POINTER(L.CpbT), C.POINTER(L.CpbT), vp, i32, i32, i32, vp, vp],
    "probe_scratch_floats": [C.POINTER(L.CpbT), i32, i32, i32, i64, i32, C.POINTER(i64)],
    "probe_ce_rows": [vp, vp, vp, vp, f32, vp, i64, i32, vp],
    "probe_bce_rows": [vp, vp, vp, vp, f32, vp, vp, i64, i32, vp],
    "probe_loss_reduce": [vp, i64, vp, vp],
}


def _bind(lib):
    for name, argtypes in PROTOTYPES.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = C.c_int
    lib.phk_launch_count.restype = C.c_int64
    lib.phk_last_error.restype = C.c_char_p
    return lib


def _objects():
    return [s[:-3] + ".o" for s in B.sources() if os.path.basename(s) != "train.cu"]


def build():
    """nvcc: train_probe.cu (-> train.cu) with the product's flags, linked with the product's other objects.  Rebuilt
    when a csrc source or header, phk.h or the probe is newer than the library (as build.py decides for libphk.so)."""
    deps = B.sources() + [os.path.join(B.CSRC, f) for f in os.listdir(B.CSRC) if f.endswith(".cuh")]
    deps += [os.path.join(os.path.dirname(B.HERE), "include", "phk.h"), SRC]
    if os.path.exists(LIB) and all(os.path.getmtime(d) <= os.path.getmtime(LIB) for d in deps):
        return LIB
    objs = _objects()
    if B.needs_build() or not all(os.path.exists(o) for o in objs):
        B.build(force=True)
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    obj = LIB[:-3] + f".{os.getpid()}.o"
    tmp = LIB + f".{os.getpid()}.tmp"
    try:
        subprocess.check_call([B.NVCC, *B.FLAGS, "-c", SRC, "-o", obj])
        subprocess.check_call([B.NVCC, *B.FLAGS[:2], "-shared", "-o", tmp, obj, *objs, "-lcudart", "-lcuda"])
        os.replace(tmp, LIB)
    finally:
        for f in (obj, tmp):
            if os.path.exists(f):
                os.remove(f)
    return LIB


def load():
    return _bind(C.CDLL(build()))


def load_emulated():
    """The CPU executor's library with the same wrappers appended to train.cu's translation unit (a library of its own:
    the shared emulated library of the other tests is left as it is)."""
    with open(SRC) as f:
        text = f.read()
    assert INCLUDE_TRAIN in text
    return _bind(emu_runtime.build_emu((SRC, text.replace(INCLUDE_TRAIN, "")), EMU_LIB))
