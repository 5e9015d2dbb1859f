"""TEST INFRASTRUCTURE: builds tests/cuda_emu (csrc/train.cu compiled by g++ for the CPU executor) and routes the
product's host path to it with CPU tensors.  Used by test_train_emulated_cpu.py and the two-rank gloo test."""
import contextlib
import ctypes
import os
import re
import subprocess

import torch

from phenaki_pytorch_b200 import _lib as L
from phenaki_pytorch_b200 import modules as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_DIR = os.path.join(ROOT, "tests", "cuda_emu")
# PHK_EMU_ASAN=1 (with libasan preloaded into the python process, see tests/test_emulated_asan_cpu.py): the kernels run under
# AddressSanitizer, i.e. every out-of-bounds access of a kernel to a torch buffer or the workspace is reported
ASAN = os.environ.get("PHK_EMU_ASAN", "0") == "1"
EMU_LIB = os.path.join(EMU_DIR, "_build", "libphk_train_emu_asan.so" if ASAN else "libphk_train_emu.so")
CSRC = os.path.join(ROOT, "phenaki_pytorch_b200", "csrc")
# the product's plain-CUDA sources (no tensor cores / TMA): compiled unchanged apart from the two textual rewrites below
KERNEL_SOURCES = ["rowops.cu", "gemm_simt.cu", "attention.cu", "sample_tail.cu", "vq.cu", "train.cu", "api.cu"]  # api.cu: the drivers (host code)
SOURCES = [os.path.join(EMU_DIR, "cuda_emu.cpp")]


def _for_emulator(text):
    """(1) the CUDA helper header -> the emulator's; (2) `extern __shared__ T name[];` (dynamic shared memory) -> a
    pointer to the launch's buffer.  Nothing else of the kernel source changes."""
    text = text.replace('#include "phk_common.cuh"', f'#include "{os.path.join(EMU_DIR, "cuda_emu.h")}"')
    return re.sub(r"extern __shared__ (?:__align__\(\d+\) )?([\w ]+?) (\w+)\[\];",
                  r"\1* \2 = reinterpret_cast<\1*>(::emu::S.dyn_smem);", text)


def build_emu(extra_source=None, lib_path=EMU_LIB):
    """extra_source: (path, text) of code appended to train.cu's translation unit (test-only wrappers around its
    internal functions), built into lib_path instead of the shared EMU_LIB."""
    kernel_paths = [os.path.join(CSRC, f) for f in KERNEL_SOURCES]
    deps = SOURCES + kernel_paths + [os.path.join(EMU_DIR, "cuda_emu.h"), os.path.join(ROOT, "include", "phk.h"),
                                     os.path.abspath(__file__)] + ([extra_source[0]] if extra_source else [])
    if not os.path.exists(lib_path) or any(os.path.getmtime(d) > os.path.getmtime(lib_path) for d in deps):
        build = os.path.dirname(lib_path)
        os.makedirs(build, exist_ok=True)
        rewritten = []
        for path in kernel_paths:
            out = os.path.join(build, f"{os.path.basename(path)}.{os.getpid()}.emu.cpp")
            with open(path) as f, open(out, "w") as g:
                g.write(_for_emulator(f.read()))
                if extra_source and os.path.basename(path) == "train.cu":
                    g.write("\n" + _for_emulator(extra_source[1]))
            rewritten.append(out)
        tmp = lib_path + f".{os.getpid()}.tmp"
        try:
            san = ["-fsanitize=address", "-fno-omit-frame-pointer", "-g"] if ASAN else []
            subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-U_FORTIFY_SOURCE",
                                   "-D_FORTIFY_SOURCE=0", "-DPHK_CUDA_EMU", *san, "-x", "c++", *SOURCES, *rewritten, "-o", tmp])
        finally:
            for r in rewritten:
                os.remove(r)
        os.replace(tmp, lib_path)
    lib = ctypes.CDLL(lib_path)
    for name, argtypes in L.PROTOTYPES.items():
        if not hasattr(lib, name):
            continue  # tensor-core / TMA entry points are not part of the emulated build
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = L._RESTYPES.get(name, ctypes.c_int)
    lib.phk_last_error.restype = ctypes.c_char_p
    lib.phk_emu_set_shuffle.argtypes = [ctypes.c_uint64]
    lib.phk_emu_set_shuffle.restype = None
    return lib


class _Setter:
    """monkeypatch-shaped setter for processes that never need to undo (spawned workers)."""

    @staticmethod
    def setattr(obj, name, value):
        setattr(obj, name, value)


def route_product_to_emulator(lib, patch=_Setter):
    """The product refuses CPU tensors by design; under test the train-step entry points are served by the emulated
    library instead of libphk.so and the CUDA-only plumbing (device guard, stream) becomes a no-op."""
    patch.setattr(L, "lib", lambda: lib)
    patch.setattr(L, "require_cuda", lambda t, name, dtype=None: t.contiguous())
    patch.setattr(L, "stream_ptr", lambda: None)
    patch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())

    def keep_t(self, tensor):
        tensor = tensor.detach().float().contiguous()
        self.refs.append(tensor)
        return tensor.data_ptr()

    patch.setattr(M.Keep, "t", keep_t)

    def keep_h(self, tensor):
        t = tensor.detach().to(torch.bfloat16).contiguous()
        self.refs.append(t)
        return t.data_ptr()

    patch.setattr(M.Keep, "h", keep_h)

    def keep_h3(self, tensor):
        t = M.split3_weight(tensor)
        self.refs.append(t)
        return t.data_ptr()

    patch.setattr(M.Keep, "h3", keep_h3)
    def poisoned_workspace(self, nbytes, device):
        # fresh host pages are zero and would hide a kernel that reads scratch it never wrote: hand out 0xFF bytes
        # (fp32 NaN, int64 -1) on every call instead
        if self.buf is None or self.buf.numel() < nbytes or self.buf.device != device:
            self.buf = torch.empty(int(nbytes), dtype=torch.uint8, device=device)
        self.buf.fill_(0xFF)
        return self.buf

    patch.setattr(M.Workspace, "get", poisoned_workspace)
    real_empty = torch.empty

    def poisoned_empty(*size, **kw):
        t = real_empty(*size, **kw)
        if t.dtype in (torch.float32, torch.bfloat16):
            t.fill_(float("nan"))
        elif t.dtype in (torch.int64, torch.uint8):
            t.fill_(-1 if t.dtype == torch.int64 else 255)
        return t

    patch.setattr(torch, "empty", poisoned_empty)  # outputs the kernels are expected to overwrite completely
    from phenaki_pytorch_b200 import phenaki as PH
    patch.setattr(PH, "_noise_seed", lambda dev: torch.initial_seed())  # no CUDA generator without a GPU
    # ... whose offset is the running noise counter on the GPU (PH._rng_take): restarted by torch.manual_seed
    counter = [0]
    real_manual_seed = torch.manual_seed

    def manual_seed(seed):
        counter[0] = 0
        return real_manual_seed(seed)

    def rng_take(dev, seed, count):
        first = counter[0]
        counter[0] = first + (int(count) + 3) // 4 * 4
        return first

    patch.setattr(torch, "manual_seed", manual_seed)
    patch.setattr(PH, "_rng_take", rng_take)
