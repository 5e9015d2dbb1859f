"""Per-phase clock64 stamps of the wgmma GEMM (debug): python tools/gemm_trace.py M N K [epilogue]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from phenaki_pytorch_b200 import _lib as L
M, N, K = (int(v) for v in sys.argv[1:4])
epi = int(sys.argv[4]) if len(sys.argv) > 4 else 0
dev = "cuda"
a = torch.randn(M, K, device=dev).bfloat16(); w = torch.randn(N, K, device=dev).bfloat16()
c = torch.zeros(M, N if epi != 2 else N // 2, device=dev, dtype=torch.float32 if epi == 0 else torch.bfloat16)
res = torch.randn(M, N, device=dev) if epi == 0 else None
trace = torch.zeros(148 * 16, dtype=torch.int64, device=dev)
lib = L.lib()
def run():
    L.check(lib.phk_gemm_bf16(L.ptr(a), K, L.ptr(w), K, L.ptr(c), c.shape[1], M, N, K, None, L.ptr(c) if epi == 0 else None, 0, 0, 0, epi, L.stream_ptr()))
for _ in range(3): run()
torch.cuda.synchronize()
lib.phk_debug_gemm_trace(L.ptr(trace))
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record(); run(); e1.record(); torch.cuda.synchronize()
lib.phk_debug_gemm_trace(None)
t = trace.cpu().reshape(148, 16)
tiles = ((M + 127) // 128) * ((N + 127) // 128)
used = t[t[:, 9] > 0]  # CTAs that ran (one-CTA kernel: min(tiles, 148); CTA-pair kernel: 2 x pairs)
names = ["setup", "tma0_issued", "tmaLast_issued", "ops0_landed", "opsLast_landed", "mma_issued", "acc_ready", "staged", "written", "cta_done", "geglu_tmem_read", "geglu_math_done"]
print(f"M={M} N={N} K={K} epi={epi} PHK_GEMM_MODE={os.environ.get('PHK_GEMM_MODE', '0')}: 128x128 tiles={tiles} CTAs={used.shape[0]} event time {e0.elapsed_time(e1)*1e3:.1f} us")
for i, n in enumerate(names):
    col = used[:, i].float()
    print(f"  {n:16s} mean {col.mean():9.0f}  min {col.min():9.0f}  max {col.max():9.0f} cycles")
