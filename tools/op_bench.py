"""Steady-state time of each building block at the benchmark shapes: N back-to-back launches inside one CUDA-event
bracket (full clocks, warm L2) -- complements the ncu launch lists, whose serialised per-kernel times are inflated for
short kernels.  usage: python tools/op_bench.py [reps]"""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from phenaki_pytorch_b200 import _lib as L  # noqa: E402
from phenaki_pytorch_b200.modules import alibi_slopes  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 50
dev = "cuda"
lib = L.lib()
sp = L.stream_ptr
R, D, I, H = 4608, 512, 512, 8
bf = torch.bfloat16


def timeit(name, fn, work=None, unit=""):
    """`reps` launches captured into ONE CUDA graph (no python/ctypes cost between launches), replayed 5 times."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    st = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(st):
        fn()
        torch.cuda.synchronize()
        with torch.cuda.graph(graph, stream=st):
            for _ in range(reps):
                fn()
    graph.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        graph.replay()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / (5 * reps)
    extra = f"  {work / us / 1e6:8.1f} {unit}" if work else ""
    print(f"{name:46s} {us:8.2f} us{extra}")


x = torch.randn(R, D, device=dev)
g, b = torch.randn(D, device=dev), torch.randn(D, device=dev)
xn_h, raw_h = torch.empty(R, D, dtype=bf, device=dev), torch.empty(R, D, dtype=bf, device=dev)
timeit("layernorm -> bf16 (+raw)", lambda: L.check(lib.phk_layernorm(L.ptr(x), L.ptr(g), L.ptr(b), L.ptr(xn_h), L.ptr(raw_h), R, D, 1, 0, 0, 0, sp())),
       R * D * 8, "TB/s")

for (M, N, K, epi, name) in [(4608, 512, 512, 0, "gemm q/out-proj (+res)"), (4608, 1024, 512, 0, "gemm kv-proj"),
                             (4608, 2816, 512, 2, "gemm FF1 + GEGLU"), (4608, 512, 1408, 0, "gemm FF2 (+res)"),
                             (4096, 512, 6144, 0, "gemm patch-embed"), (2304, 65536, 512, 0, "gemm logits head (unfused)")]:
    a = torch.randn(M, K, device=dev).to(bf)
    w = torch.randn(N, K, device=dev).to(bf)
    c = torch.zeros(M, N if epi != 2 else N // 2, device=dev, dtype=torch.float32 if epi == 0 else bf)
    res = L.ptr(c) if (epi == 0 and N == 512) else None
    timeit(name + f" {M}x{N}x{K}", lambda: L.check(lib.phk_gemm_bf16(L.ptr(a), K, L.ptr(w), K, L.ptr(c), c.shape[1], M, N, K, None, res, 0, 0, 0, epi, sp())),
           2.0 * M * N * K, "TFLOP/s")

a1 = torch.randn(R, D, device=dev).to(bf); a2 = torch.randn(R, D, device=dev).to(bf)
w1 = torch.randn(I, D, device=dev).to(bf); w2 = torch.randn(2 * I, D, device=dev).to(bf)
c1 = torch.zeros(R, I, device=dev); c2 = torch.zeros(R, 2 * I, device=dev)
timeit("gemm q + kv in one launch (x2)", lambda: L.check(lib.phk_gemm_bf16_x2(L.ptr(a1), D, L.ptr(w1), D, L.ptr(c1), I, R, I, D, None, L.ptr(a2), D, L.ptr(w2), D, L.ptr(c2), 2 * I, R, 2 * I, D, None, sp())),
       2.0 * R * 3 * I * D, "TFLOP/s")

# temporal attention (n=9, causal) on the (b,t,h,w) layout
q, kv = torch.randn(R, I, device=dev), torch.randn(R, 2 * I, device=dev)
ones = torch.ones(64, device=dev)
slopes = torch.tensor(alibi_slopes(8), dtype=torch.float32, device=dev)
o_h = torch.empty(R, I, dtype=bf, device=dev)
gt = L.AttnGeomT()
gt.n_outer, gt.n_inner, gt.n_q, gt.n_k, gt.heads, gt.dim_head, gt.causal = 8, 64, 9, 9, 8, 64, 1
gt.q_outer, gt.q_inner, gt.q_tok = 9 * 64 * I, I, 64 * I
gt.k_outer, gt.k_inner, gt.k_tok = 9 * 64 * 2 * I, 2 * I, 64 * 2 * I
gt.o_outer, gt.o_inner, gt.o_tok = gt.q_outer, gt.q_inner, gt.q_tok
gt.mask_off_from, gt.scale, gt.out_bf16 = -1, 8.0, 1
timeit("attention temporal (512 seq x 9, warp kernel)", lambda: L.check(lib.phk_attention(L.ptr(q), L.ptr(kv), None, L.ptr(ones), L.ptr(ones), None, None, L.ptr(slopes), L.ptr(o_h), C.byref(gt), sp())))

# the attention core alone on bf16 operands (as the fused q/k,v projection writes them)
qn_h, kvn_h = torch.randn(R, I, device=dev).to(bf), torch.randn(R, 2 * I, device=dev).to(bf)
for (ns, n) in [(72, 64), (8, 576)]:
    bias = torch.randn(8, n, n, device=dev)
    timeit(f"attention tc core ({ns} seq x {n})", lambda: L.check(lib.phk_attention_tc_bf16(L.ptr(qn_h), I, L.ptr(kvn_h), 2 * I, L.ptr(bias), L.ptr(o_h), ns, n, 8, sp())),
           4.0 * ns * 8 * n * n * 64, "TFLOP/s")
bias64 = torch.randn(8, 64, 64, device=dev)
timeit("attention mid mma (72 seq x 64), one CTA per (sequence, head)", lambda: L.check(lib.phk_attention_mid_bf16(L.ptr(qn_h), I, L.ptr(kvn_h), 2 * I, L.ptr(bias64), L.ptr(o_h), 72, 64, 8, sp())),
       4.0 * 72 * 8 * 64 * 64 * 64, "TFLOP/s")

# spatial attention (72 seq x 64) and MaskGit self-attention (8 seq x 576) on tensor cores
for (ns, n) in [(72, 64), (8, 576)]:
    bias = torch.randn(8, n, n, device=dev)
    nb = lib.phk_attention_tc_scratch_bytes(ns, n, 8)
    sc = torch.empty(nb, dtype=torch.uint8, device=dev)
    timeit(f"attention tc prep+core ({ns} seq x {n})", lambda: L.check(lib.phk_attention_tc(L.ptr(q), L.ptr(kv), L.ptr(ones), L.ptr(ones), L.ptr(bias), L.ptr(o_h), ns, n, 8, 8.0, L.ptr(sc), nb, sp())),
           4.0 * ns * 8 * n * n * 64, "TFLOP/s")

# cross attention: 8 sequences x 576 queries, 16 text keys + 2 null
ctx_kv = torch.randn(4 * 16, 2 * I, device=dev)
null_kv = torch.randn(8, 4, 64, device=dev)
tmask = torch.ones(4, 16, dtype=torch.uint8, device=dev)
gc = L.AttnGeomT()
gc.n_outer, gc.n_inner, gc.n_q, gc.n_k, gc.heads, gc.dim_head, gc.num_null_kv = 8, 1, 576, 16, 8, 64, 2
gc.q_outer, gc.q_tok = 576 * I, I
gc.k_outer, gc.k_tok = 16 * 2 * I, 2 * I
gc.o_outer, gc.o_tok = 576 * I, I
gc.kv_outer_mod, gc.mask_outer_mod, gc.mask_off_from, gc.scale, gc.out_bf16 = 4, 4, 4, 8.0, 1
timeit("attention cross (8 seq x 576 q x 18 keys)", lambda: L.check(lib.phk_attention(L.ptr(q), L.ptr(ctx_kv), L.ptr(null_kv), L.ptr(ones), L.ptr(ones), None, L.ptr(tmask), None, L.ptr(o_h), C.byref(gc), sp())))

# PEG
wt, bb = torch.randn(27, D, device=dev), torch.randn(D, device=dev)
y = torch.empty_like(x)
for layout in (0, 1):
    timeit(f"peg3d (8,9,8,8,512) layout {layout}", lambda: L.check(lib.phk_peg3d(L.ptr(x), L.ptr(wt), L.ptr(bb), L.ptr(y), 8, 9, 8, 8, D, 1, layout, sp())),
           R * D * 4 * 4, "TB/s (x read 3x + write)")

# LFQ
wp, bp = torch.randn(16, D, device=dev), torch.randn(16, device=dev)
ids = torch.empty(R, dtype=torch.int64, device=dev)
timeit("lfq ids", lambda: L.check(lib.phk_lfq_ids(L.ptr(x), L.ptr(wp), L.ptr(bp), L.ptr(ids), None, R, D, 16, sp())))

# patchify + LN
video = torch.randn(8, 3, 17, 256, 256, device=dev)
A = torch.empty(4096, 6144, dtype=bf, device=dev)
g2, b2 = torch.randn(6144, device=dev), torch.randn(6144, device=dev)
timeit("patchify_ln rest frames (4096 x 6144 -> bf16)", lambda: L.check(lib.phk_patchify_ln(L.ptr(video), 8, 3, 17, 256, 256, 1, 8, 2, 32, 32, L.ptr(g2), L.ptr(b2), L.ptr(A), 1, sp())),
       4096 * 6144 * 6, "TB/s")

# fused head
emb = torch.randn(2304, 512, device=dev).to(bf)
W = torch.randn(65536, 512, device=dev).to(bf)
hb = torch.randn(65536, device=dev)
mask = torch.ones(2304, dtype=torch.uint8, device=dev)
hid, pred, score = torch.zeros(2304, dtype=torch.int64, device=dev), torch.zeros(2304, dtype=torch.int64, device=dev), torch.zeros(2304, device=dev)
nb = lib.phk_head_sample_scratch_bytes(2304)
sc = torch.empty(nb, dtype=torch.uint8, device=dev)
timeit("fused head 2304 x 65536 x 512", lambda: L.check(lib.phk_head_sample(L.ptr(emb), 512, 2304, L.ptr(W), 512, L.ptr(hb), 2304, 65536, 512, 0.5, 1, 0, L.ptr(mask), L.ptr(hid), L.ptr(pred), L.ptr(score), L.ptr(sc), nb, sp())),
       2.0 * 2304 * 65536 * 512, "TFLOP/s")

# masked-rows tail of the demasking step (csrc/sample_tail.cu) at the row counts of the 18-step schedule, against the
# all-rows head above: compaction + gathered norm_out/CFG + head on b*k rows + scatter
xc, xn_ = torch.randn(2304, 512, device=dev), torch.randn(2304, 512, device=dev)
gm, bt = torch.randn(512, device=dev), torch.randn(512, device=dev)
ids2 = torch.zeros((4, 576), dtype=torch.int64, device=dev)
pred2, score2 = torch.zeros_like(ids2), torch.zeros((4, 576), device=dev)
for k in (574, 441, 288, 100):
    m2 = torch.zeros((4, 576), dtype=torch.uint8, device=dev)
    m2[:, :k] = 1
    nb2 = lib.phk_sample_tail_scratch_bytes(4, k, 512)
    sc2 = torch.empty(nb2, dtype=torch.uint8, device=dev)
    timeit(f"sample tail, {k} of 576 tokens masked (b=4)", lambda: L.check(lib.phk_sample_tail(
        L.ptr(xc), L.ptr(xn_), L.ptr(gm), L.ptr(bt), 3.0, L.ptr(W), 512, L.ptr(hb), 4, 576, k, 65536, 512, 0.5, 1, 0, None,
        L.ptr(m2), L.ptr(ids2), L.ptr(pred2), L.ptr(score2), L.ptr(sc2), nb2, sp())),
        2.0 * 4 * k * 65536 * 512, "TFLOP/s")
