"""GPU: every attention forward kernel (csrc/attention.cu, csrc/attention_tc.cu) against the float64 reference and the
per-element error bound of tests/attention_ref.py, with the exact census / dominant-key probes and the NaN-padding /
sentinel checks of tests/attention_cases.py.

DISPATCH lists, for each entry point, the conditions host code picks a kernel by -- sequence length (SMALL_N 16, MID_N
64, the 64-token tiles and key chunks), key slots (XK 32 for the cross MMA kernel, FEW_KEYS 64), dim_head, out_bf16,
strides and alignment -- with cases on both sides of each boundary.  Every case names the kernel it must reach and the
test checks the name in the torch.profiler kernel trace (CUDA activity only), so a change of a dispatch condition cannot
silently move a case to another kernel."""
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

from phenaki_pytorch_b200 import _lib as L
from tests import attention_cases as AC

pytestmark = pytest.mark.gpu
DEV = "cuda"


def sync():
    torch.cuda.synchronize()


W64, ROWS, SMALL = "attention_warp64_kernel<{}, {}>", "attention_rows_kernel<{}, {}>", "attention_small_kernel<{}, {}>"
GEN, FEW = "attention_kernel<{}>", "attention_fewkeys_kernel<{}>"
CROSS, SMMA, MID, TC = "attention_cross_mma_kernel", "attention_small_mma_kernel", "attention_mid_mma_kernel", "attention_tc_kernel"
PACKED = ("cross_kv_pack_kernel", "attention_cross_packed_kernel")


def _a(kernel, **kw):
    return dict(entry="attention", kernel=kernel, **kw)


DISPATCH = [
    # phk_attention, self-attention n_q == n_k <= 16, no null keys / bias / mask: warp64 (dim_head 64, aligned), rows
    # (dim_head 32, aligned), small_n (unaligned strides: q_tok = I + 1)
    _a(W64.format(3, "false"), n_outer=5, n_q=1, heads=3),
    _a(W64.format(3, "false"), n_outer=4, n_inner=3, n_q=3, heads=2, causal=True, temporal=True),
    _a(W64.format(5, "false"), n_outer=6, n_q=4, heads=2, out_bf16=1),
    _a(W64.format(5, "false"), n_outer=3, n_inner=2, n_q=5, heads=4, causal=True, temporal=True),
    _a(W64.format(9, "false"), n_outer=8, n_inner=16, n_q=9, heads=8, causal=True, temporal=True, out_bf16=1),
    _a(W64.format(12, "false"), n_outer=5, n_q=12, heads=2, pad_o=8),
    _a(W64.format(16, "false"), n_outer=4, n_q=16, heads=3, causal=True),
    _a(GEN.format(64), n_outer=3, n_q=17, heads=2, causal=True),                           # n = 17 > SMALL_N
    _a(FEW.format(64), n_outer=3, n_q=17, heads=2),                                        # n = 17, 17 keys, not causal
    _a(ROWS.format(32, 3), n_outer=9, n_q=3, heads=2, dh=32, causal=True),
    _a(ROWS.format(32, 5), n_outer=7, n_q=5, heads=3, dh=32),
    _a(ROWS.format(32, 9), n_outer=4, n_inner=5, n_q=9, heads=2, dh=32, causal=True, temporal=True),
    _a(ROWS.format(32, 12), n_outer=5, n_q=12, heads=2, dh=32, out_bf16=1),
    _a(ROWS.format(32, 16), n_outer=5, n_q=16, heads=2, dh=32, causal=True),
    _a(SMALL.format(64, 3), n_outer=5, n_q=3, heads=2, pad_q=1, causal=True),
    _a(SMALL.format(64, 9), n_outer=3, n_inner=4, n_q=9, heads=2, pad_q=1, causal=True, temporal=True),
    _a(SMALL.format(64, 16), n_outer=4, n_q=16, heads=2, pad_q=1, out_bf16=1),
    _a(SMALL.format(32, 5), n_outer=4, n_q=5, heads=3, dh=32, pad_q=1),
    _a(SMALL.format(32, 12), n_outer=4, n_q=12, heads=2, dh=32, pad_q=1, causal=True),
    # phk_attention, key slots = null + text: the cross MMA kernel (bf16 output, null keys, <= XK = 32 slots), fewkeys
    # (<= FEW_KEYS = 64 slots), the generic kernel above
    _a(FEW.format(64), n_outer=3, n_q=40, n_k=1, heads=2),                                 # 0 + 1
    _a(FEW.format(64), n_outer=3, n_q=40, n_k=1, heads=2, out_bf16=1),
    _a(CROSS, n_outer=4, n_q=130, n_k=0, heads=2, nnull=2, ctx_b=2, out_bf16=1),          # 2 + 0: a context of length 0
    _a(FEW.format(64), n_outer=4, n_q=130, n_k=0, heads=2, nnull=2, ctx_b=2),
    _a(CROSS, n_outer=4, n_q=130, n_k=30, heads=3, nnull=2, mask=True, ctx_b=2, cfg=True, out_bf16=1),   # 2 + 30
    _a(FEW.format(64), n_outer=4, n_q=130, n_k=30, heads=3, nnull=2, mask=True, ctx_b=2, cfg=True),
    _a(FEW.format(64), n_outer=4, n_q=130, n_k=31, heads=2, nnull=2, mask=True, ctx_b=2, cfg=True, out_bf16=1),  # 2 + 31
    _a(FEW.format(64), n_outer=4, n_q=129, n_k=31, heads=2, nnull=2, ctx_b=2, cfg=True),  # CFG half without a key mask
    _a(FEW.format(64), n_outer=4, n_q=200, n_k=62, heads=2, nnull=2, mask=True, ctx_b=2, cfg=True, out_bf16=1),  # 2 + 62
    _a(FEW.format(64), n_outer=2, n_q=70, n_k=62, heads=2, nnull=2, ctx_b=2),
    _a(FEW.format(32), n_outer=2, n_q=70, n_k=30, heads=2, dh=32, nnull=2, mask=True, ctx_b=2, out_bf16=1),
    _a(GEN.format(64), n_outer=4, n_q=130, n_k=63, heads=2, nnull=2, mask=True, ctx_b=2, cfg=True, out_bf16=1),  # 2 + 63
    _a(GEN.format(64), n_outer=2, n_q=65, n_k=63, heads=2, nnull=2, ctx_b=2),
    # phk_attention, the generic kernel: dim_head 16 / 32 / 64 / 128, null keys across the first 64-key chunk, causal with
    # n_q < n_k (row_shift), bias + key mask with bf16 output (MaskGit with a video frame mask), strided rows
    _a(GEN.format(16), n_outer=2, n_q=129, heads=2, dh=16, bias=True),
    _a(GEN.format(32), n_outer=2, n_q=65, heads=3, dh=32, bias=True, out_bf16=1),
    _a(GEN.format(64), n_outer=2, n_q=100, heads=2, bias=True, pad_q=4, pad_k=4, pad_o=4),
    _a(GEN.format(128), n_outer=2, n_q=70, heads=2, dh=128, bias=True, mask=True),
    _a(GEN.format(64), n_outer=2, n_q=9, n_k=10, heads=2, nnull=70),
    _a(GEN.format(64), n_outer=2, n_q=20, n_k=100, heads=2, causal=True),
    _a(GEN.format(64), n_outer=1, n_q=65, n_k=129, heads=2, causal=True, out_bf16=1),
    _a(GEN.format(64), n_outer=3, n_q=130, heads=2, bias=True, mask=True, out_bf16=1),
    # phk_attention_small_bf16: the MMA kernel (bf16 output, 16-byte rows), the warp64 PRE fallback otherwise
    dict(entry="small_bf16", kernel=SMMA, n_outer=4, n_inner=8, n_q=9, heads=4, causal=True, temporal=True),
    dict(entry="small_bf16", kernel=SMMA, n_outer=5, n_q=1, heads=2),
    dict(entry="small_bf16", kernel=SMMA, n_outer=3, n_q=16, heads=3, pad_o=8),
    dict(entry="small_bf16", kernel=W64.format(9, "true"), n_outer=4, n_inner=2, n_q=9, heads=2, causal=True, temporal=True,
         out_bf16=0),
    dict(entry="small_bf16", kernel=W64.format(16, "true"), n_outer=3, n_q=13, heads=2, pad_q=2, causal=True),
    dict(entry="small_bf16", kernel=W64.format(3, "true"), n_outer=3, n_q=2, heads=2, pad_q=2),
    # phk_attention_mid_bf16 (16 < n <= 64), phk_attention_tc_bf16 / phk_attention_tc (n >= 64, 64-token tiles and chunks)
    dict(entry="mid_bf16", kernel=MID, n_outer=3, n_q=17, heads=2, bias=True),
    dict(entry="mid_bf16", kernel=MID, n_outer=3, n_q=31, heads=3, bias=True, pad_q=8, pad_k=8),
    dict(entry="mid_bf16", kernel=MID, n_outer=3, n_q=33, heads=2),
    dict(entry="mid_bf16", kernel=MID, n_outer=2, n_q=63, heads=2, bias=True),
    dict(entry="mid_bf16", kernel=MID, n_outer=2, n_q=64, heads=1, bias=True),
    dict(entry="tc_bf16", kernel=TC, n_outer=2, n_q=64, heads=1, bias=True),
    dict(entry="tc_bf16", kernel=TC, n_outer=2, n_q=65, heads=3, bias=True),
    dict(entry="tc_bf16", kernel=TC, n_outer=2, n_q=127, heads=3, bias=True, pad_q=8),
    dict(entry="tc_bf16", kernel=TC, n_outer=2, n_q=128, heads=1),
    dict(entry="tc_bf16", kernel=TC, n_outer=2, n_q=129, heads=8, bias=True, pad_q=16, pad_k=8),
    dict(entry="tc_bf16", kernel=TC, n_outer=1, n_q=1024, heads=3, bias=True),
    dict(entry="tc_bf16", kernel=TC, n_outer=1, n_q=1025, heads=1, bias=True),
    dict(entry="tc", kernel=("attention_prep_kernel", TC), n_outer=2, n_q=129, heads=3, bias=True),
    dict(entry="tc", kernel=("attention_prep_kernel", TC), n_outer=1, n_q=576, heads=2),
    # phk_cross_kv_pack + phk_attention_cross_packed: L = 0, 1, 29, 30 with 2 null keys, 1 to 3 layers, CFG null half
    dict(entry="cross_packed", kernel=PACKED, ctx_b=2, n_q=130, n_k=0, heads=2, nnull=2, layers=1, cfg=True),
    dict(entry="cross_packed", kernel=PACKED, ctx_b=3, n_q=64, n_k=1, heads=2, nnull=2, layers=2, mask=True),
    dict(entry="cross_packed", kernel=PACKED, ctx_b=2, n_q=129, n_k=29, heads=3, nnull=2, layers=3, mask=True, cfg=True,
         pad_q=8, pad_o=8),
    dict(entry="cross_packed", kernel=PACKED, ctx_b=2, n_q=200, n_k=30, heads=2, nnull=2, layers=2, mask=True, cfg=True),
]

PRODUCTION = [
    dict(entry="tc_bf16", kernel=TC, n_outer=8, n_q=576, heads=8, bias=True),       # MaskGit self-attention, b = 4 x 2
    dict(entry="mid_bf16", kernel=MID, n_outer=72, n_q=64, heads=8, bias=True),     # C-ViViT spatial: 72 frames x 8 x 8
    dict(entry="small_bf16", kernel=SMMA, n_outer=8, n_inner=1024, n_q=9, heads=8, causal=True, temporal=True),  # temporal
]


def _id(c):
    k = c["kernel"] if isinstance(c["kernel"], str) else c["kernel"][-1]
    keys = ("n_outer", "n_q", "n_k", "nnull", "dh", "heads", "causal", "bias", "mask", "cfg", "out_bf16", "pad_q", "layers")
    return c["entry"] + ":" + k.replace(" ", "") + "-" + "-".join(f"{x}{int(c[x])}" for x in keys if x in c)


def _phk_kernels(prof):
    """Names of the project's kernels in the CUDA activity trace, without the 'void phk::...' prefix and arguments."""
    names = set()
    for e in prof.events():
        name = e.name.replace("(anonymous namespace)::", "")
        if "phk::" in name:
            names.add(name.split("(")[0].replace("void ", "").replace("phk::", "").strip())
    return names


def run_observed(case, modes):
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        result = AC.check(L.lib(), DEV, case, sync, modes=modes)
    return result, _phk_kernels(prof)


@pytest.mark.parametrize("case", DISPATCH, ids=_id)
def test_attention_forward_kernel_matches_fp64_reference(case):
    result, seen = run_observed(case, AC.MODES)
    assert seen == AC.kernels_of(case), f"expected {sorted(AC.kernels_of(case))}, the trace shows {sorted(seen)}"
    print(f"{_id(case)}: worst err / bound {result}")


@pytest.mark.parametrize("case", PRODUCTION, ids=_id)
def test_attention_forward_production_shapes(case):
    result, seen = run_observed(case, ("random", "census"))
    assert seen == AC.kernels_of(case), f"expected {sorted(AC.kernels_of(case))}, the trace shows {sorted(seen)}"
    print(f"{_id(case)}: worst err / bound {result}")


def test_dispatch_table_reaches_every_kernel():
    """One small random-mode run per row of DISPATCH, in this test alone (independent of test order and -k): each row
    runs exactly the kernels it names, and together the rows reach every kernel the table lists."""
    listed, observed = set(), set()
    for case in DISPATCH:
        _, seen = run_observed(case, ("random",))
        assert seen == AC.kernels_of(case), f"{_id(case)}: expected {sorted(AC.kernels_of(case))}, the trace shows {sorted(seen)}"
        listed |= AC.kernels_of(case)
        observed |= seen
    assert observed == listed
    print("worst err / bound per kernel:", {k: round(v, 4) for k, v in sorted(AC.WORST.items())})
