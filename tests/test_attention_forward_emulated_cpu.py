"""CPU (tests/cuda_emu): the attention-forward check bodies of tests/attention_cases.py on the kernels the CPU executor
compiles from csrc/attention.cu -- the generic kernel, warp64, rows, small_n, fewkeys and the PRE fallback of
phk_attention_small_bf16 -- at scaled-down shapes, so the float64 reference, the error bounds and the exact probes are
exercised without a GPU.  Without the tensor-core kernels the executor routes the bf16 cross-attention to fewkeys and
phk_attention_small_bf16 to its warp64 PRE fallback; the cases below name the kernel the executor runs."""
import pytest
import torch

from oracle import phenaki_oracle as O
from phenaki_pytorch_b200 import _lib as L
from tests import attention_cases as AC
from tests import attention_ref as R
from tests import emu_runtime

CPU = torch.device("cpu")


def _sync():
    pass


@pytest.fixture(scope="module")
def lib():
    return emu_runtime.build_emu()


@pytest.fixture(autouse=True)
def _cpu(lib, monkeypatch):
    monkeypatch.setattr(L, "stream_ptr", lambda: None)


W64 = "attention_warp64_kernel<{}, {}>"
CASES = [
    dict(entry="attention", kernel=W64.format(9, "false"), n_outer=2, n_inner=3, n_q=9, heads=2, causal=True, temporal=True),
    dict(entry="attention", kernel=W64.format(3, "false"), n_outer=3, n_q=1, heads=2, out_bf16=1),
    dict(entry="attention", kernel=W64.format(16, "false"), n_outer=2, n_q=16, heads=2, causal=True, pad_o=8),
    dict(entry="attention", kernel="attention_rows_kernel<32, 5>", n_outer=3, n_q=5, heads=2, dh=32, causal=True),
    dict(entry="attention", kernel="attention_rows_kernel<32, 16>", n_outer=2, n_q=16, heads=3, dh=32, out_bf16=1),
    dict(entry="attention", kernel="attention_small_kernel<64, 12>", n_outer=2, n_q=12, heads=2, pad_q=1, causal=True),
    dict(entry="attention", kernel="attention_small_kernel<32, 3>", n_outer=2, n_q=3, heads=2, dh=32, pad_q=1),
    # cross-attention: null keys + text; the executor has no MMA kernel, so the bf16 output also takes fewkeys
    dict(entry="attention", kernel="attention_fewkeys_kernel<64>", n_outer=4, n_q=40, n_k=30, heads=2, nnull=2, mask=True,
         ctx_b=2, cfg=True, out_bf16=1),
    dict(entry="attention", kernel="attention_fewkeys_kernel<64>", n_outer=4, n_q=20, n_k=62, heads=2, nnull=2, ctx_b=2,
         cfg=True),  # CFG half without a key mask: the text keys stay live
    dict(entry="attention", kernel="attention_fewkeys_kernel<64>", n_outer=2, n_q=20, n_k=0, heads=2, nnull=2, ctx_b=2,
         out_bf16=1),  # a text context of length 0
    dict(entry="attention", kernel="attention_fewkeys_kernel<32>", n_outer=2, n_q=140, n_k=1, heads=2, dh=32),
    dict(entry="attention", kernel="attention_kernel<64>", n_outer=4, n_q=70, n_k=63, heads=2, nnull=2, mask=True, ctx_b=2,
         cfg=True, out_bf16=1),
    dict(entry="attention", kernel="attention_kernel<64>", n_outer=1, n_q=20, n_k=70, heads=2, causal=True, pad_q=4),
    dict(entry="attention", kernel="attention_kernel<16>", n_outer=2, n_q=70, heads=2, dh=16, bias=True, mask=True, out_bf16=1),
    dict(entry="attention", kernel="attention_kernel<128>", n_outer=1, n_q=17, heads=2, dh=128, bias=True, pad_k=4),
    dict(entry="attention", kernel="attention_kernel<32>", n_outer=1, n_q=9, n_k=10, heads=2, dh=32, nnull=70),
    dict(entry="small_bf16", kernel=W64.format(9, "true"), n_outer=2, n_inner=2, n_q=9, heads=2, causal=True, temporal=True),
    dict(entry="small_bf16", kernel=W64.format(5, "true"), n_outer=3, n_q=4, heads=2, out_bf16=0),
]


def _id(c):
    keys = ("n_q", "n_k", "nnull", "dh", "causal", "bias", "mask", "cfg", "out_bf16", "pad_q")
    return c["kernel"].replace(" ", "") + "-" + "-".join(f"{k}{int(c[k])}" for k in keys if k in c)


@pytest.mark.parametrize("case", CASES, ids=_id)
def test_attention_forward_matches_fp64_reference(lib, case):
    AC.check(lib, CPU, case, _sync)


def test_reference_is_the_oracle_core():
    """The prenormalised float64 core the bounds are computed from equals oracle.attention_core in float64 on the same
    operands (null keys, a key mask, the CFG null half, bias, causal ALiBi with n_q < n_k)."""
    for case in (dict(entry="attention", kernel="attention_kernel<64>", n_outer=4, n_q=7, n_k=9, heads=3, nnull=2, mask=True,
                      ctx_b=2, cfg=True, bias=True),
                 dict(entry="attention", kernel="attention_kernel<64>", n_outer=2, n_q=5, n_k=11, heads=2, causal=True)):
        c, P = AC.make_problem(case, "random", 5)
        q, k, v, qh, kh, live, bias = AC.reference_operands(c, P, 0, torch.arange(P.S))
        o_oracle = R.oracle_core(q, k, v, P.q_scale, P.k_scale[0], live, bias, P.scale)
        o_pre = R.prenormalised_core(qh, kh, v, live, bias)[0]
        assert torch.allclose(o_oracle, o_pre, rtol=0, atol=1e-12)
    # and the causal fold equals the oracle's own causal path with its ALiBi slopes
    c, P = AC.make_problem(dict(entry="attention", kernel="attention_kernel<64>", n_outer=2, n_q=6, n_k=6, heads=4,
                                causal=True), "random", 6)
    q, k, v, _, _, live, bias = AC.reference_operands(c, P, 0, torch.arange(P.S))
    want = O.attention_core(q, k, v, P.q_scale.double(), P.k_scale[0].double(), heads=4, causal=True)
    got = R.oracle_core(q, k, v, P.q_scale, P.k_scale[0], live, bias, P.scale)
    assert torch.allclose(want, got, rtol=0, atol=1e-12)


def test_census_values_are_balanced():
    g = torch.Generator().manual_seed(0)
    live = torch.rand((50, 64, 37), generator=g) < 0.6
    live[:, :, 0] = True
    v = AC.balanced(live, g)
    s = torch.where(live, v, torch.zeros_like(v)).sum(-1)
    assert bool((s.abs() <= 2).all()) and bool((s != 0).any())
    assert bool((v[~live] == AC.CENSUS_DEAD).all()) and bool(v[live].abs().le(1).all())
    assert bool((v[live] != 0).float().mean() > 0.2)  # pairs, not an all-zero column


def test_bound_is_tight_enough_to_see_one_key():
    """At n = 576 keys one key carries ~1/576 of the weight; the bf16-operand bound must sit below that on random data,
    or the random mode could not see a dropped or doubled key."""
    c, P = AC.make_problem(dict(entry="tc_bf16", kernel="attention_tc_kernel", n_outer=1, n_q=576, heads=2), "random", 1)
    _, _, v, qh, kh, live, bias = AC.reference_operands(c, P, 0, torch.arange(1))
    o, bnd = R.bound(AC.model("attention_tc_kernel", True), qh, kh, v, live, bias)
    a = R.prenormalised_core(qh, kh, v, live, bias)[1]
    one_key = (a.unsqueeze(-1) * (v.unsqueeze(2) - o.unsqueeze(3)).abs()).amax(dim=3)  # max_j a_ij |v_jd - o_id|
    assert float(bnd.median()) < float(one_key.median())
