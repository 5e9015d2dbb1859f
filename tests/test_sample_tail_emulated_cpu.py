"""CPU (tests/cuda_emu): the masked-rows-only tail of a demasking iteration (csrc/sample_tail.cu: compaction, gathered
norm_out + guidance, head on the compact rows, scatter) executed from the shipped source, against plain torch
arithmetic.  The wgmma head itself (phk_head_sample) is represented by its contract here -- a bf16-operand product
followed by the REAL phk_sample_tokens kernel; on the H100 the same checks run through the real head
(tests/test_gpu_zz_after_last_gpu_call.py)."""
import pytest
import torch

from phenaki_pytorch_b200 import _lib as L
from tests import emu_runtime
from tests import tail_cases as T


@pytest.fixture(scope="module")
def lib():
    return emu_runtime.build_emu()


@pytest.fixture(autouse=True)
def _cpu(lib, monkeypatch):
    monkeypatch.setattr(L, "stream_ptr", lambda: None)
    monkeypatch.setattr(L, "lib", lambda: lib)


@pytest.mark.parametrize("b,n,k,dim,V", [(2, 48, 17, 128, 300), (3, 30, 1, 256, 130), (1, 300, 299, 128, 70), (2, 18, 9, 512, 64)])
def test_tail_on_exactly_k_masked_tokens(lib, b, n, k, dim, V):
    T.check_exact_k(lib, torch.device("cpu"), b, n, k, dim, V)


def test_tail_tolerates_a_mask_that_breaks_the_count_contract(lib):
    """Fewer set entries than k: all of them are served (the padding rows are ignored); more: the first k in order."""
    b, n, k, dim, V = 2, 40, 10, 128, 90
    xc, xn, gamma, beta, W, bias, mask, ids0 = T.make_inputs(b, n, k, dim, V, 7, torch.device("cpu"))
    mask[0] = 0
    mask[0, [3, 8, 30]] = 1                 # 3 < k
    mask[1] = 0
    mask[1, 5:20] = 1                       # 15 > k
    ids = ids0.clone()
    pred, score = T.run_tail(lib, xc, xn, gamma, beta, W, bias, mask, ids, b=b, n=n, k=k, V=V, dim=dim, scale=2.0,
                             temperature=0.0)
    rp, _, _ = T.reference(xc, xn, gamma, beta, W, bias, 2.0)
    rp = rp.reshape(b, n)
    assert torch.equal(ids[0, [3, 8, 30]], rp[0, [3, 8, 30]])
    untouched = torch.ones(n, dtype=torch.bool)
    untouched[[3, 8, 30]] = False
    assert torch.equal(ids[0, untouched], ids0[0, untouched])
    assert torch.equal(ids[1, 5:15], rp[1, 5:15]) and torch.equal(ids[1, 15:], ids0[1, 15:])
    assert bool((score[1, 15:] == -1e4).all())


def test_tail_sampling_is_seeded(lib):
    b, n, k, dim, V = 2, 32, 12, 128, 200
    args = T.make_inputs(b, n, k, dim, V, 9, torch.device("cpu"))
    outs = []
    for seed in (3, 3, 4):
        ids = args[7].clone()
        T.run_tail(lib, *args[:7], ids, b=b, n=n, k=k, V=V, dim=dim, scale=3.0, temperature=0.9, seed=seed)
        outs.append(ids)
    assert torch.equal(outs[0], outs[1]) and not torch.equal(outs[0], outs[2])
    assert bool(((outs[0] >= 0) & (outs[0] < V)).all())
