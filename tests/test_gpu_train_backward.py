"""GPU: the rest of the training backward one function at a time, against float64 autograd of an independent statement
of the forward (tests/train_backward_cases.py, bars derived in its docstring), through the probe library of
tests/train_probe.py, in the default and the fixed-order (deterministic) reduction modes:

  E. ln_backward: MaskGit's residual-stream LayerNorms (2304 x 512), the cross-attention context norm (64 x 768,
     dx NULL), the C-ViViT patch-embedding LayerNorms over K = 768 and 1536; too little fixed-order scratch is refused;
  F. geglu_dropout_fwd / geglu_backward at 2304 x 1365, p = 0, 0.1, 1;
  G. peg_backward on MaskGit's (4, 9, 8, 8) x 512 causal grid and a C-ViViT-sized one; D = 1025 is refused;
  H. embed_backward at 2304 x 512 over a 65537-row table;
  I. cpb_backward: MaskGit's (9, 8, 8) grid (U = 3825) and C-ViViT's spatial (8, 8), hidden 512;
  J. ce_rows + loss_reduce on the 288 x 65536 head, bce_rows on 2304 x 512;
plus every edge of tests/train_backward_params.py.  Run with -s to read the worst err / bar of every case."""
import pytest
import torch

from phenaki_pytorch_b200 import _lib as L
from tests import train_backward_cases as BC
from tests import train_backward_params as BP
from tests import train_probe

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")


def sync():
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def lib():
    return train_probe.load()


@pytest.fixture(autouse=True)
def _probe_errors(lib, monkeypatch):
    monkeypatch.setattr(L, "lib", lambda: lib)  # L.check reads the error message from the library that failed


LN = [BP.ln(2304, 512, "acc"), BP.ln(64, 768, None, False), BP.ln(2048, 768, "write"), BP.ln(1024, 1536, "write"),
      BP.ln(2304, 512, "write", False)]


@pytest.mark.parametrize("c", LN + BP.LN_EDGES_GPU, ids=lambda c: c["id"])
def test_layernorm(lib, c):
    BC.check_layernorm(lib, DEV, c, sync)


@pytest.mark.parametrize("rows,dim", [(2304, 512), (257, 33)])
def test_layernorm_refuses_small_scratch(lib, rows, dim):
    BC.check_layernorm_workspace(lib, DEV, rows, dim, sync)


@pytest.mark.parametrize("c", [BP.geglu(2304, 1365, p) for p in (0.0, 0.1, 1.0)] + BP.GEGLU_EDGES,
                         ids=lambda c: c["id"])
def test_geglu(lib, c):
    BC.check_geglu(lib, DEV, c, sync)


@pytest.mark.parametrize("c", [BP.peg(4, 9, 8, 8, 512, True), BP.peg(2, 5, 8, 8, 512, False)] + BP.PEG_EDGES,
                         ids=lambda c: c["id"])
def test_peg(lib, c):
    BC.check_peg(lib, DEV, c, sync)


def test_peg_refuses_dim_1025(lib):
    BC.check_peg_refused(lib, DEV, sync)


@pytest.mark.parametrize("c", [BP.embed(4, 576, 512, 65537, "random"), BP.embed(4, 576, 512, 65537, "mask")]
                         + BP.EMBED_EDGES, ids=lambda c: c["id"])
def test_embed(lib, c):
    BC.check_embed(lib, DEV, c, sync)


@pytest.mark.parametrize("c", [BP.cpb((9, 8, 8), 512, 8), BP.cpb((8, 8), 512, 8)] + BP.CPB_EDGES,
                         ids=lambda c: c["id"])
def test_cpb(lib, c):
    BC.check_cpb(lib, DEV, c, sync)


@pytest.mark.parametrize("c", [BP.ce(288, 65536, "partial"), BP.ce(288, 65536, "all", 0.25), BP.ce(288, 1000, "none")]
                         + BP.CE_EDGES, ids=lambda c: c["id"])
def test_ce(lib, c):
    BC.check_ce(lib, DEV, c, sync)


@pytest.mark.parametrize("c", [BP.bce(2304, 512, 1.0)] + BP.BCE_EDGES, ids=lambda c: c["id"])
def test_bce(lib, c):
    BC.check_bce(lib, DEV, c, sync)
