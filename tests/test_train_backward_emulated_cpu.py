"""CPU (tests/cuda_emu): the check bodies of tests/train_backward_cases.py on the CPU executor, at reduced sizes plus
every edge of tests/train_backward_params.py -- LayerNorm (E), GEGLU with dropout (F), PEG (G), the embeddings (H), the
position-bias MLP (I) and the head losses (J), each against float64 autograd with the bars of that module, in the
default and the fixed-order (deterministic) reduction modes.  Run with -s to read the worst err / bar of every case."""
import pytest
import torch

from phenaki_pytorch_b200 import _lib as L
from tests import train_backward_cases as BC
from tests import train_backward_params as BP
from tests import train_probe

CPU = torch.device("cpu")


def _sync():
    pass


@pytest.fixture(scope="module")
def lib():
    return train_probe.load_emulated()


@pytest.fixture(autouse=True)
def _cpu(lib, monkeypatch):
    monkeypatch.setattr(L, "lib", lambda: lib)  # L.check reads the error message from the library that failed
    monkeypatch.setattr(L, "stream_ptr", lambda: None)


@pytest.mark.parametrize("c", BP.LN_EDGES + [BP.ln(64, 512, "acc")], ids=lambda c: c["id"])
def test_layernorm(lib, c):
    BC.check_layernorm(lib, CPU, c, _sync)


@pytest.mark.parametrize("rows,dim", [(257, 33), (7, 512)])
def test_layernorm_refuses_small_scratch(lib, rows, dim):
    BC.check_layernorm_workspace(lib, CPU, rows, dim, _sync)


@pytest.mark.parametrize("c", BP.GEGLU_EDGES, ids=lambda c: c["id"])
def test_geglu(lib, c):
    BC.check_geglu(lib, CPU, c, _sync)


@pytest.mark.parametrize("c", BP.PEG_EDGES, ids=lambda c: c["id"])
def test_peg(lib, c):
    BC.check_peg(lib, CPU, c, _sync)


def test_peg_refuses_dim_1025(lib):
    BC.check_peg_refused(lib, CPU, _sync)


@pytest.mark.parametrize("c", BP.EMBED_EDGES, ids=lambda c: c["id"])
def test_embed(lib, c):
    BC.check_embed(lib, CPU, c, _sync)


@pytest.mark.parametrize("c", BP.CPB_EDGES, ids=lambda c: c["id"])
def test_cpb(lib, c):
    BC.check_cpb(lib, CPU, c, _sync)


@pytest.mark.parametrize("c", BP.CE_EDGES, ids=lambda c: c["id"])
def test_ce(lib, c):
    BC.check_ce(lib, CPU, c, _sync)


@pytest.mark.parametrize("c", BP.BCE_EDGES, ids=lambda c: c["id"])
def test_bce(lib, c):
    BC.check_bce(lib, CPU, c, _sync)
