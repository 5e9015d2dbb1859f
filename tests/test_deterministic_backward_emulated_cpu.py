"""CPU: torch.use_deterministic_algorithms(True) makes every hand-written backward bit-reproducible.  The CPU executor of
tests/cuda_emu runs the blocks of every launch in a seeded random order (phk_emu_set_shuffle), which changes the order in
which float atomics land.  In deterministic mode every gradient of the five backward entry points must not change with
that order, and must stay within the float64 bars of the existing gradient tests.  With the mode off, some gradient
does change with it, so the comparison has teeth.  The workspace queries grow only in deterministic mode, and a
workspace one byte short of what they return is refused before anything is launched."""
import ctypes
import json
import os
import subprocess
import sys

import pytest
import torch

from phenaki_pytorch_b200 import _lib as L
from phenaki_pytorch_b200.modules import GradKeep
from tests import deterministic_cases as DC
from tests import emu_runtime
from tests import encode_grad_cases as EG
from tests import text_grad_cases as TG

DEV = "cpu"
SEEDS = (0, 1, 2)


@pytest.fixture(scope="module")
def emu():
    return emu_runtime.build_emu()


@pytest.fixture
def on_cpu(emu, monkeypatch):
    emu_runtime.route_product_to_emulator(emu, monkeypatch)
    yield emu
    emu.phk_emu_set_shuffle(0)


def _runs(emu, run, seeds=SEEDS, warn_only_last=False):
    """One gradient run per executor seed; warn_only_last: the last run under warn_only=True (counted as on)."""
    out = []
    for i, s in enumerate(seeds):
        emu.phk_emu_set_shuffle(s)
        with DC.deterministic(torch.are_deterministic_algorithms_enabled(), warn_only=warn_only_last and i == len(seeds) - 1):
            out.append(run.grads())
    emu.phk_emu_set_shuffle(0)
    return out


ENTRIES = {
    # Phenaki.forward(...).backward(): a cross-attention TokenCritic, dropout, text_embeds.requires_grad
    "train_step_dropout": lambda: DC.TrainStep(TG.SMALL["token_critic"], 0.2, DEV),
    # f(critic(ids, text_embeds)).backward(): cross-attention with null key / values
    "maskgit_backward_critic": lambda: DC.ForwardBackward("emu_critic", DEV),
    "decode_backward_ids": lambda: DC.Decode("rect", "ids", DEV),
    "encode_backward": lambda: DC.Encode("rect", DEV),
    "recon_backward": lambda: DC.Recon("image", DEV),
}


@pytest.mark.parametrize("name", list(ENTRIES))
def test_deterministic_mode_gradients_do_not_depend_on_the_block_order(on_cpu, name):
    run = ENTRIES[name]()
    with DC.deterministic():
        # warn_only=True behaves as True: the third run takes it
        DC.assert_bitwise_equal(name, _runs(on_cpu, run, warn_only_last=True))
        run.check_bars(name)  # and the deterministic path computes what the float64 reference does


def test_default_mode_gradients_do_depend_on_the_block_order(on_cpu):
    """The comparison above has teeth: with the switch off the atomics land in the shuffled order and some gradient
    changes (the executor is deterministic for a fixed seed, so this is not flaky)."""
    run = ENTRIES["maskgit_backward_critic"]()
    with DC.deterministic(False):
        runs = _runs(on_cpu, run, seeds=(1, 2))
    assert DC.differing(runs), "no gradient depends on the block order with the switch off"


def _queries():
    return {k: q for k, q in DC.workspace_queries(DEV).items() if not k.startswith("_")}


def test_workspace_queries_grow_only_in_deterministic_mode(on_cpu):
    lib = L.lib()
    qs = DC.workspace_queries(DEV)
    prev = lib.phk_train_set_deterministic(0)
    try:
        off = {k: q() for k, q in qs.items() if not k.startswith("_")}
        assert lib.phk_train_set_deterministic(1) == 0
        on = {k: q() for k, q in qs.items() if not k.startswith("_")}
        assert lib.phk_train_set_deterministic(0) == 1
        again = {k: q() for k, q in qs.items() if not k.startswith("_")}
    finally:
        lib.phk_train_set_deterministic(prev)
    assert all(v > 0 for v in off.values()), off
    assert again == off
    for k in off:
        assert on[k] > off[k], f"{k}: {on[k]} in deterministic mode, {off[k]} without"


def test_default_mode_queries_match_a_process_that_never_set_the_mode(on_cpu):
    """The queries of the default mode do not depend on whether the setter was ever called in the process."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = ("import sys, json; sys.path.insert(0, %r); from tests import emu_runtime, deterministic_cases as DC; "
            "from phenaki_pytorch_b200 import _lib as L; lib = emu_runtime.build_emu(); emu_runtime.route_product_to_emulator(lib); "
            "qs = DC.workspace_queries('cpu'); "
            "print(json.dumps({k: q() for k, q in qs.items() if not k.startswith('_')}))") % root
    fresh = subprocess.run([sys.executable, "-c", code], check=True, capture_output=True, text=True).stdout
    want = json.loads(fresh.strip().splitlines()[-1])
    lib = L.lib()
    prev = lib.phk_train_set_deterministic(1)
    lib.phk_train_set_deterministic(0)
    try:
        got = {k: q() for k, q in _queries().items()}
    finally:
        lib.phk_train_set_deterministic(prev)
    assert got == want


def test_deterministic_mode_refuses_a_workspace_one_byte_short(on_cpu):
    """phk_cvivit_encode_backward in deterministic mode with one byte less than its query returned in that mode:
    PHK_E_WORKSPACE, and nothing launched."""
    lib = L.lib()
    module = DC.DG.build_module("rect")
    tok = EG.inputs("rect")
    b, tp = tok.shape[:2]
    table = module._table()
    gk = GradKeep(module._encode_params())
    gtable = module._enc_grad_table(gk, False)
    out = torch.zeros_like(tok)
    prev = lib.phk_train_set_deterministic(1)
    try:
        need = lib.phk_cvivit_encode_backward_workspace_bytes(ctypes.byref(table), b, tp, L.PREC_F32)
        ws = torch.zeros(need, dtype=torch.uint8)
        before = lib.phk_launch_count()
        rc = lib.phk_cvivit_encode_backward(ctypes.byref(table), ctypes.byref(gtable), L.ptr(tok), b, tp, L.ptr(tok),
                                            L.ptr(out), L.ptr(ws), need - 1, L.PREC_F32, None)
        assert rc == EG.PHK_E_WORKSPACE, rc
        assert lib.phk_launch_count() == before, "a refused call launched kernels"
        assert not out.any() and not gk.flat.any(), "a refused call wrote its outputs"
    finally:
        lib.phk_train_set_deterministic(prev)
