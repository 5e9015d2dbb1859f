"""Shared bodies of the deterministic-mode tests (torch.use_deterministic_algorithms(True) -> phk_train_set_deterministic):
one gradient run per backward entry point, on the case modules of the existing gradient tests, returning every gradient
it produces (parameters, text embeddings, tokens, video) so that runs can be compared bit for bit."""
import contextlib

import torch

from phenaki_pytorch_b200 import _lib as L
from tests import cases as C
from tests import decode_grad_cases as DG
from tests import encode_grad_cases as EG
from tests import forward_grad_cases as FG
from tests import recon_loss_cases as RL
from tests import text_grad_cases as TG
from tests import train_at_size_cases as T


@contextlib.contextmanager
def deterministic(on=True, warn_only=False):
    """torch.use_deterministic_algorithms(on) for the block, restored afterwards."""
    was, was_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on, warn_only=warn_only)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=was_warn)


def _set_train_precision(phenaki, precision):
    phenaki.maskgit.precision = precision
    if isinstance(phenaki.critic, torch.nn.Module) and hasattr(phenaki.critic, "precision"):
        phenaki.critic.precision = precision


class TrainStep:
    """Phenaki.forward(...).backward() through phk_maskgit_train_step, with text_embeds.requires_grad."""

    def __init__(self, case, dropout, device):
        self.case, self.device = case, device
        self.module = TG.build(case, dropout=dropout, device=device)
        self.draws = TG.decisive_draws(case)

    def grads(self, precision=L.PREC_F32):
        _set_train_precision(self.module, precision)
        ids, ctx = C.train_inputs(self.case)
        torch.manual_seed(1234)  # the same dropout masks every run
        loss, grads, e_grad = TG.product(self.module, ids, ctx, self.draws)
        return dict(grads, text_embeds=e_grad, loss=loss)

    def check_bars(self, name):
        """The loss and every gradient against the float64 reference at the fp32 parity bars."""
        torch.manual_seed(1234)
        _set_train_precision(self.module, L.PREC_F32)
        loss, grads, e_grad, ref = TG.run_and_reference(self.case, self.module, self.draws,
                                                        ref_device=self.device if self.device != "cpu" else "cpu")
        return TG.check(name, loss, grads, e_grad, ref)


class ForwardBackward:
    """f(maskgit(...)).backward() through phk_maskgit_backward."""

    def __init__(self, name, device):
        self.name, self.device = name, device
        self.module = T.build_module(FG.ALL_CASES[name]["base"]).to(device)

    def grads(self, precision=L.PREC_F32):
        return FG.product_grads(self.name, self.module, self.device, precision)

    def check_bars(self, name):
        return FG.check_fp32(None, self.device, lambda: None, self.module, self.name)


class Decode:
    """f(cvivit.decode*(...)).backward() through phk_cvivit_decode_backward."""

    def __init__(self, name, entry, device):
        self.name, self.entry, self.device = name, entry, device
        self.module = DG.build_module(name).to(device)

    def grads(self, precision=L.PREC_F32):
        return DG.product_grads(self.name, self.entry, self.module, self.device, precision)

    def check_bars(self, name):
        return DG.check_fp32(self.device, lambda: None, self.module, self.name, self.entry)


class Encode:
    """f(cvivit.encode(tokens)).backward() through phk_cvivit_encode_backward."""

    def __init__(self, name, device):
        self.name, self.device = name, device
        self.module = DG.build_module(name).to(device)

    def grads(self, precision=L.PREC_F32):
        return EG.product_grads(self.name, self.module, self.device, precision)

    def check_bars(self, name):
        return EG.check_fp32(self.device, lambda: None, self.module, self.name)


class Recon:
    """cvivit(video).backward() through phk_cvivit_backward, with video.requires_grad."""

    def __init__(self, name, device):
        self.name, self.device = name, device
        self.module = RL.build_module(name).to(device)

    def grads(self, precision=L.PREC_F32):
        loss, grads, _ = RL.product_run(self.name, self.module, self.device, precision)
        return dict(grads, loss=torch.tensor(loss))

    def check_bars(self, name):
        return RL.check_fp32(self.device, lambda: None, self.module, self.name)


def assert_bitwise_equal(label, runs):
    """Every gradient of every run equal, bit for bit, to the first run's; the same tensors are None."""
    first = runs[0]
    assert any(g is not None and g.numel() and bool(g.any()) for g in first.values()), f"{label}: no gradient at all"
    for i, other in enumerate(runs[1:], 1):
        assert first.keys() == other.keys(), label
        for k, g in first.items():
            assert (g is None) == (other[k] is None), f"{label} {k}: None in one run only"
            if g is not None:
                assert torch.equal(g, other[k]), (
                    f"{label} {k}: run {i} differs from run 0 by {float((g - other[k]).abs().max()):.3e}")


def differing(runs):
    """Names of the gradients that are not bit-identical between the first two runs."""
    a, b = runs[0], runs[1]
    return [k for k, g in a.items() if g is not None and not torch.equal(g, b[k])]


def workspace_queries(device):
    """{query name: a callable returning its byte count} for the five backward entry points on small case tables."""
    lib = L.lib()
    fg = T.build_module(FG.ALL_CASES["emu_critic"]["base"]).to(device)
    dec = DG.build_module("rect").to(device)
    import ctypes
    mt = fg._table()
    dt, et = dec._dec_table(), dec._table()
    keep = (fg, dec)  # the tables point into the modules' buffers
    return {"_modules": keep,
        "phk_maskgit_train_workspace_bytes": lambda: lib.phk_maskgit_train_workspace_bytes(ctypes.byref(mt), 2, 24, 5, 1, L.PREC_F32),
        "phk_maskgit_backward_workspace_bytes": lambda: lib.phk_maskgit_backward_workspace_bytes(
            ctypes.byref(mt), 2, 24, 5, 1, L.HEAD_SCORE, L.PREC_F32),
        "phk_cvivit_decode_backward_workspace_bytes": lambda: lib.phk_cvivit_decode_backward_workspace_bytes(
            ctypes.byref(dt), 2, 3, L.PREC_F32),
        "phk_cvivit_encode_backward_workspace_bytes": lambda: lib.phk_cvivit_encode_backward_workspace_bytes(
            ctypes.byref(et), 2, 3, L.PREC_F32),
        "phk_cvivit_backward_workspace_bytes": lambda: lib.phk_cvivit_backward_workspace_bytes(
            ctypes.byref(et), ctypes.byref(dt), 2, 7, L.PREC_F32),
    }
