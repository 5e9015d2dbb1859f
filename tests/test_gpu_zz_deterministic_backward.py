"""GPU: torch.use_deterministic_algorithms(True) makes every hand-written backward bit-reproducible at production shapes.

- Each of the five backward entry points runs three times in fp32 and in bf16 mode under the switch: every gradient is
  bit-identical across the runs (the bf16 tensor-core products included), and the fp32 runs stay within the float64
  bars of the existing gradient tests.
- With the switch off, the library issues the same kernels and asks for the same workspace as in a process that never
  touched the switch.
- With the switch on, every progress event of the reconstruction-loss backward still marks its group final.
- The public flows raise nothing under the switch with warn_only=False, and sampling returns the ids it returns without it.
"""
import ctypes as C
import json
import os
import subprocess
import sys

import pytest
import torch

from phenaki_pytorch_b200 import _lib as L
from tests import cases as CS
from tests import deterministic_cases as DC
from tests import text_grad_cases as TG

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ENTRIES = {
    # configs[3]: MaskGit dim 512, depth 6, V 65536, 4 x 576 tokens, 16 text tokens, a cross-attention TokenCritic, dropout
    "train_step": lambda: DC.TrainStep(TG.AT_SIZE_CASE, 0.1, DEV),
    # the production TokenCritic forward with cross-attention (null key / values) and its backward
    "maskgit_backward": lambda: DC.ForwardBackward("prod_critic", DEV),
    # configs[1]: dim 512, 8 x 64 heads, depth 4 + 4, 256^2 images, B = 2
    "decode_backward": lambda: DC.Decode("at_size", "ids", DEV),
    "encode_backward": lambda: DC.Encode("at_size", DEV),
    "recon_backward": lambda: DC.Recon("at_size", DEV),
}


@pytest.fixture(scope="module")
def runs():
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = ENTRIES[name]()
        return cache[name]

    yield get
    cache.clear()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("precision", [L.PREC_F32, L.PREC_BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("name", list(ENTRIES))
def test_three_runs_are_bit_identical(runs, name, precision):
    run = runs(name)
    with DC.deterministic():
        DC.assert_bitwise_equal(f"{name} ({precision})", [run.grads(precision) for _ in range(3)])
    torch.cuda.synchronize()


@pytest.mark.parametrize("name", list(ENTRIES))
def test_deterministic_gradients_stay_within_the_float64_bars(runs, name):
    with DC.deterministic():
        runs(name).check_bars(name)
    torch.cuda.synchronize()


_PROBE = r"""
import json, sys
sys.path.insert(0, {root!r})
import torch
from torch.profiler import ProfilerActivity, profile
from phenaki_pytorch_b200 import _lib as L
from tests import deterministic_cases as DC
if {touch}:
    L.lib().phk_train_set_deterministic(1)
    L.lib().phk_train_set_deterministic(0)
qs = DC.workspace_queries("cuda:0")
out = dict(queries={{k: q() for k, q in qs.items() if not k.startswith("_")}}, kernels={{}})
for name, run in [("decode", DC.Decode("rect", "ids", "cuda:0")), ("recon", DC.Recon("rect_mask", "cuda:0")),
                  ("train", DC.TrainStep(DC.TG.SMALL["token_critic"], 0.2, "cuda:0"))]:
    run.grads()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run.grads()
        torch.cuda.synchronize()
    ops = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    out["kernels"][name] = [e.name for e in sorted(ops, key=lambda e: e.time_range.start)]
print("RESULT" + json.dumps(out))
"""


def _probe(touch):
    code = _PROBE.format(root=ROOT, touch=touch)
    res = subprocess.run([sys.executable, "-c", code], check=True, capture_output=True, text=True, cwd=ROOT)
    return json.loads([ln for ln in res.stdout.splitlines() if ln.startswith("RESULT")][-1][len("RESULT"):])


def test_switch_off_is_the_library_that_never_saw_the_switch():
    never, toggled = _probe(False), _probe(True)
    assert never["queries"] == toggled["queries"]
    for name, ops in never["kernels"].items():
        assert len(ops) > 10, name
        assert ops == toggled["kernels"][name], f"{name}: the kernel sequence changed after the switch was toggled"


def test_progress_events_mark_their_groups_final_under_the_switch(monkeypatch):
    from tests import recon_loss_cases as RL
    from tests import test_gpu_zz_recon_loss_sync as SYNC
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = RL.build_module(name).to(DEV)
        return cache[name]

    with DC.deterministic():
        for precision in (L.PREC_F32, L.PREC_BF16):
            SYNC.test_each_progress_event_marks_its_group_final(get, monkeypatch, precision, True)


def test_public_flows_raise_nothing_under_the_switch():
    from phenaki_pytorch_b200 import phenaki as P
    with DC.deterministic(True, warn_only=False):
        run = DC.TrainStep(TG.SMALL["token_critic"], 0.2, DEV)  # Phenaki.forward(...).backward(), e.requires_grad
        g = run.grads()
        assert g["text_embeds"] is not None
        DC.ForwardBackward("emu_critic", DEV).grads()          # critic(ids, text_embeds) then backward()
        DC.Recon("rect", DEV).grads()                          # cvivit(video).backward()
    case = CS.SAMPLE_CASES["confidence"]
    torch.manual_seed(case["seed"])
    ph = P.Phenaki(cvivit=P.CViViT(**CS.SAMPLE_CVIVIT).to(DEV), maskgit=P.MaskGit(**CS.SAMPLE_MASKGIT).to(DEV),
                   steps=case["steps"], text_embed_dim=CS.SAMPLE_MASKGIT["dim_context"])
    ctx = CS.synthetic_text_embeds(2, 6, CS.SAMPLE_MASKGIT["dim_context"], (6, 3), 7).to(DEV)
    ids = []
    for on in (False, True):
        with DC.deterministic(on):
            torch.manual_seed(5)
            ids.append(ph.sample(num_frames=7, text_embeds=ctx, return_token_ids=True).cpu())
    assert torch.equal(ids[0], ids[1])
