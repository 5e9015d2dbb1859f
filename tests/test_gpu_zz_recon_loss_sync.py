"""GPU: the data-parallel hooks of the C-ViViT reconstruction-loss backward (``CViViT.sync_gradients``).

- The gradient groups partition the flat gradient bucket, one contiguous span each, as many as
  phk_cvivit_backward_progress_groups reports.
- Every progress event phk_cvivit_backward records marks its group final: a side stream that waits on the event and
  copies the group's slice at once copies the final gradient, bit for bit, in fp32 and bf16 mode, training and eval mode,
  at the configs[1] shape (B = 2, F = 17).
- Without registered events loss.backward() runs the kernel sequence tests/golden/cvivit_backward_kernels.json pins
  (taken before the events existed), in fp32 and bf16 mode, training and eval mode; with events registered it runs the
  same sequence.
- The overlapped NCCL all-reduce, forced in a one-rank NCCL group, runs and leaves every gradient as computed.

The file sorts after every other GPU file for the reason tests/test_gpu_zz_encode_backward.py gives; its profiler traces
and its NCCL group run in processes of their own."""
import ctypes as C
import json
import os
import subprocess
import sys

import pytest
import torch

from phenaki_pytorch_b200 import _lib as L
from phenaki_pytorch_b200 import sharding
from phenaki_pytorch_b200.modules import GradKeep
from tests import recon_loss_cases as RL

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNELS_GOLDEN = os.path.join(ROOT, "tests", "golden", "cvivit_backward_kernels.json")


@pytest.fixture(scope="module")
def modules():
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = RL.build_module(name).to(DEV)
        return cache[name]

    yield get
    cache.clear()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name", ["rect", "at_size"])
def test_gradient_groups_partition_the_bucket(modules, name):
    cv = modules(name)
    groups = cv._recon_gradient_groups()
    params = [p for g in groups for p in g]
    assert len(params) == len(set(params)) and set(params) == set(cv.parameters())
    n = L.lib().phk_cvivit_backward_progress_groups(C.byref(cv._table()), C.byref(cv._dec_table()))
    assert n == len(groups) == 2 * (cv.enc_spatial_transformer.depth + cv.enc_temporal_transformer.depth) + 5
    gk = GradKeep(params)
    spans = sharding.bucket_spans(gk.flat, gk.views, groups)
    assert spans is not None and all(len(s) == 1 for s in spans)  # one contiguous span per group
    covered = torch.zeros(gk.flat.numel(), dtype=torch.int32)
    for (lo, hi), in spans:
        covered[lo:hi] += 1
    assert int(covered.min()) == 1 and int(covered.max()) == 1
    assert [s[0][0] for s in spans] == sorted(s[0][0] for s in spans)  # laid out in completion order


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("precision", [L.PREC_F32, L.PREC_BF16], ids=["f32", "bf16"])
def test_each_progress_event_marks_its_group_final(modules, monkeypatch, precision, training):
    """A side stream waits on every event and copies that group's slice of the bucket: each copy must equal the gradient
    the backward leaves, bit for bit (a group written after its event would be caught mid-way)."""
    cv = modules("at_size")
    cv.precision = precision
    cv.train(training)
    taken = {}

    def plan(owner, flat, n_events, dev):
        events = [torch.cuda.Event() for _ in range(n_events)]
        for e in events:
            e.record()
        return dict(events=events, handles=(C.c_void_p * n_events)(*[e.cuda_event for e in events]),
                    stream=torch.cuda.Stream(device=dev))

    def launch(flat, p, groups):
        side = p["stream"]
        flat.record_stream(side)
        copies = []
        for ev, spans in zip(p["events"], groups):
            side.wait_event(ev)
            with torch.cuda.stream(side):
                copies.append([(lo, hi, flat[lo:hi].clone()) for lo, hi in spans])
        taken.update(flat=flat, copies=copies, n=len(p["events"]))
        done = torch.cuda.Event()
        done.record(side)
        return done

    monkeypatch.setattr(sharding, "overlap_plan", plan)
    monkeypatch.setattr(sharding, "launch_overlapped_all_reduce", launch)
    cv.sync_gradients = True
    try:
        video, _ = RL.inputs("at_size")
        cv.zero_grad(set_to_none=True)
        cv(video.to(DEV)).backward()
        torch.cuda.synchronize()
    finally:
        cv.sync_gradients = False
        cv.zero_grad(set_to_none=True)
    assert taken and taken["n"] == len(taken["copies"]) == len(cv._recon_gradient_groups())
    flat = taken["flat"]
    assert float(flat.abs().max()) > 0
    for k, spans in enumerate(taken["copies"]):
        for lo, hi, copy in spans:
            assert torch.equal(copy, flat[lo:hi]), f"group {k}: slice [{lo}, {hi}) changed after its event"


@pytest.fixture(scope="module")
def backward_kernels():
    code = (f"import json, sys; sys.path.insert(0, {ROOT!r}); from tests import test_gpu_zz_recon_loss_sync as T; "
            f"print(json.dumps(T.backward_kernel_sequences()))")
    flags = ["-s"] if sys.flags.no_user_site else []
    run = subprocess.run([sys.executable, *flags, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert run.returncode == 0, run.stderr[-4000:]
    return json.loads(run.stdout.strip().splitlines()[-1])


def backward_kernel_sequences():
    """{"case": [device ops of loss.backward() without events, with events registered]} at the configs[1] shape, fp32 and
    bf16 mode, training and eval mode: the kernel names of one backward each in a torch.profiler trace, after a warm-up."""
    from torch.profiler import ProfilerActivity, profile
    cv = RL.build_module("at_size").to(DEV)
    video = RL.inputs("at_size")[0].to(DEV)
    n = L.lib().phk_cvivit_backward_progress_groups(C.byref(cv._table()), C.byref(cv._dec_table()))
    events = [torch.cuda.Event() for _ in range(n)]
    for e in events:
        e.record()
    handles = (C.c_void_p * n)(*[e.cuda_event for e in events])

    def device_ops(register):
        loss = cv(video)
        torch.cuda.synchronize()
        if register:
            L.check(L.lib().phk_train_set_progress_events(handles, n), "phk_train_set_progress_events")
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            loss.backward()
            torch.cuda.synchronize()
        cv.zero_grad(set_to_none=True)
        ops = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        return [e.name for e in sorted(ops, key=lambda e: e.time_range.start)]

    out = {}
    for prec_name, prec in (("f32", L.PREC_F32), ("bf16", L.PREC_BF16)):
        for mode in ("train", "eval"):
            cv.precision = prec
            cv.train(mode == "train")
            device_ops(False)
            out[f"{prec_name}/{mode}"] = [device_ops(False), device_ops(True)]
    return out


@pytest.mark.parametrize("case", ["f32/train", "f32/eval", "bf16/train", "bf16/eval"])
def test_backward_kernel_sequence_is_unchanged(backward_kernels, case):
    plain, with_events = backward_kernels[case]
    with open(KERNELS_GOLDEN) as f:
        golden = json.load(f)
    want = [golden["names"][i] for i in golden[case]]
    # the profiler now and then loses the first record of a trace (here the bucket's zero fill): the same sequence
    # without it is accepted, nothing else
    for ops, what in ((plain, "without events"), (with_events, "with events registered")):
        assert ops == want or ops == want[1:], \
            f"{case} {what}: {len(ops)} device ops differ from the {len(want)} pinned before progress events existed"


def overlapped_at_world_size_1():
    """In a one-rank NCCL group with sharding.OVERLAP_AT_WORLD_SIZE_1: (whether the overlapped all-reduce ran, whether
    it left the bucket bit for bit as the backward computed it, the largest |sync - no sync| gradient difference over the
    largest gradient) per precision mode."""
    import torch.distributed as dist
    port = 29000 + os.getpid() % 2000
    dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1,
                            device_id=torch.device(DEV))
    sharding.OVERLAP_AT_WORLD_SIZE_1 = True
    real = sharding.launch_overlapped_all_reduce
    seen = {}

    def launch(flat, plan, groups):
        torch.cuda.synchronize()
        seen["before"] = flat.clone()
        done = real(flat, plan, groups)
        seen["flat"] = flat
        return done

    sharding.launch_overlapped_all_reduce = launch
    cv = RL.build_module("at_size").to(DEV)
    video = RL.inputs("at_size")[0].to(DEV)
    out = {}
    try:
        for prec_name, prec in (("f32", L.PREC_F32), ("bf16", L.PREC_BF16)):
            cv.precision = prec
            grads = {}
            for sync in (False, True):
                seen.clear()
                cv.sync_gradients = sync
                cv.zero_grad(set_to_none=True)
                cv(video).backward()
                torch.cuda.synchronize()
                grads[sync] = {k: p.grad.clone() for k, p in cv.named_parameters() if p.grad is not None}
                if sync:
                    ran = "before" in seen
                    unchanged = ran and torch.equal(seen["before"], seen["flat"])
            top = max(float(g.abs().max()) for g in grads[False].values() if g.numel())
            diff = max(float((grads[True][k] - g).abs().max()) for k, g in grads[False].items() if g.numel())
            out[prec_name] = dict(ran=ran, unchanged=unchanged, same_keys=grads[True].keys() == grads[False].keys(),
                                  rel_diff=diff / top)
    finally:
        dist.destroy_process_group()
    return out


def test_overlapped_all_reduce_in_a_one_rank_nccl_group_leaves_the_gradients():
    code = (f"import json, sys; sys.path.insert(0, {ROOT!r}); from tests import test_gpu_zz_recon_loss_sync as T; "
            f"print(json.dumps(T.overlapped_at_world_size_1()))")
    flags = ["-s"] if sys.flags.no_user_site else []
    run = subprocess.run([sys.executable, *flags, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert run.returncode == 0, run.stderr[-4000:]
    res = json.loads(run.stdout.strip().splitlines()[-1])
    for prec, r in res.items():
        assert r["ran"], f"{prec}: the overlapped all-reduce did not run"
        assert r["unchanged"], f"{prec}: the one-rank all-reduce changed the bucket"
        assert r["same_keys"], prec
        # two backwards differ only by the order of their atomic adds (tests/recon_loss_cases.py check_deterministic)
        assert r["rel_diff"] <= 1e-6, f"{prec}: sync vs no sync differ by {r['rel_diff']:.3e} of the largest gradient"
