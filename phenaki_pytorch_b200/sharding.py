"""Batch sharding for the N-GPU path (SURVEY 8e): every unit of work on the hot path is one video (encode) or one
sample (demasking loop), so ranks take contiguous batch shards, weights are replicated and the data path has no
collective.  The only exchanges are off the timed path: an optional gather of the ids to rank 0 and the max-over-ranks
reduction of the measured time.  Works over any ``torch.distributed`` backend (nccl on the GPU box, gloo in the CPU
tests).

Training (SURVEY 8e / 8f-2) adds the one collective the reference implies (DDP's gradient all-reduce in
PhenakiTrainer): the training step writes every gradient of a network into ONE flat fp32 bucket
(modules.GradKeep.flat), so the exchange is a single all-reduce over that buffer -- no bucket packing copy.
"""
import ctypes

import torch
import torch.distributed as dist


def world():
    """(rank, world_size) of the default process group, (0, 1) when there is none."""
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def shard_range(n, rank, world_size):
    """Contiguous shard [lo, hi) of `n` units for `rank`; the first n % world_size ranks take one extra unit, a rank
    past the end gets an empty shard (n < world_size)."""
    assert n >= 0 and world_size >= 1 and 0 <= rank < world_size
    base, extra = divmod(n, world_size)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def shard_batch(t, rank=None, world_size=None, dim=0):
    """This rank's contiguous slice of a batch tensor."""
    r, w = world()
    rank = r if rank is None else rank
    world_size = w if world_size is None else world_size
    lo, hi = shard_range(t.shape[dim], rank, world_size)
    return t.narrow(dim, lo, hi - lo)


def gather_batch(local, total, dim=0):
    """Inverse of shard_batch: every rank gets the full batch (ragged shards are padded to the largest one for the
    collective and trimmed afterwards).  Not on the timed path."""
    rank, w = world()
    if w == 1:
        return local
    sizes = [shard_range(total, r, w) for r in range(w)]
    most = max(hi - lo for lo, hi in sizes)
    pad = most - local.shape[dim]
    if pad:
        shape = list(local.shape)
        shape[dim] = pad
        local = torch.cat([local, local.new_zeros(shape)], dim=dim)
    parts = [torch.empty_like(local) for _ in range(w)]
    dist.all_gather(parts, local.contiguous())
    return torch.cat([p.narrow(dim, 0, hi - lo) for p, (lo, hi) in zip(parts, sizes)], dim=dim)


def max_over_ranks(value, device=None):
    """A timing is the MAX over ranks (the job is as slow as its slowest shard)."""
    _, w = world()
    if w == 1:
        return float(value)
    t = torch.tensor([float(value)], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def rank_seed(seed, rank=None):
    """Per-rank noise seed for sharded sampling: rank r draws the stream `seed + r` (documented deviation from a
    single-process run, whose one global generator would interleave all samples)."""
    r, _ = world()
    return int(seed) + (r if rank is None else rank)


def all_reduce_mean_(flat, group=None):
    """In-place mean over ranks of a flat gradient bucket (what DistributedDataParallel does to every bucket); a
    no-op without a process group.  NCCL over NVLink on the GPU box, gloo in the CPU tests."""
    _, w = world()
    if w == 1:
        return flat
    dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
    flat.div_(w)
    return flat


# Test-only: take the overlapped path below in a one-rank NCCL group too, so that a single GPU exercises it (the mean
# over one rank leaves every gradient bit for bit as it was).
OVERLAP_AT_WORLD_SIZE_1 = False


def bucket_spans(flat, views, groups):
    """Slices of a flat gradient bucket (modules.GradKeep: ``views`` maps a parameter to its view of ``flat``) for
    groups of parameters: per group, the [lo, hi) element spans its parameters' padded views cover, adjacent spans merged.
    A group's parameters need not be adjacent in the bucket; zero-element parameters have no address and are skipped.
    None when spans of different groups overlap (then the bucket cannot be sliced by group)."""
    base, esz = flat.data_ptr(), flat.element_size()
    out = []
    for params in groups:
        spans = []
        for p in params:
            if p.numel():
                lo = (views[p].data_ptr() - base) // esz
                spans.append((lo, lo + (p.numel() + 63) // 64 * 64))
        merged = []
        for lo, hi in sorted(spans):
            if merged and lo <= merged[-1][1]:
                merged[-1][1] = max(merged[-1][1], hi)
            else:
                merged.append([lo, hi])
        out.append(merged)
    flat_spans = sorted(sp for spans in out for sp in spans)
    if any(a[1] > b[0] for a, b in zip(flat_spans, flat_spans[1:])):
        return None
    return out


def overlap_plan(owner, flat, n_events, dev):
    """Data parallel over NCCL (world size > 1, or OVERLAP_AT_WORLD_SIZE_1): dict(events, handles, stream) -- one CUDA
    event per gradient group for phk_train_set_progress_events and the side stream the slices are reduced on, created
    once per (device, n_events) and kept on ``owner``.  None when there is nothing to overlap (single process, non-NCCL
    backend, CPU bucket)."""
    if not (dist.is_available() and dist.is_initialized() and flat.is_cuda and dist.get_backend() == "nccl"
            and (dist.get_world_size() > 1 or OVERLAP_AT_WORLD_SIZE_1)):
        return None
    cache = owner.__dict__.setdefault("_overlap_cache", {})
    key = (dev, n_events)
    if key not in cache:
        events = [torch.cuda.Event() for _ in range(n_events)]
        for e in events:
            e.record()  # creates the CUDA event behind the (lazily initialised) torch object
        handles = (ctypes.c_void_p * n_events)(*[e.cuda_event for e in events])
        cache[key] = dict(events=events, handles=handles, stream=torch.cuda.Stream(device=dev))
    return cache[key]


def launch_overlapped_all_reduce(flat, plan, groups):
    """One all-reduce (mean) per slice of ``flat`` on the plan's side stream, each group's slices waiting only for that
    group's event (``groups``: bucket_spans, in event order): the collective of the groups the backward finished first
    runs while it is still computing the rest.  Returns the event recorded on the side stream after the last slice."""
    side, w = plan["stream"], dist.get_world_size()
    flat.record_stream(side)
    for ev, spans in zip(plan["events"], groups):
        if not spans:
            continue
        side.wait_event(ev)
        with torch.cuda.stream(side):
            for lo, hi in spans:
                part = flat[lo:hi]
                dist.all_reduce(part, op=dist.ReduceOp.SUM)
                part.div_(w)
    done = torch.cuda.Event()
    done.record(side)
    return done
