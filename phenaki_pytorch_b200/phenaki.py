"""MaskGit / TokenCritic / SelfCritic / Phenaki / make_video -- drop-ins for the reference classes of
/root/reference/phenaki_pytorch/phenaki_pytorch.py on the sampling hot path.

Constructor keywords, attribute names, state-dict layout and the ``forward`` / ``forward_with_cond_scale``
/ ``sample`` signatures follow the reference (phenaki_pytorch.py:105-147, 217-249, 307-336, 341-430,
691-714).  All arithmetic runs in libphk.so; torch is used for device memory, streams and the (tiny)
boolean plumbing around the calls.  ``Phenaki.forward`` (the training loss, :562-687) needs backward
kernels and is a next-tier row (SURVEY.md 8f-2).
"""
import ctypes as C
import math
from functools import partial
from typing import List, Optional, Union

import numpy as np
import torch
from torch import nn

from . import _lib as L
from . import sharding
from .cvivit import CViViT

from .modules import (ContinuousPositionBias, GradKeep, Keep, Transformer, Workspace, _NoParams, cpb_grad_table,
                      cpb_table, transformer_grad_table, transformer_table, weights_signature)


def _noise_seed(dev):
    """Key of the in-kernel Philox noise: the seed of torch's CUDA generator of that device (``torch.manual_seed``
    sets it), so seeded runs repeat."""
    return torch.cuda.default_generators[dev.index if dev.index is not None else torch.cuda.current_device()].initial_seed()


def _rng_take(dev, seed, count):
    """Reserves `count` consecutive Philox counters of the in-kernel noise on `dev` and returns the first one.
    The running counter IS the offset of torch's CUDA generator of that device: process-wide, per device, restarted by
    ``torch.manual_seed`` -- so calls of any shape (scene chains with primed, shorter scenes; several Phenaki objects;
    interleaved training steps) draw from disjoint counter ranges and seeded runs repeat."""
    gen = torch.cuda.default_generators[dev.index if dev.index is not None else torch.cuda.current_device()]
    first = int(gen.get_offset())
    gen.set_offset(first + (int(count) + 3) // 4 * 4)  # torch requires multiples of 4
    return first & (2 ** 64 - 1)


def _noise_stride(rows, vocab):
    """Philox counters one V-wide gumbel draw over `rows` tokens consumes (4 uniforms per counter), rounded up to a
    multiple of 4 (the granularity of torch's generator offset); phk_maskgit_demask_iteration advances the device-side
    counter by the same amount (csrc/api.cu: noise_stride)."""
    return (rows * ((vocab + 3) // 4) + 1 + 3) // 4 * 4


def _prod(xs):
    r = 1
    for x in xs:
        r *= int(x)
    return r


class _TokenTransformer(nn.Module):
    """Shared libphk plumbing of MaskGit and TokenCritic (both: embeddings -> Transformer -> head)."""

    is_critic = False

    def _init_runtime(self):
        self.precision = L.default_precision()
        self._tables, self._sig = None, None
        self._ws = Workspace()
        self._bias_cache = {}

    def __deepcopy__(self, memo):
        """copy.deepcopy (EMA wrappers, `copy_for_eval`-style users of the reference): parameters and buffers are
        copied by torch; the ctypes weight tables, workspace and cached position-bias tables are per-object runtime
        state and are rebuilt lazily by the copy."""
        import copy
        cls = self.__class__
        new = cls.__new__(cls)
        memo[id(self)] = new
        runtime = ("_tables", "_sig", "_ws", "_bias_cache", "_phk_sig_cache")
        for k, v in self.__dict__.items():
            if k not in runtime:
                new.__dict__[k] = copy.deepcopy(v, memo)
        precision = self.precision
        new._init_runtime()
        new.precision = precision
        return new

    def _table(self):
        sig = (weights_signature(self), self.precision)
        if self._tables is None or sig != self._sig:
            keep = Keep()
            h16 = self.precision == L.PREC_BF16
            t = L.MaskgitT()
            tf = self.transformer
            t.dim, t.heads, t.dim_head = tf.dim, tf.heads, tf.dim_head
            t.num_tokens = self.token_emb.weight.shape[0] - 1
            t.max_seq_len = self.pos_emb.weight.shape[0]
            t.is_critic = int(self.is_critic)
            t.has_bias = int(not self.is_critic)
            t.shrink_alpha = float(getattr(self, "gradient_shrink_alpha", 0.0))
            t.token_emb, t.pos_emb = keep.t(self.token_emb.weight), keep.t(self.pos_emb.weight)
            if not self.is_critic:
                t.pos_bias = cpb_table(self.continuous_pos_bias, keep)
                t.head_w, t.head_b = keep.t(self.to_logits.weight), keep.t(self.to_logits.bias)
                if self.precision:
                    t.head_w_h = keep.w16(self.to_logits.weight, self.precision)
            else:
                t.head_w, t.head_b = keep.t(self.to_logits[0].weight), keep.t(self.to_logits[0].bias)
            t.transformer = transformer_table(tf, keep, self.precision)
            self._tables, self._sig = (t, keep), sig
            self._bias_cache = {}
        return self._tables[0]

    def _pos_bias(self, table, patch_shape, device):
        """3-D continuous position bias (phenaki_pytorch.py:186): weight-only, cached per shape."""
        if self.is_critic:
            return None
        key = (tuple(patch_shape), device)
        if key not in self._bias_cache:
            lib = L.lib()
            n = _prod(patch_shape)
            out = torch.empty((self.transformer.heads, n, n), dtype=torch.float32, device=device)
            scratch = torch.empty(int(lib.phk_cpb_scratch_floats(C.byref(table.pos_bias), *patch_shape)),
                                  dtype=torch.float32, device=device)
            L.check(lib.phk_cpb_bias(C.byref(table.pos_bias), *patch_shape, L.ptr(scratch), L.ptr(out),
                                     L.stream_ptr()), "phk_cpb_bias")
            self._bias_cache[key] = out
        return self._bias_cache[key]

    def context_kv(self, context):
        """Per-layer context_norm + to_kv of the text embedding (attention.py:137-144): (depth, b*L, 2I)."""
        lib = L.lib()
        context = L.require_cuda(context, "context", torch.float32)
        b, l, dc = context.shape
        tf = self.transformer
        assert tf.layers[0][2] is not None, "model has no cross attention"
        assert dc == tf.layers[0][2].dim_context, "text embedding dimension is not correct"
        table = self._table()
        inner2 = 2 * tf.heads * tf.dim_head
        out = torch.empty((tf.depth, b * l, inner2), dtype=torch.float32, device=context.device)
        scratch = torch.empty((b * l, 3 * dc), dtype=torch.float32, device=context.device)  # (+ the split-bf16 operands)
        L.check(lib.phk_maskgit_context_kv(C.byref(table), L.ptr(context), b, l, L.ptr(out), L.ptr(scratch),
                                           self.precision, L.stream_ptr()), "phk_maskgit_context_kv")
        return out

    def _run(self, ids, patch_shape, *, ctx_kv=None, ctx_len=0, text_mask=None, video_mask=None, cfg_pair=False,
             return_embeds=False):
        """ids (b, n) int64 -> logits ((1+cfg) * b, n, V) | embeds (.., dim)."""
        lib = L.lib()
        ids = L.require_cuda(ids, "token ids", torch.int64)
        b, n = ids.shape
        assert _prod(patch_shape) == n, "video patch shape must cover the token sequence"
        dev = ids.device
        with torch.cuda.device(dev):
            table = self._table()
            assert n <= table.max_seq_len, \
                f"the video token sequence length you are passing in ({n}) is greater than the `max_seq_len` ({table.max_seq_len})"
            reps = 2 if cfg_pair else 1
            embeds_only = return_embeds or self.is_critic
            width = table.dim if embeds_only else table.num_tokens
            out = torch.empty((reps * b, n, width), dtype=torch.float32, device=dev)
            nbytes = lib.phk_maskgit_workspace_bytes(C.byref(table), b, n, ctx_len, int(cfg_pair), self.precision)
            ws = self._ws.get(nbytes, dev)
            bias = self._pos_bias(table, patch_shape, dev)
            if text_mask is not None:
                text_mask = L.require_cuda(text_mask.to(torch.uint8), "text mask")
            if video_mask is not None:
                video_mask = L.require_cuda(video_mask.to(torch.uint8), "video mask")
            pt, ph, pw = (int(v) for v in patch_shape)
            L.check(lib.phk_maskgit_forward(C.byref(table), L.ptr(ids), b, n, pt, ph, pw, L.ptr(ctx_kv), ctx_len,
                                            L.ptr(text_mask), L.ptr(video_mask), int(cfg_pair), int(embeds_only),
                                            L.ptr(bias), L.ptr(out), L.ptr(ws), ws.numel(), self.precision,
                                            L.stream_ptr()), "phk_maskgit_forward")
        return out

    def _sample_step(self, ids_in, patch_shape, *, ctx_kv, ctx_len, text_mask, cond_scale, temperature, seed,
                     offset, mask, ids, pred, scores, masked_per_seq=0, prime_len=0):
        """Fused demasking iteration (bf16 mode): CFG-pair forward + logits head + gumbel argmax + confidence in
        libphk (phk_maskgit_sample_step); the (2b, n, V) logits are never materialised.  ``masked_per_seq``: how many
        tokens of EVERY sequence are masked, when known (the demasking schedule knows it): the final LayerNorm, the
        guidance and the logits head then run on those rows only."""
        lib = L.lib()
        b, n = ids_in.shape
        dev = ids_in.device
        with torch.cuda.device(dev):
            table = self._table()
            nbytes = lib.phk_maskgit_sample_workspace_bytes(C.byref(table), b, n, ctx_len)
            ws = self._ws.get(nbytes, dev)
            bias = self._pos_bias(table, patch_shape, dev)
            if text_mask is not None:
                text_mask = L.require_cuda(text_mask.to(torch.uint8), "text mask")
            pt, ph, pw = (int(v) for v in patch_shape)
            # ids_in = prime ids + the tokens being sampled; mask / ids / pred / scores cover the latter
            L.check(lib.phk_maskgit_sample_step(C.byref(table), L.ptr(ids_in), b, n, pt, ph, pw, L.ptr(ctx_kv), ctx_len,
                                                L.ptr(text_mask), L.ptr(bias), float(cond_scale), float(temperature), seed,
                                                offset, L.ptr(mask), L.ptr(ids), L.ptr(pred), L.ptr(scores),
                                                int(masked_per_seq), int(prime_len), L.ptr(ws), ws.numel(),
                                                L.stream_ptr()),
                    "phk_maskgit_sample_step")

    def _grad_table(self, with_cross, owner=None, head=None):
        """Zero-filled gradient buffers (one flat fp32 bucket in ``owner.parameters()`` order) and the
        phk_maskgit_t-shaped table that addresses them; same member-by-member layout as ``_table``.
        ``head``: an nn.Linear(dim, 1) that replaces the network's own head (SelfCritic.to_pred)."""
        # one bucket + table per (owner, head, cross) is kept and re-zeroed while no backward() is pending on it (building the
        # 150-entry table and a 380 MB allocation per step cost more host time than the step's launches)
        cache = self.__dict__.setdefault("_grad_cache", {})
        key = (id(owner), id(head), bool(with_cross), weights_signature(owner if owner is not None else self)[:1],
               next(self.parameters()).device)
        hit = cache.get(key)
        if hit is not None and not hit[1].busy and hit[2] == [id(p) for p in (owner if owner is not None else self).parameters()]:
            hit[1].flat.zero_()
            hit[1].reduced = None
            hit[1].busy = True
            return hit[0], hit[1]
        gk = GradKeep((owner if owner is not None else self).parameters())
        gk.busy, gk.reduced = True, None
        t = L.MaskgitT()
        tf = self.transformer
        t.dim, t.heads, t.dim_head = tf.dim, tf.heads, tf.dim_head
        t.num_tokens = self.token_emb.weight.shape[0] - 1
        t.max_seq_len = self.pos_emb.weight.shape[0]
        t.is_critic, t.has_bias = int(self.is_critic), int(not self.is_critic)
        t.token_emb, t.pos_emb = gk.g(self.token_emb.weight), gk.g(self.pos_emb.weight)
        if not self.is_critic:
            t.pos_bias = cpb_grad_table(self.continuous_pos_bias, gk)
        if head is not None:
            t.head_w, t.head_b = gk.g(head.weight), gk.g(head.bias)
        elif not self.is_critic:
            t.head_w, t.head_b = gk.g(self.to_logits.weight), gk.g(self.to_logits.bias)
        else:
            t.head_w, t.head_b = gk.g(self.to_logits[0].weight), gk.g(self.to_logits[0].bias)
        t.transformer = transformer_grad_table(tf, gk, with_cross)
        if hit is None or not hit[1].busy:
            cache[key] = (t, gk, [id(p) for p in (owner if owner is not None else self).parameters()])
        return t, gk

    def train_step(self, ids_in, patch_shape, *, targets=None, token_mask=None, labels=None, context=None,
                   text_mask=None, video_mask=None, loss_scale=1.0, keep_logits=False, head=None, owner=None,
                   overlap_all_reduce=False):
        """One forward + loss + backward in libphk (phk_maskgit_train_step; ``self.precision`` selects fp32 FFMA or
        wgmma bf16 products, everything else is fp32 in both modes): returns (loss 0-d tensor,
        GradKeep with d(loss_scale * loss)/d(parameter), logits or None).  ``labels`` given: Linear(dim, 1) head + BCE
        with logits (TokenCritic; or ``head`` = SelfCritic.to_pred on this MaskGit, gradients laid out for
        ``owner.parameters()``); otherwise masked cross entropy against ``targets`` at ``token_mask``.
        In training mode (``self.training``) the transformer's ``attn_dropout`` / ``ff_dropout`` apply as the
        reference's nn.Dropout does; the masks come from fresh counters of the device's noise generator (include/phk.h,
        phk_dropout_t), so every call draws new masks and ``torch.manual_seed`` repeats them."""
        lib = L.lib()
        bce = labels is not None
        assert bce or not self.is_critic, "a TokenCritic trains against labels"
        attn_p, ff_p = float(self.transformer.attn_dropout), float(self.transformer.ff_dropout)
        for name, p in (("attn_dropout", attn_p), ("ff_dropout", ff_p)):
            if not 0.0 <= p <= 1.0:
                raise ValueError(f"{name} has to be between 0 and 1, but got {p}")
        dropout_on = self.training and (attn_p > 0 or ff_p > 0)
        ids_in = L.require_cuda(ids_in, "token ids", torch.int64)
        b, n = ids_in.shape
        assert _prod(patch_shape) == n, "video patch shape must cover the token sequence"
        dev = ids_in.device
        with torch.cuda.device(dev):
            table = self._table()
            assert n <= table.max_seq_len, \
                f"the video token sequence length you are passing in ({n}) is greater than the `max_seq_len` ({table.max_seq_len})"
            keep = Keep()
            if head is not None:  # same body, another head: a shallow copy of the table with the head members swapped
                table = L.MaskgitT.from_buffer_copy(table)
                table.head_w, table.head_b, table.head_w_h = keep.t(head.weight), keep.t(head.bias), None
            has_cross = context is not None and self.transformer.layers[0][2] is not None
            ctx_len = 0
            if has_cross:
                context = L.require_cuda(context, "text embeds", torch.float32)
                assert context.shape[0] == b and context.shape[-1] == self.transformer.layers[0][2].dim_context, \
                    "text embedding dimension is not correct"
                ctx_len = context.shape[1]
                if text_mask is None:
                    text_mask = torch.ones((b, ctx_len), device=dev, dtype=torch.bool)
                text_mask = L.require_cuda(text_mask.to(torch.uint8), "text mask")
            else:
                context = text_mask = None
            if video_mask is not None:
                video_mask = L.require_cuda(video_mask.to(torch.uint8), "video mask")
            if bce:
                labels = L.require_cuda(labels.reshape(b, n).float(), "critic labels", torch.float32)
                targets = token_mask = None
            else:
                targets = L.require_cuda(targets.reshape(b, n), "target ids", torch.int64)
                token_mask = L.require_cuda(token_mask.reshape(b, n).to(torch.uint8), "token mask")
            gtable, gk = self._grad_table(has_cross, owner=owner, head=head)
            logits = None
            if keep_logits and not bce:
                logits = torch.empty((b, n, table.num_tokens), dtype=torch.float32, device=dev)
            loss = torch.zeros((), dtype=torch.float32, device=dev)
            prec = L.PREC_BF16 if self.precision == L.PREC_BF16 else L.PREC_F32  # (split-bf16 is an inference mode)
            nbytes = lib.phk_maskgit_train_workspace_bytes(C.byref(table), b, n, ctx_len, int(bce), prec)
            ws = self._ws.get(nbytes, dev)
            pt, ph, pw = (int(v) for v in patch_shape)
            dropout = None
            if dropout_on:  # reserve exactly the counters the step's masks use (the C side owns the layout)
                counters = int(lib.phk_maskgit_train_dropout_counters(C.byref(table), b, n, ctx_len))
                assert counters >= 0, "phk_maskgit_train_dropout_counters: bad arguments"
                seed = _noise_seed(dev)
                offset = _rng_take(dev, seed, counters)
                dropout = C.byref(L.DropoutT(attn_p, ff_p, seed & (2 ** 64 - 1), offset))
            plan = self._overlap_plan(gk, owner if owner is not None else self, dev) if overlap_all_reduce else None
            if plan is not None:  # the C call records these events as gradient groups become final
                L.check(lib.phk_train_set_progress_events(plan["handles"], len(plan["events"])), "phk_train_set_progress_events")
            L.check(lib.phk_maskgit_train_step(C.byref(table), C.byref(gtable), L.ptr(ids_in), L.ptr(targets),
                                               L.ptr(token_mask), L.ptr(labels), b, n, pt, ph, pw, L.ptr(context),
                                               ctx_len, L.ptr(text_mask), L.ptr(video_mask), float(loss_scale),
                                               L.ptr(loss), L.ptr(logits), L.ptr(ws), ws.numel(), prec,
                                               L.stream_ptr(), dropout),
                    "phk_maskgit_train_step")
            if plan is not None:
                self._launch_overlapped_all_reduce(gk, plan)
        return loss, gk, logits

    def _gradient_groups(self, gk, owner):
        """Spans [lo, hi) (elements of the flat gradient bucket) by completion index of the backward: 0 = head + norm_out,
        1 .. depth = transformer layers depth-1 .. 0, depth + 1 = embeddings + position-bias MLP.  A group's parameters need
        not be adjacent in the bucket (token_emb / pos_emb open it, the position-bias MLP sits behind the layers): adjacent
        spans are merged, every element of the bucket belongs to exactly one span."""
        depth = self.transformer.depth
        base, esz = gk.flat.data_ptr(), gk.flat.element_size()
        groups = [[] for _ in range(depth + 2)]  # spans [lo, hi) in elements, by completion index
        for name, p in owner.named_parameters():
            lo = (gk.views[p].data_ptr() - base) // esz
            hi = lo + (p.numel() + 63) // 64 * 64
            idx = depth + 1  # embeddings, position-bias MLP: final at the very end
            if "transformer.layers." in name:
                idx = 1 + (depth - 1 - int(name.split("transformer.layers.")[1].split(".")[0]))
            elif "norm_out" in name or "to_logits" in name or "to_pred" in name:
                idx = 0
            if p.numel():
                groups[idx].append((lo, hi))
        for i, spans in enumerate(groups):  # a group's parameters need not be adjacent in the bucket: merge what is
            merged = []
            for lo, hi in sorted(spans):
                if merged and lo <= merged[-1][1]:
                    merged[-1][1] = max(merged[-1][1], hi)
                else:
                    merged.append([lo, hi])
            groups[i] = merged
        flat = sorted(sp for spans in groups for sp in spans)
        if any(a[1] > b[0] for a, b in zip(flat, flat[1:])):  # (padded spans of different groups overlap: no slicing)
            return None
        return groups

    def _overlap_plan(self, gk, owner, dev):
        """Data parallel, NCCL: slices of the flat gradient bucket in the order the backward finishes them (head +
        norm_out, layers depth-1 .. 0, embeddings + position-bias MLP) and one CUDA event per slice for
        phk_train_set_progress_events.  None when there is nothing to overlap (single process, non-NCCL backend)."""
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1 and gk.flat.is_cuda
                and dist.get_backend() == "nccl"):
            return None
        groups = self._gradient_groups(gk, owner)
        if groups is None:
            return None
        depth = self.transformer.depth
        cache = self.__dict__.setdefault("_overlap_cache", {})
        key = (dev, depth)
        if key not in cache:
            events = [torch.cuda.Event() for _ in range(depth + 2)]
            for e in events:
                e.record()  # creates the CUDA event behind the (lazily initialised) torch object
            handles = (C.c_void_p * len(events))(*[e.cuda_event for e in events])
            cache[key] = dict(events=events, handles=handles, stream=torch.cuda.Stream(device=dev))
        return dict(cache[key], groups=groups)

    def _launch_overlapped_all_reduce(self, gk, plan):
        """One all-reduce (mean) per finished slice on a side stream, each waiting only for its own event: the
        collective of the head / upper layers runs while the layers below are still in their backward kernels."""
        import torch.distributed as dist
        side, world = plan["stream"], dist.get_world_size()
        gk.flat.record_stream(side)
        for ev, spans in zip(plan["events"], plan["groups"]):
            if not spans:
                continue
            side.wait_event(ev)
            with torch.cuda.stream(side):
                for lo, hi in spans:
                    part = gk.flat[lo:hi]
                    dist.all_reduce(part, op=dist.ReduceOp.SUM)
                    part.div_(world)
        gk.reduced = torch.cuda.Event()
        gk.reduced.record(side)

    def _check_ids(self, x):
        """nn.Embedding raises on an id outside the table (phenaki_pytorch.py:194); the kernels only clamp.  One device
        sync, paid at the public forward entries only (the sampling loop produces its ids itself)."""
        rows = self.token_emb.weight.shape[0]
        lo, hi = int(x.min()), int(x.max())
        if lo < 0 or hi >= rows:
            raise IndexError(f"index out of range in self: token ids span [{lo}, {hi}], the embedding has {rows} rows")

    def _prepare(self, x, text_mask, video_patch_shape, context, cond_drop_prob):
        self._check_ids(x)
        if x.ndim == 4:
            video_patch_shape = tuple(x.shape[1:])
            x = x.reshape(x.shape[0], -1)
        assert video_patch_shape is not None, "video patch shape must be given"
        b = x.shape[0]
        ctx_kv, ctx_len = None, 0
        if context is not None and self.transformer.layers[0][2] is not None:
            ctx_len = context.shape[1]
            if text_mask is None:
                text_mask = torch.ones((b, ctx_len), device=x.device, dtype=torch.bool)
            if cond_drop_prob is not None and cond_drop_prob > 0:
                # prob_mask_like (phenaki_pytorch.py:73-79): p in {0,1} consume no RNG
                if cond_drop_prob >= 1:
                    keep = torch.zeros((b,), device=x.device, dtype=torch.bool)
                else:
                    keep = torch.rand((b,), device=x.device) < (1 - cond_drop_prob)
                text_mask = keep[:, None] & text_mask
            ctx_kv = self.context_kv(context)
        return x, tuple(int(v) for v in video_patch_shape), ctx_kv, ctx_len, text_mask


class MaskGit(_TokenTransformer):
    def __init__(self, *, dim, num_tokens, max_seq_len, gradient_shrink_alpha=0.1, heads=8, dim_head=64,
                 unconditional=False, attn_dropout=0.0, ff_dropout=0.0, **kwargs):
        super().__init__()
        self.dim = dim
        self.mask_id = num_tokens
        self.unconditional = unconditional
        self.token_emb = nn.Embedding(num_tokens + 1, dim)  # last token is the mask id
        self.max_seq_len = max_seq_len
        self.pos_emb = nn.Embedding(max_seq_len, dim)
        self.gradient_shrink_alpha = gradient_shrink_alpha
        self.continuous_pos_bias = ContinuousPositionBias(dim=dim_head, heads=heads, num_dims=3)
        self.transformer = Transformer(dim=dim, attn_num_null_kv=2, has_cross_attn=not unconditional,
                                       dim_head=dim_head, heads=heads, attn_dropout=attn_dropout,
                                       ff_dropout=ff_dropout, peg=True, **kwargs)
        self.to_logits = nn.Linear(dim, num_tokens)
        self._init_runtime()

    def forward(self, x, cond_drop_prob=0.0, text_mask=None, video_mask=None, video_patch_shape=None,
                return_embeds=False, context=None, **kwargs):
        assert x.ndim in {2, 4}, "video token ids must be of shape (batch, seq) or (batch, frame, height, width)"
        x, shape, ctx_kv, ctx_len, text_mask = self._prepare(x, text_mask, video_patch_shape, context, cond_drop_prob)
        return self._run(x, shape, ctx_kv=ctx_kv, ctx_len=ctx_len, text_mask=text_mask, video_mask=video_mask,
                         return_embeds=return_embeds)

    def forward_with_cond_scale(self, x, *, cond_scale=3, text_mask=None, video_mask=None, video_patch_shape=None,
                                context=None, return_embeds=False, **kwargs):
        """phenaki_pytorch.py:149-161.  Both passes run as ONE batch of 2b sequences (the second half sees
        an all-False text mask) and are combined by phk_cfg_combine."""
        if cond_scale == 1:
            return self.forward(x, cond_drop_prob=0.0, text_mask=text_mask, video_mask=video_mask,
                                video_patch_shape=video_patch_shape, context=context, return_embeds=return_embeds)
        x, shape, ctx_kv, ctx_len, text_mask = self._prepare(x, text_mask, video_patch_shape, context, 0.0)
        both = self._run(x, shape, ctx_kv=ctx_kv, ctx_len=ctx_len, text_mask=text_mask, video_mask=video_mask,
                         cfg_pair=True, return_embeds=return_embeds)
        b = x.shape[0]
        out = torch.empty_like(both[:b])
        L.check(L.lib().phk_cfg_combine(L.ptr(both[:b]), L.ptr(both[b:]), float(cond_scale), L.ptr(out),
                                        out.numel(), L.stream_ptr()), "phk_cfg_combine")
        return out


class TokenCritic(_TokenTransformer):
    is_critic = True

    def __init__(self, *, dim, num_tokens, max_seq_len, has_cross_attn=False, attn_dropout=0.0, ff_dropout=0.0,
                 **kwargs):
        super().__init__()
        self.has_cross_attn = has_cross_attn
        self.mask_id = num_tokens
        self.token_emb = nn.Embedding(num_tokens + 1, dim)
        self.pos_emb = nn.Embedding(max_seq_len, dim)
        self.transformer = Transformer(dim=dim, peg=True, attn_dropout=attn_dropout, ff_dropout=ff_dropout,
                                       has_cross_attn=has_cross_attn, **kwargs)
        self.to_logits = nn.Sequential(nn.Linear(dim, 1), _NoParams())
        self._init_runtime()

    def _scores(self, embeds_cond, embeds_null, cond_scale, rows, noise=None, noise_K=0.0, noise_mult=0.0,
                seg=(0, 0, 0)):
        table = self._table()
        out = torch.empty((rows,), dtype=torch.float32, device=embeds_cond.device)
        L.check(L.lib().phk_critic_scores(L.ptr(embeds_cond), L.ptr(embeds_null), table.head_w, table.head_b,
                                          L.ptr(noise), float(cond_scale), float(noise_K), float(noise_mult),
                                          L.ptr(out), rows, table.dim, *seg, L.stream_ptr()), "phk_critic_scores")
        return out

    def forward(self, x, text_mask=None, cond_drop_prob=None, context=None, video_mask=None,
                video_patch_shape=None, **kwargs):
        shape = tuple(video_patch_shape) if video_patch_shape is not None else tuple(x.shape[1:])
        x = x.reshape(x.shape[0], -1)
        if context is not None and cond_drop_prob is None:
            raise TypeError("cond_drop_prob must be given when a context is passed (phenaki_pytorch.py:286)")
        x, shape, ctx_kv, ctx_len, text_mask = self._prepare(x, text_mask, shape, context, cond_drop_prob)
        emb = self._run(x, shape, ctx_kv=ctx_kv, ctx_len=ctx_len, text_mask=text_mask, video_mask=video_mask)
        b, n = x.shape
        return self._scores(emb, None, 1.0, b * n).reshape(b, n)

    def forward_with_cond_scale(self, x, *, cond_scale=3, text_mask=None, context=None, video_mask=None,
                                video_patch_shape=None, **kwargs):
        if cond_scale == 1:
            return self.forward(x, text_mask=text_mask, cond_drop_prob=0.0, context=context, video_mask=video_mask,
                                video_patch_shape=video_patch_shape)
        shape = tuple(video_patch_shape) if video_patch_shape is not None else tuple(x.shape[1:])
        x = x.reshape(x.shape[0], -1)
        x, shape, ctx_kv, ctx_len, text_mask = self._prepare(x, text_mask, shape, context, 0.0)
        both = self._run(x, shape, ctx_kv=ctx_kv, ctx_len=ctx_len, text_mask=text_mask, video_mask=video_mask,
                         cfg_pair=True)
        b, n = x.shape
        return self._scores(both[:b], both[b:], cond_scale, b * n).reshape(b, n)


class SelfCritic(nn.Module):
    """phenaki_pytorch.py:307-336: Linear(dim,1) on the MaskGit embeddings."""

    def __init__(self, maskgit: MaskGit):
        super().__init__()
        self.maskgit = maskgit
        self.to_pred = nn.Sequential(nn.Linear(maskgit.dim, 1), _NoParams())
        self.has_cross_attn = not maskgit.unconditional

    def _head(self, cond, null, cond_scale, rows, **kw):
        w = L.require_cuda(self.to_pred[0].weight.detach(), "to_pred.weight", torch.float32)
        bb = L.require_cuda(self.to_pred[0].bias.detach(), "to_pred.bias", torch.float32)
        out = torch.empty((rows,), dtype=torch.float32, device=cond.device)
        L.check(L.lib().phk_critic_scores(L.ptr(cond), L.ptr(null), L.ptr(w), L.ptr(bb), L.ptr(kw.get("noise")),
                                          float(cond_scale), float(kw.get("noise_K", 0.0)),
                                          float(kw.get("noise_mult", 0.0)), L.ptr(out), rows, self.maskgit.dim,
                                          *kw.get("seg", (0, 0, 0)), L.stream_ptr()), "phk_critic_scores")
        return out

    def forward(self, x, *args, **kwargs):
        emb = self.maskgit(x, *args, return_embeds=True, **kwargs)
        b, n = emb.shape[:2]
        return self._head(emb, None, 1.0, b * n).reshape(b, n)

    def train_step(self, ids_in, patch_shape, *, labels, **kw):
        """BCE training step of the self critic: the MaskGit body with ``to_pred`` as its head; the gradient bucket
        follows ``self.parameters()`` (MaskGit's parameters, then to_pred)."""
        return self.maskgit.train_step(ids_in, patch_shape, labels=labels, head=self.to_pred[0], owner=self, **kw)

    def forward_with_cond_scale(self, x, *, cond_scale=3, **kwargs):
        if cond_scale == 1:
            return self.forward(x, cond_drop_prob=0.0, **kwargs)
        mg = self.maskgit
        xx, shape, ctx_kv, ctx_len, text_mask = mg._prepare(x, kwargs.get("text_mask"), kwargs.get("video_patch_shape"),
                                                            kwargs.get("context"), 0.0)
        both = mg._run(xx, shape, ctx_kv=ctx_kv, ctx_len=ctx_len, text_mask=text_mask,
                       video_mask=kwargs.get("video_mask"), cfg_pair=True, return_embeds=True)
        b, n = xx.shape
        return self._head(both[:b], both[b:], cond_scale, b * n).reshape(b, n)


class _TrainStepFn(torch.autograd.Function):
    """Connects phk_maskgit_train_step to torch autograd: forward returns the loss that libphk computed, backward hands
    the gradients libphk computed in the same call to the parameters (scaled by the upstream gradient), so
    ``loss.backward()`` followed by any torch optimizer works as with the reference."""

    @staticmethod
    def forward(ctx, loss, grad_keep, sync, *params):
        ctx.keep, ctx.sync = grad_keep, sync
        ctx.grads = [grad_keep.grad_of(p) for p in params]
        return loss.clone()

    @staticmethod
    def backward(ctx, gout):
        if ctx.sync:  # data parallel: average the one flat gradient bucket over the ranks (DDP's all-reduce)
            reduced = getattr(ctx.keep, "reduced", None)
            if reduced is not None:  # already launched slice by slice on the side stream, overlapped with the backward
                torch.cuda.current_stream().wait_event(reduced)
            else:
                sharding.all_reduce_mean_(ctx.keep.flat)
            ctx.sync = False
        out = (None, None, None, *[None if g is None else g * gout for g in ctx.grads])  # copies: the bucket is free again
        ctx.keep.busy = False
        return out


def get_mask_subset_with_prob(mask, prob, u=None):
    """phenaki_pytorch.py:43-55: chooses round(prob * n_valid) (>= 1) positions per row by the RANK of a uniform draw.
    ``u`` (b, n) injects the draw (tests); boolean plumbing on the device, no arithmetic of the network."""
    batch, seq_len = mask.shape
    num_tokens = mask.sum(dim=-1)
    num_pads = seq_len - num_tokens
    num_masked = (prob * num_tokens).round().clamp(min=1)
    if u is None:
        u = torch.rand((batch, seq_len), device=mask.device)
    ranks = u.argsort(dim=-1) - num_pads[:, None]
    ranks = ranks.masked_fill(ranks < 0, seq_len)
    return ranks < num_masked[:, None]


def demask_counts(num_tokens, steps):
    """k_s = clamp(round(N * cos(pi/2 * s/S)), 1) for s = 1..S-1 in fp32, round-half-even
    (phenaki_pytorch.py:485-486), precomputed on the host: no per-step device sync."""
    ks = []
    for step in range(1, steps):
        t = np.float32(step / steps)
        a = np.float32(np.float32(t * np.float32(math.pi)) * np.float32(0.5))
        v = np.float32(np.float32(num_tokens) * np.cos(a, dtype=np.float32))
        ks.append(max(int(np.rint(v)), 1))
    return ks


_T5_DIMS = {"t5-small": 512, "t5-base": 768, "t5-large": 1024, "t5-3b": 1024, "t5-11b": 1024,
            "google/t5-v1_1-small": 512, "google/t5-v1_1-base": 768, "google/t5-v1_1-large": 1024,
            "google/t5-v1_1-xl": 2048, "google/t5-v1_1-xxl": 4096}
DEFAULT_T5_NAME = "google/t5-v1_1-base"


def _t5_encode_text(texts, name=DEFAULT_T5_NAME, output_device=None):
    """Text side (t5.py:64-103) is a third-party model outside the hot path (SURVEY row 9): thin lazy
    glue around HF transformers; padded positions are zero-filled so `any(emb != 0)` recovers the mask."""
    from transformers import AutoTokenizer, T5EncoderModel  # needs local weights
    cache = _t5_encode_text.__dict__.setdefault("cache", {})
    if name not in cache:
        cache[name] = (AutoTokenizer.from_pretrained(name), T5EncoderModel.from_pretrained(name).eval())
    tok, model = cache[name]
    dev = output_device if output_device is not None else "cpu"
    model.to(dev)
    enc = tok(texts, return_tensors="pt", padding="longest", max_length=256, truncation=True).to(dev)
    with torch.no_grad():
        out = model(input_ids=enc.input_ids, attention_mask=enc.attention_mask).last_hidden_state
    return out.masked_fill(~enc.attention_mask[..., None].bool(), 0.0).float()


class Phenaki(nn.Module):
    def __init__(self, *, maskgit: MaskGit, cvivit: CViViT, critic: Optional[Union[TokenCritic, SelfCritic]] = None,
                 steps=18, t5_name=DEFAULT_T5_NAME, sample_temperature=0.0, text_embed_dim=None,
                 cond_drop_prob=0.25, max_text_len=128, self_token_critic=False, critic_loss_weight=1.0,
                 critic_noise_anneal_schedule="decay", critic_train_sample_temperature=1.0):
        super().__init__()
        self.cvivit = cvivit.copy_for_eval()
        self.maskgit = maskgit
        self.unconditional = maskgit.unconditional
        self.mask_id = maskgit.mask_id
        assert not (self_token_critic and critic is not None)
        if self_token_critic:
            critic = SelfCritic(maskgit)
        if critic is not None:
            critic = critic.eval()
        assert critic is None or self_token_critic or (not maskgit.unconditional) == critic.has_cross_attn
        self.critic = critic
        self.critic_noise_anneal_schedule = critic_noise_anneal_schedule
        self.critic_loss_weight = critic_loss_weight
        self.critic_train_sample_temperature = critic_train_sample_temperature
        self.steps = steps
        self.sample_temperature = sample_temperature
        if text_embed_dim is None:
            assert t5_name in _T5_DIMS, f"unknown T5 name {t5_name}: pass text_embed_dim"
            text_embed_dim = _T5_DIMS[t5_name]
        self.encode_texts = partial(_t5_encode_text, name=t5_name)
        self.text_embed_dim = text_embed_dim
        self.max_text_len = max_text_len
        assert cond_drop_prob > 0.0
        self.cond_drop_prob = cond_drop_prob
        # training under torch.distributed: average the gradient bucket over the ranks in backward() (what the
        # reference gets from Accelerate's DDP wrapper, phenaki_trainer.py); no-op without a process group
        self.sync_gradients = True
        # bf16 mode: ONE C call per demasking iteration with all state in device memory
        # (phk_maskgit_demask_iteration), replayed as ONE CUDA-graph launch per iteration from the third sample() with the
        # same shapes on (BASELINE north_star: one launch per decode iteration).  Validated on the H100 against the
        # per-step loop (identical ids: same noise counters).  False restores the per-step loop.
        self.iteration_call = True
        self._iter_bufs = {}
        self.fused_head = True  # bf16 mode: logits head + CFG + gumbel argmax fused into one GEMM (no (b,n,V) logits)

    def _fused_step_supported(self):
        """Shape limits of the fused demasking step (phk_maskgit_sample_step / phk_head_sample keep the whole
        embedding row of a token tile in shared memory): other widths take phk_maskgit_forward + phk_sample_tokens."""
        dim = self.maskgit.dim
        return dim <= 512 and dim % 128 == 0

    # ---- the demasking loop (phenaki_pytorch.py:473-550) -------------------------------------------------
    @torch.no_grad()
    def sample_token_ids(self, *, num_tokens, patch_shape, batch_size, text_embeds=None, text_mask=None,
                         prime_token_ids=None, cond_scale=3.0, starting_temperature=0.9, noise_K=1.0,
                         noise_fn=None, trace=None):
        """Runs the ``steps`` demasking iterations and returns the final ids (b, num_tokens) int64.

        Per iteration: phk_topk_mask (re-mask) -> phk_maskgit_forward (CFG pair) -> phk_sample_tokens
        (CFG + gumbel argmax + confidence) [-> critic forward + phk_critic_scores].  No host sync.
        ``noise_fn(shape, tag)`` (tests) injects the uniform draws; default: in-kernel Philox for the
        V-wide gumbel noise, torch.rand for the (b, n) critic noise."""
        lib = L.lib()
        mg = self.maskgit
        dev = next(mg.parameters()).device
        steps, n, b = self.steps, num_tokens, batch_size
        plen = 0 if prime_token_ids is None else prime_token_ids.shape[-1]
        with torch.cuda.device(dev):
            ctx_kv = critic_kv = None
            ctx_len = 0
            if text_embeds is not None:
                text_embeds = L.require_cuda(text_embeds, "text embeds", torch.float32)
                if text_mask is None:
                    text_mask = torch.any(text_embeds != 0, dim=-1)  # phenaki_pytorch.py:461
                text_mask = text_mask.to(torch.uint8)  # once per sample: the per-step calls take it as it is
                ctx_len = text_embeds.shape[1]
                ctx_kv = mg.context_kv(text_embeds)  # once per sample, not once per forward
                if isinstance(self.critic, TokenCritic) and self.critic.has_cross_attn:
                    critic_kv = self.critic.context_kv(text_embeds)
            ids = torch.full((b, n), self.mask_id, dtype=torch.int64, device=dev)
            mask = torch.ones((b, n), dtype=torch.uint8, device=dev)
            scores = torch.empty((b, n), dtype=torch.float32, device=dev)
            pred = torch.empty((b, n), dtype=torch.int64, device=dev)
            inp = ids if plen == 0 else torch.cat((prime_token_ids, ids), dim=-1)
            seg = (0, 0, 0) if plen == 0 else (n, plen + n, plen)
            ks = demask_counts(n, steps)
            seed = _noise_seed(dev)
            vocab = mg.to_logits.weight.shape[0]
            have_scores = False
            iterations = (self.iteration_call and self.fused_head and mg.precision == L.PREC_BF16 and noise_fn is None
                          and cond_scale != 1 and trace is None and self._fused_step_supported())
            # an unknown anneal schedule takes the per-step loop, which raises on it
            critic_ok = self.critic is None or (
                self.critic_noise_anneal_schedule in ("fixed", "decay", "increase")
                and (isinstance(self.critic, SelfCritic)
                     or (isinstance(self.critic, TokenCritic) and self.critic.precision == L.PREC_BF16)))
            if iterations and critic_ok:
                return self._sample_by_iterations(b, n, plen, prime_token_ids, patch_shape, ctx_kv, critic_kv, ctx_len,
                                                  text_mask, cond_scale, starting_temperature, noise_K, ks, seed, vocab, dev)
            # the whole sample's V-wide noise counters are reserved up front (iteration s uses first + s * stride), as the
            # iteration path does: the critic's torch.rand draws then follow them in the generator stream on every path
            stride = _noise_stride(b * n, vocab)
            first_offset = _rng_take(dev, seed, stride * steps)
            for step in range(steps):
                last = step == steps - 1
                til_x0 = steps - (step + 1)
                if step > 0 and have_scores:
                    L.check(lib.phk_topk_mask(L.ptr(scores), b, n, ks[step - 1], L.ptr(mask), L.ptr(ids),
                                              self.mask_id, L.stream_ptr()), "phk_topk_mask")
                if plen:
                    inp[:, plen:].copy_(ids)
                use_cfg = cond_scale != 1
                temperature = starting_temperature * (til_x0 / steps)
                offset = first_offset + step * stride
                fused = (self.fused_head and mg.precision == L.PREC_BF16 and noise_fn is None and use_cfg
                         and trace is None and self._fused_step_supported())
                if fused:
                    # one launch sequence per iteration, logits never leave the SM (statistical-noise mode)
                    # exactly ks[step - 1] tokens per sequence were re-masked above (all n at the first step): the head
                    # only has to look at those rows
                    mg._sample_step(inp, patch_shape, ctx_kv=ctx_kv, ctx_len=ctx_len, text_mask=text_mask,
                                    cond_scale=cond_scale, temperature=temperature, seed=seed & (2 ** 64 - 1),
                                    offset=offset, mask=mask, ids=ids, pred=pred, scores=scores,
                                    masked_per_seq=n if step == 0 else ks[step - 1], prime_len=plen)
                else:
                    logits = mg._run(inp, patch_shape, ctx_kv=ctx_kv, ctx_len=ctx_len, text_mask=text_mask,
                                     cfg_pair=use_cfg)
                    u = None
                    if noise_fn is not None:
                        u = L.require_cuda(noise_fn((b, n, vocab), f"gumbel{step}"), "gumbel noise", torch.float32)
                    cond = logits[:b]
                    null = logits[b:] if use_cfg else None
                    L.check(lib.phk_sample_tokens(L.ptr(cond), L.ptr(null), vocab, L.ptr(u), seed & (2 ** 64 - 1),
                                                  offset, float(cond_scale), float(temperature), L.ptr(mask),
                                                  L.ptr(ids), L.ptr(pred), L.ptr(scores), b * n, vocab, *seg,
                                                  L.stream_ptr()), "phk_sample_tokens")
                have_scores = True
                if trace is not None:
                    trace.append(dict(step=step, mask=mask.bool().clone(), pred=pred.clone(), ids=ids.clone()))
                if last:
                    break
                if self.critic is not None:
                    if plen:
                        inp[:, plen:].copy_(ids)
                    mult = {"fixed": 1.0, "decay": til_x0 / steps, "increase": (step + 1) / steps}.get(
                        self.critic_noise_anneal_schedule)
                    if mult is None:
                        raise ValueError("invalid critic noise anneal schedule name")
                    noise = (noise_fn((b, n), f"critic{step}") if noise_fn is not None
                             else torch.rand((b, n), device=dev, dtype=torch.float32))
                    noise = L.require_cuda(noise, "critic noise", torch.float32)
                    if isinstance(self.critic, SelfCritic):
                        both = mg._run(inp, patch_shape, ctx_kv=ctx_kv, ctx_len=ctx_len, text_mask=text_mask,
                                       cfg_pair=use_cfg, return_embeds=True)
                        head = self.critic._head
                    else:
                        both = self.critic._run(inp, patch_shape, ctx_kv=critic_kv,
                                                ctx_len=ctx_len if critic_kv is not None else 0,
                                                text_mask=text_mask if critic_kv is not None else None,
                                                cfg_pair=use_cfg)
                        head = None
                    c_e, n_e = both[:b], (both[b:] if use_cfg else None)
                    if head is not None:
                        scores = head(c_e, n_e, cond_scale, b * n, noise=noise, noise_K=noise_K, noise_mult=mult,
                                      seg=seg).reshape(b, n)
                    else:
                        scores = self.critic._scores(c_e, n_e, cond_scale, b * n, noise=noise, noise_K=noise_K,
                                                     noise_mult=mult, seg=seg).reshape(b, n)
                if trace is not None:
                    trace[-1]["scores"] = scores.clone()
        return ids

    def _sample_by_iterations(self, b, n, plen, prime_token_ids, patch_shape, ctx_kv, critic_kv, ctx_len, text_mask,
                              cond_scale, starting_temperature, noise_K, ks, seed, vocab, dev):
        """The demasking loop as ``steps`` calls of phk_maskgit_demask_iteration: re-mask, MaskGit CFG pair + tail and,
        with a critic, critic CFG pair + scores are ONE launch sequence per iteration.  Token state, mask, scores, the
        text keys / values and the noise key live in buffers that persist across ``sample`` calls, so the library sees
        the same arguments at iteration s of every sample (temperature, k and the critic-noise multiplier of iteration s
        are the same in every sample) and can replay one captured CUDA graph per iteration."""
        lib, mg, steps, critic = L.lib(), self.maskgit, self.steps, self.critic
        token_critic = isinstance(critic, TokenCritic)
        key = (b, n, plen, ctx_len, dev, None if critic is None else id(critic),
               None if critic_kv is None else tuple(critic_kv.shape))
        bufs = self._iter_bufs.get(key)
        if bufs is None:
            z = lambda shape, dt: torch.empty(shape, dtype=dt, device=dev)
            bufs = self._iter_bufs[key] = dict(
                ids=z((b, n), torch.int64), mask=z((b, n), torch.uint8), scores=z((b, n), torch.float32),
                pred=z((b, n), torch.int64), rng=z((2,), torch.int64), noise=z((b, n), torch.float32),
                inp=z((b, plen + n), torch.int64) if plen else None,
                ctx_kv=None if ctx_kv is None else torch.empty_like(ctx_kv),
                critic_kv=None if critic_kv is None else torch.empty_like(critic_kv),
                text_mask=None if text_mask is None else z(tuple(text_mask.shape), torch.uint8))
        bufs["ids"].fill_(self.mask_id)
        bufs["mask"].fill_(1)
        bufs["scores"].zero_()
        if plen:
            bufs["inp"][:, :plen].copy_(prime_token_ids)
        if ctx_kv is not None:
            bufs["ctx_kv"].copy_(ctx_kv)
            bufs["text_mask"].copy_(text_mask.to(torch.uint8))
        if critic_kv is not None:
            bufs["critic_kv"].copy_(critic_kv)
        stride = _noise_stride(b * n, vocab)
        as_i64 = lambda v: v - (1 << 64) if v >= (1 << 63) else v  # uint64 bit pattern in an int64 tensor
        first = _rng_take(dev, seed, stride * steps)  # the library advances the device-side counter by `stride` per iteration
        # two scalar fills, not a host tensor: a pageable H2D copy synchronises the stream first, which stalled the host at the
        # start of every sample until the previous scene's decode had drained (make_video was host-bound through it)
        bufs["rng"][0].fill_(as_i64(seed & (2 ** 64 - 1)))
        bufs["rng"][1].fill_(as_i64(first))
        with torch.cuda.device(dev):
            table = mg._table()
            ctable, head_w, head_b, keep = None, None, None, None
            if token_critic:
                ctable = critic._table()
                head_w, head_b = ctable.head_w, ctable.head_b
            elif critic is not None:  # SelfCritic: Linear(dim, 1) on the MaskGit's embeddings
                keep = (L.require_cuda(critic.to_pred[0].weight.detach(), "to_pred.weight", torch.float32),
                        L.require_cuda(critic.to_pred[0].bias.detach(), "to_pred.bias", torch.float32))
                head_w, head_b = L.ptr(keep[0]), L.ptr(keep[1])
            cref = C.byref(ctable) if ctable is not None else None
            nbytes = lib.phk_maskgit_demask_iteration_workspace_bytes(C.byref(table), cref, b, plen + n, ctx_len)
            ws = mg._ws.get(nbytes, dev)
            bias = mg._pos_bias(table, patch_shape, dev)
            pt, ph, pw = (int(v) for v in patch_shape)
            inp = bufs["inp"] if plen else bufs["ids"]
            for step in range(steps):
                til_x0 = steps - (step + 1)
                temperature = starting_temperature * (til_x0 / steps)
                with_critic = critic is not None and step < steps - 1
                mult = 0.0
                if with_critic:
                    mult = {"fixed": 1.0, "decay": til_x0 / steps, "increase": (step + 1) / steps}[
                        self.critic_noise_anneal_schedule]
                    bufs["noise"].uniform_()  # torch.rand((b, n)) of the per-step loop, drawn into the stable buffer
                L.check(lib.phk_maskgit_demask_iteration(
                    C.byref(table), cref, head_w, head_b, L.ptr(inp), L.ptr(bufs["ids"]), L.ptr(bufs["mask"]),
                    L.ptr(bufs["scores"]), L.ptr(bufs["pred"]), b, n, plen, pt, ph, pw, L.ptr(bufs["ctx_kv"]),
                    L.ptr(bufs["critic_kv"]) if token_critic else None, ctx_len, L.ptr(bufs["text_mask"]), L.ptr(bias),
                    float(cond_scale), float(temperature), L.ptr(bufs["rng"]), 0 if step == 0 else ks[step - 1],
                    L.ptr(bufs["noise"]) if with_critic else None, float(noise_K), float(mult), int(not with_critic),
                    L.ptr(ws), ws.numel(), L.stream_ptr()), "phk_maskgit_demask_iteration")
        return bufs["ids"].clone()

    @torch.no_grad()
    def sample(self, *, num_frames, texts: Union[List[str], str, None] = None, prime_frames=None, batch_size=1,
               cond_scale=3.0, starting_temperature=0.9, noise_K=1.0, text_embeds=None, return_token_ids=False,
               noise_fn=None):
        """phenaki_pytorch.py:418-560.  Extra keywords: ``text_embeds`` (precomputed T5 output, SURVEY 8f-4),
        ``return_token_ids`` (skip the final C-ViViT decode), ``noise_fn`` (inject the uniform draws)."""
        # eval_decorator (phenaki_pytorch.py:31-38).  The mode flags only matter to dropout, which only the training step
        # applies (the sampling kernels have none); the walk over ~600 submodules cost ~2 ms of host time per call,
        # twice per sample, so it is skipped when the model is already in eval mode.
        was_training = self.training
        if was_training:
            self.eval()
        try:
            prime_ids, prime_num_frames = None, 0
            if prime_frames is not None:
                pids = self.cvivit(prime_frames, return_only_codebook_ids=True)
                prime_ids = pids.reshape(pids.shape[0], -1)
                prime_num_frames = prime_frames.shape[2]
            num_tokens = self.cvivit.num_tokens_per_frames(num_frames, include_first_frame=prime_frames is None)
            text_mask = None
            dev = next(self.maskgit.parameters()).device
            if texts is not None and text_embeds is None:
                if isinstance(texts, str):
                    texts = [texts]
                text_embeds = self.encode_texts(texts, output_device=dev)
            if text_embeds is not None:
                text_embeds = text_embeds.to(dev)
                text_mask = torch.any(text_embeds != 0, dim=-1)
                batch_size = text_embeds.shape[0]
            patch_shape = self.cvivit.get_video_patch_shape(num_frames + prime_num_frames, include_first_frame=True)
            ids = self.sample_token_ids(num_tokens=num_tokens, patch_shape=patch_shape, batch_size=batch_size,
                                        text_embeds=text_embeds, text_mask=text_mask, prime_token_ids=prime_ids,
                                        cond_scale=cond_scale, starting_temperature=starting_temperature,
                                        noise_K=noise_K, noise_fn=noise_fn)
            if prime_ids is not None:
                ids_full = torch.cat((prime_ids, ids), dim=-1)
            else:
                ids_full = ids
            if return_token_ids:
                return ids
            video = self.cvivit.decode_from_codebook_indices(ids_full)
            if prime_ids is not None:
                video = video[:, :, prime_num_frames:]
            return video
        finally:
            if was_training:
                self.train(True)

    def sample_images(self, *, texts=None, batch_size=1, cond_scale=3.0, starting_temperature=0.9, noise_K=1.0):
        video = self.sample(texts=texts, num_frames=1, cond_scale=cond_scale,
                            starting_temperature=starting_temperature, noise_K=noise_K)
        return video.squeeze(2)

    def forward(self, videos=None, *, texts: Optional[List[str]] = None, video_codebook_ids=None,
                video_frame_mask=None, text_embeds=None, cond_drop_prob=None, only_train_generator=False,
                only_train_critic=False, draw_fn=None):
        """Training loss (phenaki_pytorch.py:562-687): masked-token cross entropy of MaskGit (+ TokenCritic BCE).
        The returned scalar is connected to the parameters through ``_TrainStepFn``: ``loss.backward()`` fills
        ``p.grad`` with the gradients the hand-written backward kernels computed (phk_maskgit_train_step).
        ``draw_fn(shape, tag)`` (tests) injects the draws 'rand_step' (b,), 'perm' (b, n) and 'gumbel' (b, n, V).
        ``maskgit.precision`` selects fp32 (parity) or bf16 tensor-core products.  Validated on the H100 against the
        reference's autograd loss and every parameter gradient (tests/test_gpu_train.py, both precision modes)."""
        assert not (only_train_generator and only_train_critic)
        assert (videos is not None) ^ (video_codebook_ids is not None), "either raw video or codebook ids"
        assert ((text_embeds is not None) ^ (texts is not None)) ^ self.unconditional, \
            "either raw text of text embeds must be given, and if unconditional, none should be given"
        assert not (text_embeds is not None and text_embeds.shape[-1] != self.text_embed_dim), \
            "text embedding dimension is not correct"
        mg = self.maskgit
        dev = next(mg.parameters()).device
        if video_codebook_ids is None:
            assert videos.ndim in {4, 5}
            if videos.ndim == 4:
                videos = videos.unsqueeze(2)
            with torch.no_grad():
                self.cvivit.eval()
                video_codebook_ids = self.cvivit(videos, return_only_codebook_ids=True)
        text_mask = None
        if not self.unconditional:
            if text_embeds is None:
                with torch.no_grad():
                    text_embeds = self.encode_texts(texts, output_device=dev)
            text_embeds = text_embeds.to(dev)
            text_mask = torch.any(text_embeds != 0, dim=-1)
        # the reference overwrites cond_drop_prob with 0 here (:594, SURVEY defects): no text dropout while training
        video_mask = None
        if video_frame_mask is not None:
            video_mask = self.cvivit.calculate_video_token_mask(videos, video_frame_mask=video_frame_mask)
        patch_shape = tuple(int(v) for v in video_codebook_ids.shape[1:])
        ids = video_codebook_ids.reshape(video_codebook_ids.shape[0], -1).to(dev)
        if videos is None:  # caller-supplied ids: nn.Embedding would raise on an id outside the table (one device sync)
            mg._check_ids(ids)
        batch, seq = ids.shape
        draw = draw_fn if draw_fn is not None else (lambda shape, tag: None)
        rand_step = draw((batch,), "rand_step")
        if rand_step is None:
            rand_step = torch.randint(0, self.steps, (batch,), device=dev)
        mask_token_prob = torch.cos(rand_step.to(dev) * math.pi * 0.5 / self.steps)  # cosine schedule (:615)
        if video_mask is None:
            video_mask = torch.ones((batch, seq), device=dev, dtype=torch.bool)
        u = draw((batch, seq), "perm")
        mask_token_mask = get_mask_subset_with_prob(video_mask, mask_token_prob, None if u is None else u.to(dev))
        masked_input = torch.where(mask_token_mask, self.mask_id, ids)
        need_critic = self.critic is not None and not only_train_generator
        kw = dict(context=text_embeds, text_mask=text_mask, video_mask=video_mask)
        loss = None
        if only_train_critic:
            with torch.no_grad():
                logits = mg._run(masked_input, patch_shape, ctx_kv=None if text_embeds is None else mg.context_kv(text_embeds),
                                 ctx_len=0 if text_embeds is None else text_embeds.shape[1], text_mask=text_mask,
                                 video_mask=video_mask)
        else:
            ce, gk, logits = mg.train_step(masked_input, patch_shape, targets=ids, token_mask=mask_token_mask,
                                           keep_logits=need_critic, overlap_all_reduce=self.sync_gradients, **kw)
            loss = _TrainStepFn.apply(ce, gk, self.sync_gradients, *mg.parameters())
        if not need_critic:
            return loss
        # sample the predicted masked tokens (:646) and train the critic to tell which ones were changed (:650-675)
        vocab = logits.shape[-1]
        gu = draw((batch, seq, vocab), "gumbel")
        pred = torch.empty((batch, seq), dtype=torch.int64, device=dev)
        ones = torch.ones((batch, seq), dtype=torch.uint8, device=dev)
        scratch_ids = torch.empty_like(pred)
        seed = _noise_seed(dev)
        offset = _rng_take(dev, seed, _noise_stride(batch * seq, vocab))
        gu_dev = None if gu is None else L.require_cuda(gu.to(dev), "gumbel noise", torch.float32)  # kept alive past the launch
        L.check(L.lib().phk_sample_tokens(L.ptr(logits), None, vocab, L.ptr(gu_dev), seed & (2 ** 64 - 1), offset, 1.0,
                                          float(self.critic_train_sample_temperature), L.ptr(ones), L.ptr(scratch_ids),
                                          L.ptr(pred), None, batch * seq, vocab, 0, 0, 0, L.stream_ptr()),
                "phk_sample_tokens")
        critic_input = torch.where(mask_token_mask, pred, ids)
        labels = (ids != pred).float()
        weight = 1.0 if only_train_critic else self.critic_loss_weight
        ckw = kw if self.critic.has_cross_attn else dict(video_mask=video_mask)
        # (a SelfCritic differentiates MaskGit a second time: autograd adds the two contributions to p.grad)
        bce, cgk, _ = self.critic.train_step(critic_input, patch_shape, labels=labels,
                                             overlap_all_reduce=self.sync_gradients, **ckw)
        critic_loss = _TrainStepFn.apply(bce, cgk, self.sync_gradients, *self.critic.parameters())
        return critic_loss * weight if loss is None else loss + critic_loss * weight


def make_video(phenaki: Phenaki, texts: List[str], num_frames, prime_lengths):
    """phenaki_pytorch.py:691-714: scenes chained through `prime_lengths` trailing frames."""
    num_scenes = len(texts)
    num_frames = num_frames if isinstance(num_frames, tuple) else (num_frames,) * num_scenes
    prime_lengths = prime_lengths if isinstance(prime_lengths, tuple) else (prime_lengths,) * (num_scenes - 1)
    prime_lengths = (*prime_lengths, 0)
    scenes, prime = [], None
    for text, scene_frames, next_prime in zip(texts, num_frames, prime_lengths):
        video = phenaki.sample(texts=text, prime_frames=prime, num_frames=scene_frames)
        scenes.append(video)
        prime = video[:, :, -next_prime:]
    return torch.cat(scenes, dim=2), scenes
