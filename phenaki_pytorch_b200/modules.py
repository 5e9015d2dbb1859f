"""Host-side mirror of the reference's transformer building blocks (attention.py).

These classes are PARAMETER HOLDERS with the reference's attribute names, shapes and
construction order, so that (a) ``load_state_dict(reference.state_dict())`` is strict-clean and
(b) seeded default construction yields bit-identical weights (SURVEY.md 8b).  They contain no
math: all compute happens in libphk.so, which receives the weights through the ctypes tables
built by ``*_table`` below.
"""
import ctypes as C
import math

import torch
from torch import nn

from . import _lib as L


class LayerNorm(nn.Module):
    """attention.py:29-36: learnable gamma, constant zero beta kept as a (persistent) buffer."""

    def __init__(self, dim):
        super().__init__()
        self.gamma = nn.Parameter(torch.ones(dim))
        self.register_buffer("beta", torch.zeros(dim))


class _NoParams(nn.Module):
    """Stands in for parameter-free members of a reference nn.Sequential (Rearrange, GEGLU, ...)
    so that the numeric child names (hence state-dict keys) line up."""


def feed_forward_holder(dim, mult=4, dropout=0.0):
    """attention.py:45-53 -> keys 0.weight, 0.bias, 1.weight, 4.weight."""
    inner = int(mult * (2 / 3) * dim)
    return nn.Sequential(nn.LayerNorm(dim), nn.Linear(dim, inner * 2, bias=False), _NoParams(),
                         nn.Dropout(dropout), nn.Linear(inner, dim, bias=False))


class PEG(nn.Module):
    """attention.py:57-61."""

    def __init__(self, dim, causal=False):
        super().__init__()
        self.causal = causal
        self.dsconv = nn.Conv3d(dim, dim, 3, groups=dim)


def alibi_slopes(heads):
    """attention.py:201-212 (geometric slopes, closest-power-of-two interleave for odd head counts)."""

    def pow2(n):
        start = 2 ** (-2 ** -(math.log2(n) - 3))
        return [start * start ** i for i in range(n)]

    if math.log2(heads).is_integer():
        return pow2(heads)
    c = 2 ** math.floor(math.log2(heads))
    return pow2(c) + pow2(2 * c)[0::2][: heads - c]


class Attention(nn.Module):
    """attention.py:89-126 (parameters only)."""

    def __init__(self, dim, dim_context=None, dim_head=64, heads=8, causal=False, num_null_kv=0,
                 norm_context=True, dropout=0.0, scale=8):
        super().__init__()
        assert scale == 8, "the kernels implement the reference's fixed scale of 8"
        self.heads, self.dim_head, self.causal, self.scale = heads, dim_head, causal, scale
        inner = dim_head * heads
        dim_context = dim if dim_context is None else dim_context
        self.dim_context = dim_context
        self.norm = LayerNorm(dim)
        self.context_norm = LayerNorm(dim_context) if norm_context else nn.Identity()
        self.num_null_kv = num_null_kv
        self.null_kv = nn.Parameter(torch.randn(heads, 2 * num_null_kv, dim_head))
        self.to_q = nn.Linear(dim, inner, bias=False)
        self.to_kv = nn.Linear(dim_context, inner * 2, bias=False)
        self.q_scale = nn.Parameter(torch.ones(dim_head))
        self.k_scale = nn.Parameter(torch.ones(dim_head))
        self.to_out = nn.Linear(inner, dim, bias=False)


class ContinuousPositionBias(nn.Module):
    """attention.py:229-255 (parameters only; default two hidden layers)."""

    def __init__(self, *, dim, heads, num_dims=2, layers=2, log_dist=True, cache_rel_pos=False):
        super().__init__()
        assert layers == 2 and log_dist, "kernels implement the reference defaults (2 hidden layers, log distance)"
        self.num_dims, self.dim, self.heads = num_dims, dim, heads
        self.net = nn.ModuleList([])
        self.net.append(nn.Sequential(nn.Linear(num_dims, dim), nn.LeakyReLU(0.1)))
        self.net.append(nn.Sequential(nn.Linear(dim, dim), nn.LeakyReLU(0.1)))
        self.net.append(nn.Linear(dim, heads))


class Transformer(nn.Module):
    """attention.py:279-308 (parameters only): layers.{i} = [PEG|None, self-attn, cross|None, FF]."""

    def __init__(self, dim, *, depth, dim_context=None, causal=False, dim_head=64, heads=8, ff_mult=4,
                 peg=False, peg_causal=False, attn_num_null_kv=2, has_cross_attn=False, attn_dropout=0.0,
                 ff_dropout=0.0):
        super().__init__()
        self.dim, self.depth, self.causal, self.dim_head, self.heads = dim, depth, causal, dim_head, heads
        self.attn_dropout, self.ff_dropout = attn_dropout, ff_dropout  # inference ignores them; the training step refuses > 0
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                PEG(dim=dim, causal=peg_causal) if peg else None,
                Attention(dim=dim, dim_head=dim_head, heads=heads, causal=causal, dropout=attn_dropout),
                Attention(dim=dim, dim_head=dim_head, dim_context=dim_context, heads=heads, causal=False,
                          num_null_kv=attn_num_null_kv, dropout=attn_dropout) if has_cross_attn else None,
                feed_forward_holder(dim=dim, mult=ff_mult, dropout=ff_dropout)]))
        self.norm_out = LayerNorm(dim)


# ------------------------------------------------------------------------------------------------
# ctypes weight tables
# ------------------------------------------------------------------------------------------------


class Keep:
    """Owns everything a table points to (packed tensors, ctypes arrays) for the table's lifetime."""

    def __init__(self):
        self.refs = []

    def t(self, tensor):
        if not tensor.is_cuda:
            raise L.PhkError("module parameters must be on a CUDA device (no CPU path): call .cuda() first")
        tensor = tensor.detach()
        if tensor.dtype != torch.float32 or not tensor.is_contiguous():
            tensor = tensor.float().contiguous()
        self.refs.append(tensor)
        return tensor.data_ptr()

    def obj(self, o):
        self.refs.append(o)
        return o

    def h(self, tensor):
        """bf16 copy (the wgmma GEMM operand); leading dimension must be a multiple of 8 for TMA."""
        if not tensor.is_cuda:
            raise L.PhkError("module parameters must be on a CUDA device (no CPU path): call .cuda() first")
        t = tensor.detach().to(torch.bfloat16).contiguous()
        assert t.shape[-1] % 8 == 0, "bf16 mode needs every GEMM K dimension to be a multiple of 8"
        self.refs.append(t)
        return t.data_ptr()

    def h3(self, tensor):
        """[hi | lo | hi] split-bf16 pack of a weight (PHK_PREC_BF16X3)."""
        if not tensor.is_cuda:
            raise L.PhkError("module parameters must be on a CUDA device (no CPU path): call .cuda() first")
        t = split3_weight(tensor)
        self.refs.append(t)
        return t.data_ptr()

    def w16(self, tensor, mode):
        """Tensor-core copy of a weight for precision mode `mode` (None in parity mode)."""
        return self.h(tensor) if mode == L.PREC_BF16 else self.h3(tensor) if mode == L.PREC_BF16X3 else None


def split3_weight(w):
    """PHK_PREC_BF16X3 weight pack: [N, K] fp32 -> bf16 [N, 3 * Kp] = [hi | lo | hi] with hi = bf16(w), lo = bf16(w - hi),
    Kp = K rounded up to 8 (zero padding); the activation side is split [hi | hi | lo] by phk_split3, so ONE bf16 GEMM over
    K' = 3 Kp computes a_hi w_hi + a_hi w_lo + a_lo w_hi (include/phk.h)."""
    w = w.detach().float()
    n, k = w.shape
    kp = (k + 7) // 8 * 8
    hi = w.to(torch.bfloat16)
    lo = (w - hi.float()).to(torch.bfloat16)
    out = torch.zeros((n, 3 * kp), dtype=torch.bfloat16, device=w.device)
    out[:, :k], out[:, kp:kp + k], out[:, 2 * kp:2 * kp + k] = hi, lo, hi
    return out


def pack_geglu_w1(w1, inner, inner_pad):
    """[2*inner, dim] -> [2*inner_pad, dim] bf16 with rows grouped as [64 value rows | 64 gate rows] per
    128-row tile, so the GEMM epilogue can apply gelu(gate) * value inside one accumulator tile
    (attention.py:40-43: value = first half, gate = second half).  Padding rows are zero."""
    dim = w1.shape[1]
    w = w1.detach().to(torch.bfloat16)
    val = torch.zeros((inner_pad, dim), dtype=torch.bfloat16, device=w.device)
    gate = torch.zeros_like(val)
    val[:inner], gate[:inner] = w[:inner], w[inner:]
    g = inner_pad // 64
    return torch.stack((val.reshape(g, 64, dim), gate.reshape(g, 64, dim)), dim=1).reshape(2 * inner_pad, dim).contiguous()


def pack_w2(w2, inner, inner_pad):
    """[dim, inner] -> [dim, inner_pad] bf16, zero-padded K."""
    out = torch.zeros((w2.shape[0], inner_pad), dtype=torch.bfloat16, device=w2.device)
    out[:, :inner] = w2.detach().to(torch.bfloat16)
    return out


def attn_table(a: Attention, keep: Keep, mode=0):
    """mode: L.PREC_* -- which tensor-core weight copies (`*_h`) the table carries (bool accepted: True = PREC_BF16)."""
    t = L.AttnT()
    mode = int(mode)
    if mode:
        t.wq_h, t.wkv_h, t.wo_h = keep.w16(a.to_q.weight, mode), keep.w16(a.to_kv.weight, mode), keep.w16(a.to_out.weight, mode)
    t.norm_g, t.norm_b = keep.t(a.norm.gamma), keep.t(a.norm.beta)
    if isinstance(a.context_norm, LayerNorm):
        t.ctx_g, t.ctx_b = keep.t(a.context_norm.gamma), keep.t(a.context_norm.beta)
    t.null_kv = keep.t(a.null_kv) if a.num_null_kv > 0 else None
    t.q_scale, t.k_scale = keep.t(a.q_scale), keep.t(a.k_scale)
    t.wq, t.wkv, t.wo = keep.t(a.to_q.weight), keep.t(a.to_kv.weight), keep.t(a.to_out.weight)
    t.num_null_kv, t.dim_context = a.num_null_kv, a.dim_context
    return t


def transformer_table(tf: Transformer, keep: Keep, mode=0):
    mode = int(mode)
    bf16 = mode == L.PREC_BF16
    layers = (L.LayerT * tf.depth)()
    for i, (peg, self_attn, cross, ff) in enumerate(tf.layers):
        ly = layers[i]
        ly.has_peg, ly.has_cross = int(peg is not None), int(cross is not None)
        if peg is not None:
            d = peg.dsconv.weight.shape[0]
            w = peg.dsconv.weight.detach().reshape(d, 27).t().contiguous()  # tap-major [27, dim]
            ly.peg.w, ly.peg.b, ly.peg.causal = keep.t(w), keep.t(peg.dsconv.bias), int(peg.causal)
        ly.self_attn = attn_table(self_attn, keep, mode)
        if cross is not None:
            ly.cross_attn = attn_table(cross, keep, mode)
        ly.ff.ln_g, ly.ff.ln_b = keep.t(ff[0].weight), keep.t(ff[0].bias)
        ly.ff.w1, ly.ff.w2 = keep.t(ff[1].weight), keep.t(ff[4].weight)
        ly.ff.inner = ff[4].weight.shape[1]
        ly.ff.inner_pad = (ly.ff.inner + 63) // 64 * 64
        if bf16:
            w1h = pack_geglu_w1(ff[1].weight, ly.ff.inner, ly.ff.inner_pad)
            w2h = pack_w2(ff[4].weight, ly.ff.inner, ly.ff.inner_pad)
            keep.refs += [w1h, w2h]
            ly.ff.w1_h, ly.ff.w2_h = w1h.data_ptr(), w2h.data_ptr()
        elif mode == L.PREC_BF16X3:  # plain row order (GEGLU stays a separate fp32 kernel), split operands
            ly.ff.w1_h, ly.ff.w2_h = keep.h3(ff[1].weight), keep.h3(ff[4].weight)
    keep.obj(layers)
    t = L.TransformerT()
    t.dim, t.heads, t.dim_head, t.depth, t.causal = tf.dim, tf.heads, tf.dim_head, tf.depth, int(tf.causal)
    t.layers = C.cast(layers, C.POINTER(L.LayerT))
    t.out_g, t.out_b = keep.t(tf.norm_out.gamma), keep.t(tf.norm_out.beta)
    if tf.causal:
        dev = tf.norm_out.gamma.device
        t.alibi_slopes = keep.t(torch.tensor(alibi_slopes(tf.heads), dtype=torch.float32, device=dev))
    return t


def cpb_table(c: ContinuousPositionBias, keep: Keep):
    t = L.CpbT()
    t.w0, t.b0 = keep.t(c.net[0][0].weight), keep.t(c.net[0][0].bias)
    t.w1, t.b1 = keep.t(c.net[1][0].weight), keep.t(c.net[1][0].bias)
    t.w2, t.b2 = keep.t(c.net[2].weight), keep.t(c.net[2].bias)
    t.num_dims, t.hidden, t.heads = c.num_dims, c.dim, c.heads
    return t


class GradKeep:
    """Gradient twin of ``Keep`` for phk_maskgit_train_step: hands out pointers into zero-filled gradient buffers of
    the parameters' shapes and remembers which parameters were given one (the reference leaves ``p.grad = None`` for
    the rest, e.g. the self-attention ``context_norm``)."""

    def __init__(self, params):
        """params: iterable of nn.Parameter, all on one CUDA device.  One flat fp32 buffer, one view per parameter
        in iteration order (a single contiguous bucket for a data-parallel gradient all-reduce); every view starts on
        a 256-byte boundary so that the tensor-core wgrad can write it through the TMA epilogue."""
        self.params = list(params)
        dev = self.params[0].device
        offsets, off = [], 0
        for p in self.params:
            offsets.append(off)
            off += (p.numel() + 63) // 64 * 64
        self.flat = torch.zeros(off, dtype=torch.float32, device=dev)
        self.views = {p: self.flat[o:o + p.numel()].view(p.shape) for p, o in zip(self.params, offsets)}
        self.used, self.refs = set(), []

    def g(self, param):
        self.used.add(param)
        return self.views[param].data_ptr()

    def obj(self, o):
        self.refs.append(o)
        return o

    def grad_of(self, param):
        return self.views[param] if param in self.used else None


def attn_grad_table(a: Attention, gk: GradKeep, cross: bool):
    t = L.AttnT()
    t.norm_g = gk.g(a.norm.gamma)
    if cross and isinstance(a.context_norm, LayerNorm):
        t.ctx_g = gk.g(a.context_norm.gamma)
    t.null_kv = gk.g(a.null_kv) if a.num_null_kv > 0 else None
    gk.used.add(a.null_kv)  # autograd hands an (empty) gradient to a (heads, 0, dim_head) parameter too
    t.q_scale, t.k_scale = gk.g(a.q_scale), gk.g(a.k_scale)
    t.wq, t.wkv, t.wo = gk.g(a.to_q.weight), gk.g(a.to_kv.weight), gk.g(a.to_out.weight)
    t.num_null_kv, t.dim_context = a.num_null_kv, a.dim_context
    return t


def transformer_grad_table(tf: Transformer, gk: GradKeep, with_cross: bool):
    """Same layout as ``transformer_table`` with every float pointer addressing the parameter's gradient buffer."""
    layers = (L.LayerT * tf.depth)()
    for i, (peg, self_attn, cross, ff) in enumerate(tf.layers):
        ly = layers[i]
        ly.has_peg, ly.has_cross = int(peg is not None), int(cross is not None)
        if peg is not None:
            # gradient in the parameter's own [D, 1, 3, 3, 3] = [D, 27] layout (the WEIGHT table is tap-major [27, D])
            ly.peg.w, ly.peg.b, ly.peg.causal = gk.g(peg.dsconv.weight), gk.g(peg.dsconv.bias), int(peg.causal)
        ly.self_attn = attn_grad_table(self_attn, gk, cross=False)
        if cross is not None and with_cross:
            ly.cross_attn = attn_grad_table(cross, gk, cross=True)
        ly.ff.ln_g, ly.ff.ln_b = gk.g(ff[0].weight), gk.g(ff[0].bias)
        ly.ff.w1, ly.ff.w2 = gk.g(ff[1].weight), gk.g(ff[4].weight)
        ly.ff.inner = ff[4].weight.shape[1]
        ly.ff.inner_pad = (ly.ff.inner + 63) // 64 * 64
    gk.obj(layers)
    t = L.TransformerT()
    t.dim, t.heads, t.dim_head, t.depth, t.causal = tf.dim, tf.heads, tf.dim_head, tf.depth, int(tf.causal)
    t.layers = C.cast(layers, C.POINTER(L.LayerT))
    t.out_g = gk.g(tf.norm_out.gamma)
    return t


def cpb_grad_table(c: ContinuousPositionBias, gk: GradKeep):
    t = L.CpbT()
    t.w0, t.b0 = gk.g(c.net[0][0].weight), gk.g(c.net[0][0].bias)
    t.w1, t.b1 = gk.g(c.net[1][0].weight), gk.g(c.net[1][0].bias)
    t.w2, t.b2 = gk.g(c.net[2].weight), gk.g(c.net[2].bias)
    t.num_dims, t.hidden, t.heads = c.num_dims, c.dim, c.heads
    return t


_SIG_REFRESH = 64


def weights_signature(module):
    """Changes whenever a parameter / buffer is moved, modified in place or REPLACED (`.to()`, `load_state_dict`,
    optimizer steps, `mod.weight = nn.Parameter(...)`): the tuple of (data_ptr, _version) of every tensor, read live
    from the `_parameters` / `_buffers` dicts of the submodules on every call.  Only the LIST OF SUBMODULES is cached
    (walking the module tree is the expensive part, ~0.25 ms for a C-ViViT) and re-walked every 64 calls, which picks up
    a replaced submodule.  Not visible from here: writes through `.data` (`p.data.copy_()`, `p.data.lerp_()` do not
    bump `_version`) into tensors with derived copies (bf16 weights, packed GEGLU / PEG weights, cached position-bias
    tables) -- call `invalidate_weights(module)` after such an update."""
    cache = module.__dict__.get("_phk_sig_cache")
    if cache is None or cache[1] <= 0:
        cache = [[(m._parameters, m._buffers) for m in module.modules()], _SIG_REFRESH]
        module.__dict__["_phk_sig_cache"] = cache
    cache[1] -= 1
    sig = []
    for params, bufs in cache[0]:
        for t in params.values():
            if t is not None:
                sig.append((t.data_ptr(), t._version))
        for t in bufs.values():
            if t is not None:
                sig.append((t.data_ptr(), t._version))
    return tuple(sig)


def invalidate_weights(module):
    """Forces the weight tables (and every derived copy) of `module` and its submodules to be rebuilt at the next call:
    for updates the signature cannot see (`p.data.copy_()` style writes, e.g. hand-written EMA)."""
    for m in module.modules():
        m.__dict__.pop("_phk_sig_cache", None)
        for name in ("_sig", "_dec_sig"):
            if name in m.__dict__:
                m.__dict__[name] = None


class Workspace:
    """One grow-only device scratch buffer per module (the C library allocates nothing)."""

    def __init__(self):
        self.buf = None

    def get(self, nbytes, device):
        if self.buf is None or self.buf.numel() < nbytes or self.buf.device != device:
            self.buf = torch.empty(int(nbytes), dtype=torch.uint8, device=device)
        return self.buf
