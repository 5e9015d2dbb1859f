"""C-ViViT video tokenizer -- drop-in for ``phenaki_pytorch.CViViT`` on the encode hot path.

Same constructor keywords, attribute names and state-dict layout as the reference
(/root/reference/phenaki_pytorch/cvivit.py:226-335); ``forward(video,
return_only_codebook_ids=True)`` (cvivit.py:518-574) runs entirely in libphk.so
(phk_cvivit_encode).  Training losses, discriminator and VGG (cvivit.py:59-213, 576-671) are out
of scope (SURVEY.md section 2, rows 8/10) and raise.
"""
import copy
import ctypes as C
import math
from pathlib import Path

import torch
from torch import nn

from . import _lib as L
from .modules import (ContinuousPositionBias, Keep, Transformer, Workspace, _NoParams, cpb_table,
                      transformer_table, weights_signature)


def _pair(v):
    r = (v, v) if not isinstance(v, tuple) else v
    assert len(r) == 2
    return r


class LFQ(nn.Module):
    """Parameter holder with upstream ``vector_quantize_pytorch.LFQ`` state-dict names
    (``mask``, ``project_in.*``, ``project_out.*``); arithmetic restated in oracle/lfq.py, executed by
    phk_lfq_ids."""

    def __init__(self, *, dim, codebook_size, **kwargs):
        super().__init__()
        bits = int(math.log2(codebook_size))
        assert 2 ** bits == codebook_size, "codebook size must be a power of two"
        assert dim != bits, "LFQ without projections is not supported"
        self.codebook_dim, self.codebook_size = bits, codebook_size
        self.project_in = nn.Linear(dim, bits)
        self.project_out = nn.Linear(bits, dim)
        self.register_buffer("mask", 2 ** torch.arange(bits - 1, -1, -1))


class _CosineSimCodebook(nn.Module):
    """Buffers of upstream ``CosineSimCodebook`` (one codebook, no k-means init): unit-norm kaiming-uniform rows."""

    def __init__(self, dim, codebook_size):
        super().__init__()
        embed = torch.empty(1, codebook_size, dim)
        nn.init.kaiming_uniform_(embed)
        embed = torch.nn.functional.normalize(embed, dim=-1)
        self.register_buffer("initted", torch.Tensor([True]))
        self.register_buffer("cluster_size", torch.zeros(1, codebook_size))
        self.register_buffer("embed_avg", embed.clone())
        self.register_buffer("embed", embed)


class VectorQuantize(nn.Module):
    """Buffer holder with upstream ``vector_quantize_pytorch.VectorQuantize(use_cosine_sim=True)`` state-dict names
    (``_codebook.{initted, cluster_size, embed_avg, embed}``) for ``lookup_free_quantization=False`` (cvivit.py:321);
    arithmetic restated in oracle/lfq.py, executed by phk_vq_cosine_ids."""

    def __init__(self, *, dim, codebook_size, use_cosine_sim=True, **kwargs):
        super().__init__()
        assert use_cosine_sim
        self.dim, self.codebook_size = dim, codebook_size
        self._codebook = _CosineSimCodebook(dim, codebook_size)

    @property
    def codebook(self):
        return self._codebook.embed[0]


class CViViT(nn.Module):
    def __init__(self, *, dim, codebook_size, image_size, patch_size, temporal_patch_size, spatial_depth,
                 temporal_depth, discr_base_dim=16, dim_head=64, heads=8, channels=3, use_vgg_and_gan=True,
                 vgg=None, discr_attn_res_layers=(16,), use_hinge_loss=True, attn_dropout=0.0, ff_dropout=0.0,
                 lookup_free_quantization=True, lookup_free_quantization_kwargs: dict = {}):
        super().__init__()
        self.image_size = _pair(image_size)
        self.patch_size = _pair(patch_size)
        ph, pw = self.patch_size
        self.temporal_patch_size = temporal_patch_size
        self.dim, self.heads, self.dim_head, self.channels = dim, heads, dim_head, channels
        # construction order below follows the reference so seeded inits coincide
        self.spatial_rel_pos_bias = ContinuousPositionBias(dim=dim, heads=heads)
        ih, iw = self.image_size
        assert (ih % ph) == 0 and (iw % pw) == 0
        k1 = channels * pw * ph
        self.to_patch_emb_first_frame = nn.Sequential(_NoParams(), nn.LayerNorm(k1), nn.Linear(k1, dim),
                                                      nn.LayerNorm(dim))
        k2 = k1 * temporal_patch_size
        self.to_patch_emb = nn.Sequential(_NoParams(), nn.LayerNorm(k2), nn.Linear(k2, dim), nn.LayerNorm(dim))
        spatial_kw = dict(dim=dim, dim_head=dim_head, heads=heads, attn_dropout=attn_dropout,
                          ff_dropout=ff_dropout, causal=False, peg=False)
        temporal_kw = dict(dim=dim, dim_head=dim_head, heads=heads, attn_dropout=attn_dropout,
                           ff_dropout=ff_dropout, causal=True, peg=True, peg_causal=True)
        self.enc_spatial_transformer = Transformer(depth=spatial_depth, **spatial_kw)
        self.enc_temporal_transformer = Transformer(depth=temporal_depth, **temporal_kw)
        self.lookup_free_quantization = lookup_free_quantization
        if lookup_free_quantization:
            self.vq = LFQ(dim=dim, codebook_size=codebook_size, **lookup_free_quantization_kwargs)
        else:
            self.vq = VectorQuantize(dim=dim, codebook_size=codebook_size, use_cosine_sim=True)
        self.dec_spatial_transformer = Transformer(depth=spatial_depth, **spatial_kw)
        self.dec_temporal_transformer = Transformer(depth=temporal_depth, **temporal_kw)
        self.to_pixels_first_frame = nn.Sequential(nn.Linear(dim, k1), _NoParams())
        self.to_pixels = nn.Sequential(nn.Linear(dim, k2), _NoParams())
        self.vgg = None
        self.discr = None
        # the reference's default (use_vgg_and_gan=True, cvivit.py:345-363) builds a VGG16 and a Discriminator that only
        # the GAN / perceptual TRAINING losses use.  Those losses are out of scope (SURVEY section 2 row 8), so neither is
        # built here: the tokenizer constructs with the reference's defaults, encodes and decodes, and loads the
        # reference's checkpoints (load_state_dict drops their `discr.*` entries); forward() raises for the loss paths.
        self.use_vgg_and_gan = use_vgg_and_gan
        self.precision = L.default_precision()
        self._tables = None
        self._sig = None
        self._dec_tables = None
        self._dec_sig = None
        self._ws = Workspace()
        self._bias_cache = {}
        self._ids_buf = {}

    # ---- shape helpers (cvivit.py:365-410, 445-447) -----------------------------------------
    @property
    def patch_height_width(self):
        return self.image_size[0] // self.patch_size[0], self.image_size[1] // self.patch_size[1]

    @property
    def image_num_tokens(self):
        h, w = self.patch_height_width
        return h * w

    def get_video_patch_shape(self, num_frames, include_first_frame=True):
        patch_frames = 0
        if include_first_frame:
            num_frames -= 1
            patch_frames += 1
        return (patch_frames + num_frames // self.temporal_patch_size, *self.patch_height_width)

    def num_tokens_per_frames(self, num_frames, include_first_frame=True):
        total = 0
        if include_first_frame:
            num_frames -= 1
            total += self.image_num_tokens
        assert (num_frames % self.temporal_patch_size) == 0
        return total + (num_frames // self.temporal_patch_size) * self.image_num_tokens

    def frames_per_num_tokens(self, num_tokens):
        per = self.image_num_tokens
        assert (num_tokens % per) == 0 and num_tokens > 0
        return (num_tokens // per - 1) * self.temporal_patch_size + 1

    def calculate_video_token_mask(self, videos, video_frame_mask):
        *_, h, w = videos.shape
        ph, pw = self.patch_size
        pt = self.temporal_patch_size
        assert torch.all(((video_frame_mask.sum(dim=-1) - 1) % pt) == 0), \
            "number of frames must be divisible by temporal patch size, subtracting off the first frame"
        first, rest = video_frame_mask[:, :1], video_frame_mask[:, 1:]
        rest = rest.reshape(rest.shape[0], -1, pt).any(dim=-1)
        m = torch.cat((first, rest), dim=-1)
        return m.repeat_interleave((h // ph) * (w // pw), dim=-1)

    def copy_for_eval(self):
        device = next(self.parameters()).device
        saved = (self._tables, self._sig, self._dec_tables, self._dec_sig, self._ws, self._bias_cache, self._ids_buf)
        self._tables, self._sig, self._dec_tables, self._dec_sig = None, None, None, None  # ctypes tables are not copyable
        self._ws, self._bias_cache, self._ids_buf = Workspace(), {}, {}
        c = copy.deepcopy(self)
        self._tables, self._sig, self._dec_tables, self._dec_sig, self._ws, self._bias_cache, self._ids_buf = saved
        return c.eval().to(device)

    def load_state_dict(self, state_dict, *args, **kwargs):
        """Reference checkpoints of a tokenizer trained with use_vgg_and_gan=True carry the discriminator
        (`discr.*`; the VGG is already hidden by the reference's remove_vgg, cvivit.py:35-49): those entries belong
        to the training losses this module does not build and are dropped; everything else loads as given."""
        kept = {k: v for k, v in state_dict.items() if not (k.startswith("discr.") or k.startswith("vgg."))}
        return super().load_state_dict(kept, *args, **kwargs)

    def load(self, path):
        path = Path(path)
        assert path.exists()
        self.load_state_dict(torch.load(str(path)))

    # ---- libphk plumbing ---------------------------------------------------------------------
    def _table(self):
        sig = (weights_signature(self), self.precision)
        if self._tables is None or sig != self._sig:
            keep = Keep()
            h16 = self.precision == L.PREC_BF16
            mode = self.precision  # which tensor-core weight copies the table carries (none in parity mode)
            t = L.CvivitT()
            t.dim, t.heads, t.dim_head, t.channels = self.dim, self.heads, self.dim_head, self.channels
            t.image_h, t.image_w = self.image_size
            t.patch_h, t.patch_w = self.patch_size
            t.patch_t = self.temporal_patch_size
            t.codebook_bits = self.vq.codebook_dim if self.lookup_free_quantization else 0
            f, r = self.to_patch_emb_first_frame, self.to_patch_emb
            t.pf_ln1_g, t.pf_ln1_b, t.pf_w, t.pf_b = keep.t(f[1].weight), keep.t(f[1].bias), keep.t(f[2].weight), keep.t(f[2].bias)
            t.pf_ln2_g, t.pf_ln2_b = keep.t(f[3].weight), keep.t(f[3].bias)
            t.pr_ln1_g, t.pr_ln1_b, t.pr_w, t.pr_b = keep.t(r[1].weight), keep.t(r[1].bias), keep.t(r[2].weight), keep.t(r[2].bias)
            t.pr_ln2_g, t.pr_ln2_b = keep.t(r[3].weight), keep.t(r[3].bias)
            t.spatial_bias = cpb_table(self.spatial_rel_pos_bias, keep)
            t.spatial = transformer_table(self.enc_spatial_transformer, keep, mode)
            t.temporal = transformer_table(self.enc_temporal_transformer, keep, mode)
            if mode:
                t.pf_w_h, t.pr_w_h = keep.w16(f[2].weight, mode), keep.w16(r[2].weight, mode)
            if self.lookup_free_quantization:
                t.vq_w, t.vq_b = keep.t(self.vq.project_in.weight), keep.t(self.vq.project_in.bias)
            else:  # cosine-sim codebook (unit rows)
                t.codebook, t.codebook_size = keep.t(self.vq.codebook), self.vq.codebook_size
                if h16:
                    t.codebook_h = keep.h(self.vq.codebook)
            self._tables, self._sig = (t, keep), sig
            self._bias_cache = {}
        return self._tables[0]

    def _dec_table(self):
        sig = (weights_signature(self), self.precision)
        if self._dec_tables is None or sig != self._dec_sig:
            keep = Keep()
            mode = self.precision
            t = L.CvivitDecT()
            t.dim, t.heads, t.dim_head, t.channels = self.dim, self.heads, self.dim_head, self.channels
            t.image_h, t.image_w = self.image_size
            t.patch_h, t.patch_w = self.patch_size
            t.patch_t = self.temporal_patch_size
            if self.lookup_free_quantization:
                t.codebook_bits = self.vq.codebook_dim
                t.vq_out_w, t.vq_out_b = keep.t(self.vq.project_out.weight), keep.t(self.vq.project_out.bias)
            # (cosine-sim codebook: decode_from_codebook_indices gathers the codes and decodes float tokens)
            t.spatial_bias = cpb_table(self.spatial_rel_pos_bias, keep)
            t.temporal = transformer_table(self.dec_temporal_transformer, keep, mode)
            t.spatial = transformer_table(self.dec_spatial_transformer, keep, mode)
            f, r = self.to_pixels_first_frame[0], self.to_pixels[0]
            t.px_first_w, t.px_first_b = keep.t(f.weight), keep.t(f.bias)
            t.px_w, t.px_b = keep.t(r.weight), keep.t(r.bias)
            if mode:
                t.px_first_w_h, t.px_w_h = keep.w16(f.weight, mode), keep.w16(r.weight, mode)
            self._dec_tables, self._dec_sig = (t, keep), sig
        return self._dec_tables[0]

    def _spatial_bias(self, table, device):
        """ContinuousPositionBias is a function of the weights only: computed once per weight version."""
        h, w = self.patch_height_width
        key = (h, w, device)
        if key not in self._bias_cache:
            lib = L.lib()
            n = h * w
            out = torch.empty((self.heads, n, n), dtype=torch.float32, device=device)
            scratch = torch.empty(int(lib.phk_cpb_scratch_floats(C.byref(table.spatial_bias), h, w, 1)),
                                  dtype=torch.float32, device=device)
            L.check(lib.phk_cpb_bias(C.byref(table.spatial_bias), h, w, 1, L.ptr(scratch), L.ptr(out),
                                     L.stream_ptr()), "phk_cpb_bias")
            self._bias_cache[key] = out
        return self._bias_cache[key]

    def encode_ids(self, video, taps=None):
        """video (b,c,f,H,W) fp32 CUDA -> ids (b,T',H',W') int64.  ``taps``: optional dict that receives the
        intermediate activations (parity tests)."""
        lib = L.lib()
        video = L.require_cuda(video, "video", torch.float32)
        b, c, f, *image_dims = video.shape
        assert tuple(image_dims) == self.image_size
        assert c == self.channels
        assert (f - 1) % self.temporal_patch_size == 0, \
            f"number of frames ({f}) minus one ({f - 1}) must be divisible by temporal patch size ({self.temporal_patch_size})"
        with torch.cuda.device(video.device):
            table = self._table()
            tp, hh, ww = self.get_video_patch_shape(f)
            # the kernels write into a module-owned buffer with a STABLE address (the library replays a captured CUDA
            # graph when every pointer of the call repeats); the caller gets its own copy, as in the reference
            key = (b, tp, hh, ww, video.device)
            ids = self._ids_buf.get(key)
            if ids is None:
                ids = self._ids_buf[key] = torch.empty((b, tp, hh, ww), dtype=torch.int64, device=video.device)
            nbytes = lib.phk_cvivit_workspace_bytes(C.byref(table), b, f, self.precision)
            ws = self._ws.get(nbytes, video.device)
            bias = self._spatial_bias(table, video.device)
            tap_ptrs = [None] * 4
            if taps is not None:
                rows = b * tp * hh * ww
                taps["patch"] = torch.empty((b, tp, hh, ww, self.dim), dtype=torch.float32, device=video.device)
                taps["spatial"] = torch.empty_like(taps["patch"])
                taps["temporal"] = torch.empty_like(taps["patch"])
                if self.lookup_free_quantization:
                    taps["proj"] = torch.empty((rows, self.vq.codebook_dim), dtype=torch.float32, device=video.device)
                tap_ptrs = [L.ptr(taps.get(k)) for k in ("patch", "spatial", "temporal", "proj")]
            L.check(lib.phk_cvivit_encode(C.byref(table), L.ptr(video), b, f, L.ptr(ids), L.ptr(ws), ws.numel(),
                                          self.precision, L.ptr(bias), *tap_ptrs, L.stream_ptr()),
                    "phk_cvivit_encode")
            return ids.clone()

    def encode_host_iter(self, videos, device=None, depth=2):
        """Tokenises a stream of HOST batches: `videos` yields (b,c,f,H,W) fp32 CPU tensors of one shape (pinned memory
        gives the full PCIe rate); yields the (b,T',H',W') int64 ids of each batch as CPU tensors, in order.  The H2D
        copy of batch i+1 overlaps the encode of batch i (phk_encode_pipe_*); nothing is staged by torch."""
        lib = L.lib()
        device = torch.device(device) if device is not None else next(self.parameters()).device
        assert device.type == "cuda", "this framework has no CPU path"
        pipe = C.c_void_p()
        L.check(lib.phk_encode_pipe_create(C.byref(pipe), depth), "phk_encode_pipe_create")
        shape, inflight, submitted = None, [], 0
        try:
            with torch.cuda.device(device):
                table = self._table()
                bias = self._spatial_bias(table, device)

                def retire():
                    ticket, host_ids, _keep = inflight.pop(0)
                    L.check(lib.phk_encode_pipe_wait(pipe, ticket), "phk_encode_pipe_wait")
                    return host_ids

                for video in videos:
                    if video.is_cuda or video.dtype != torch.float32:
                        raise L.PhkError("encode_host_iter takes fp32 CPU batches (use forward() for device tensors)")
                    video = video.contiguous()
                    if shape is None:
                        shape = tuple(video.shape)
                        b, c, f, *image_dims = shape
                        assert tuple(image_dims) == self.image_size and c == self.channels
                        assert (f - 1) % self.temporal_patch_size == 0
                        tp, hh, ww = self.get_video_patch_shape(f)
                        stage = torch.empty((depth, *shape), dtype=torch.float32, device=device)
                        dev_ids = torch.empty((depth, b, tp, hh, ww), dtype=torch.int64, device=device)
                        host = [torch.empty((b, tp, hh, ww), dtype=torch.int64).pin_memory() for _ in range(depth)]
                        nbytes = lib.phk_cvivit_workspace_bytes(C.byref(table), b, f, self.precision)
                        ws = self._ws.get(nbytes, device)
                    assert tuple(video.shape) == shape, "all batches of one stream must have the same shape"
                    if len(inflight) == depth:
                        yield retire().clone()
                    ticket = C.c_int64()
                    slot_host = host[submitted % depth]
                    L.check(lib.phk_encode_pipe_submit(pipe, C.byref(table), L.ptr(video), b, f, L.ptr(slot_host),
                                                       L.ptr(stage), L.ptr(dev_ids), L.ptr(ws), ws.numel(),
                                                       self.precision, L.ptr(bias), L.stream_ptr(), C.byref(ticket)),
                            "phk_encode_pipe_submit")
                    assert ticket.value == submitted
                    submitted += 1
                    inflight.append((ticket.value, slot_host, video))
                while inflight:
                    yield retire().clone()
        finally:
            torch.cuda.synchronize(device)
            lib.phk_encode_pipe_destroy(pipe)

    def encode_host(self, video, device=None):
        """One host batch -> host ids (H2D, encode, D2H, synchronise)."""
        return next(self.encode_host_iter([video], device=device, depth=1))

    def forward(self, video, mask=None, return_recons=False, return_recons_only=False, return_discr_loss=False,
                apply_grad_penalty=True, return_only_codebook_ids=False):
        assert video.ndim in {4, 5}
        is_image = video.ndim == 4
        if is_image:
            video = video.unsqueeze(2)  # 'b c h w -> b c 1 h w'
            assert mask is None
        assert mask is None or mask.shape[-1] == video.shape[2]
        if return_only_codebook_ids:
            return self.encode_ids(video)
        if return_recons_only:
            # decode(project_out(sign(project_in(tokens)))) = decode(indices_to_codes(ids))  (cvivit.py:570-581)
            recon = self.decode_from_codebook_indices(self.encode_ids(video))
            return recon.squeeze(2) if is_image else recon
        raise NotImplementedError("C-ViViT training losses (reconstruction / GAN / perceptual, cvivit.py:576-671) "
                                  "are out of scope of the H100 hot path (SURVEY.md section 2 row 8)")

    def _decode(self, ids, tokens, b, tp, device, taps=None):
        lib = L.lib()
        with torch.cuda.device(device):
            enc = self._table()  # the position-bias cache is keyed on the encoder table's weight version
            table = self._dec_table()
            f = 1 + (tp - 1) * self.temporal_patch_size
            video = torch.empty((b, self.channels, f, *self.image_size), dtype=torch.float32, device=device)
            nbytes = lib.phk_cvivit_decode_workspace_bytes(C.byref(table), b, tp, self.precision)
            ws = self._ws.get(nbytes, device)
            bias = self._spatial_bias(enc, device)
            tap_ptrs = [None] * 3
            if taps is not None:
                h, w = self.patch_height_width
                for k in ("codes", "temporal", "spatial"):
                    taps[k] = torch.empty((b, tp, h, w, self.dim), dtype=torch.float32, device=device)
                tap_ptrs = [L.ptr(taps[k]) for k in ("codes", "temporal", "spatial")]
            L.check(lib.phk_cvivit_decode(C.byref(table), L.ptr(ids), L.ptr(tokens), b, tp, L.ptr(video), L.ptr(ws),
                                          ws.numel(), self.precision, L.ptr(bias), *tap_ptrs, L.stream_ptr()),
                    "phk_cvivit_decode")
        return video

    def decode_from_codebook_indices(self, indices, taps=None):
        """ids (b, n) or (b, t, h, w) int64 CUDA -> video (b, c, f, H, W) fp32 (cvivit.py:437-443): LFQ
        indices_to_codes, decoder transformers and to_pixels, all inside phk_cvivit_decode."""
        indices = L.require_cuda(indices, "indices", torch.int64)
        b = indices.shape[0]
        n = indices[0].numel()
        per = self.image_num_tokens
        assert n > 0 and n % per == 0, f"number of tokens ({n}) must be a multiple of tokens per frame ({per})"
        if not self.lookup_free_quantization:
            # codes = vq.codebook[indices] (cvivit.py:441): a row gather (data movement), then decode of float tokens
            codes = self.vq.codebook.index_select(0, indices.reshape(-1)).reshape(b, n, self.dim).contiguous()
            return self._decode(None, codes, b, n // per, indices.device, taps)
        return self._decode(indices.reshape(b, n), None, b, n // per, indices.device, taps)

    def decode(self, tokens):
        """tokens (b, t, h, w, d) or (b, (t h w), d) fp32 CUDA -> video (cvivit.py:476-516)."""
        tokens = L.require_cuda(tokens, "tokens", torch.float32)
        b, d = tokens.shape[0], tokens.shape[-1]
        assert d == self.dim
        n = tokens[0].numel() // d
        per = self.image_num_tokens
        assert n > 0 and n % per == 0
        return self._decode(None, tokens.reshape(b, n, d), b, n // per, tokens.device)
