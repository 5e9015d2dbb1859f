"""TEST INFRASTRUCTURE ONLY (oracle) -- never imported by the product path.

CPU (torch fp32, eager ATen) restatement of the phenaki-pytorch hot path:
C-ViViT encode (patch-embed -> spatial attn -> temporal attn -> LFQ ids) and the
MaskGIT iterative masked sampling loop.  Purely functional: every function
takes the reference ``state_dict`` (plain ``{name: tensor}``) and a key prefix,
so it shares no code or structure with either the reference modules or the
product.  Each function cites the reference file:line it follows
(paths relative to /root/reference/phenaki_pytorch/).  The MaskGit / critic functions compute in
the dtype of the state dict they are given: tests/train_at_size_cases.py runs them in float64.

Pinning: ``tests/golden/make_golden.py`` runs this file against the UNMODIFIED
reference modules imported in the build container (oracle/reference_loader.py)
and asserts bit-identical outputs on CPU before writing the golden fixtures in
``tests/golden/``; ``tests/test_oracle_golden.py`` re-checks the oracle against
those committed fixtures everywhere (no /root/reference needed).
The LFQ step is "parity unpinned" upstream (see oracle/lfq.py).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
reference leg may import this module.
"""
import math

import torch
import torch.nn.functional as F

# --------------------------------------------------------------------------------------
# primitives (attention.py)
# --------------------------------------------------------------------------------------


def layer_norm(x, weight, bias):
    """attention.py:29-36 (gamma / zero beta buffer) and nn.LayerNorm (:48); eps 1e-5."""
    return F.layer_norm(x, x.shape[-1:], weight, bias)


def feed_forward(x, sd, p):
    """attention.py:40-53.  LN(affine) -> Linear(dim, 2*inner) -> x,gate=chunk; gelu(gate)*x -> Linear(inner, dim)."""
    h = layer_norm(x, sd[p + "0.weight"], sd[p + "0.bias"])
    h = F.linear(h, sd[p + "1.weight"])
    val, gate = h.chunk(2, dim=-1)
    h = F.gelu(gate) * val
    return F.linear(h, sd[p + "4.weight"])


def peg(x, shape, sd, p, causal):
    """attention.py:57-85.  NOTE the raw ``reshape`` (:71): a ``(b h w) t d`` buffer is
    *reinterpreted* as (b,t,h,w,d), not rearranged; replicated as is."""
    orig_shape = x.shape
    if x.ndim == 3:
        x = x.reshape(*shape, -1)
    x = x.movedim(-1, 1)  # b d t h w
    frame_pad = (2, 0) if causal else (1, 1)
    x = F.pad(x, (1, 1, 1, 1, *frame_pad), value=0.0)
    w = sd[p + "dsconv.weight"]
    x = F.conv3d(x, w, sd[p + "dsconv.bias"], groups=w.shape[0])
    x = x.movedim(1, -1)
    return x.reshape(orig_shape)


def alibi_slopes(heads):
    """attention.py:201-212."""

    def pow2(n):
        start = 2 ** (-2 ** -(math.log2(n) - 3))
        return [start * start ** i for i in range(n)]

    if math.log2(heads).is_integer():
        return pow2(heads)
    c = 2 ** math.floor(math.log2(heads))
    return pow2(c) + pow2(2 * c)[0::2][: heads - c]


def alibi_bias(heads, i, j, device=None):
    """attention.py:195-227 -> (h, i, j) fp32, ``-|col - row| * slope``."""
    rows = torch.arange(j - i, j, device=device)
    cols = torch.arange(j, device=device)
    bias = -(cols[None, None, :] - rows[None, :, None]).abs()
    slopes = torch.tensor(alibi_slopes(heads), dtype=torch.float32, device=device)[:, None, None]
    return bias * slopes


def attention_core(q, k, v, q_scale, k_scale, *, heads, causal=False, num_null_kv=0, mask=None,
                   attn_bias=None, scale=8):
    """attention.py:153-179 on already split heads: q (b,h,i,d), k/v (b,h,j,d) with the null
    keys/values already prepended.  Returns (b,h,i,d)."""
    q = F.normalize(q, dim=-1) * q_scale
    k = F.normalize(k, dim=-1) * k_scale
    sim = torch.einsum("bhid,bhjd->bhij", q, k) * scale
    i, j = sim.shape[-2:]
    if attn_bias is not None:
        sim = sim + F.pad(attn_bias, (num_null_kv, 0), value=0.0)
    neg = -torch.finfo(sim.dtype).max
    if mask is not None:
        m = F.pad(mask, (num_null_kv, 0), value=True)
        sim = sim.masked_fill(~m[:, None, None, :], neg)
    if causal:
        sim = sim + alibi_bias(heads, i, j, sim.device)
        sim = sim.masked_fill(torch.ones((i, j), dtype=torch.bool, device=sim.device).triu(j - i + 1), neg)
    attn = sim.softmax(dim=-1)
    return torch.einsum("bhij,bhjd->bhid", attn, v)


def attention(x, sd, p, *, heads, causal=False, num_null_kv=0, mask=None, context=None,
              attn_bias=None, scale=8):
    """attention.py:128-182.  Quirk kept: for self-attention k,v are projected from the
    UN-normalised x (``kv_input`` is bound before ``x = self.norm(x)``, :140-142)."""
    b = x.shape[0]
    if context is not None:
        context = layer_norm(context, sd[p + "context_norm.gamma"], sd[p + "context_norm.beta"])
    kv_input = context if context is not None else x
    xn = layer_norm(x, sd[p + "norm.gamma"], sd[p + "norm.beta"])
    q = F.linear(xn, sd[p + "to_q.weight"])
    k, v = F.linear(kv_input, sd[p + "to_kv.weight"]).chunk(2, dim=-1)

    def split(t):
        return t.reshape(t.shape[0], t.shape[1], heads, -1).permute(0, 2, 1, 3)

    q, k, v = split(q), split(k), split(v)
    null_kv = sd[p + "null_kv"]  # (h, 2*nnull, dh), interleaved k0 v0 k1 v1 ...
    nk = null_kv[:, 0::2].unsqueeze(0).expand(b, -1, -1, -1)
    nv = null_kv[:, 1::2].unsqueeze(0).expand(b, -1, -1, -1)
    k = torch.cat((nk, k), dim=-2)
    v = torch.cat((nv, v), dim=-2)
    out = attention_core(q, k, v, sd[p + "q_scale"], sd[p + "k_scale"], heads=heads, causal=causal,
                         num_null_kv=num_null_kv, mask=mask, attn_bias=attn_bias, scale=scale)
    i = out.shape[-2]
    out = out.permute(0, 2, 1, 3).reshape(b, i, -1)
    return F.linear(out, sd[p + "to_out.weight"])


def continuous_position_bias(sd, p, dims):
    """attention.py:229-275 -> (heads, n, n), n = prod(dims).  Weight-only function."""
    w0 = sd[p + "net.0.0.weight"]
    pos = [torch.arange(d, device=w0.device) for d in dims]
    grid = torch.stack(torch.meshgrid(*pos, indexing="ij")).reshape(len(dims), -1).t()
    rel = (grid[:, None, :] - grid[None, :, :]).to(w0.dtype)  # the weights' dtype (fp32: the same values as before)
    h = torch.sign(rel) * torch.log(rel.abs() + 1)
    n_layers = len({k[len(p):].split(".")[1] for k in sd if k.startswith(p + "net.")})
    for li in range(n_layers - 1):
        h = F.leaky_relu(F.linear(h, sd[f"{p}net.{li}.0.weight"], sd[f"{p}net.{li}.0.bias"]), 0.1)
    h = F.linear(h, sd[f"{p}net.{n_layers - 1}.weight"], sd[f"{p}net.{n_layers - 1}.bias"])
    return h.permute(2, 0, 1)


def transformer(x, sd, p, *, heads, causal=False, peg_causal=False, video_shape=None,
                attn_bias=None, context=None, self_attn_mask=None, cross_attn_context_mask=None,
                attn_num_null_kv=2):
    """attention.py:311-332.  layers.{i}.0 PEG, .1 self-attn, .2 cross-attn, .3 FF; then norm_out."""
    depth = 1 + max(int(k[len(p):].split(".")[1]) for k in sd if k.startswith(p + "layers."))
    for i in range(depth):
        lp = f"{p}layers.{i}."
        if lp + "0.dsconv.weight" in sd:
            x = peg(x, video_shape, sd, lp + "0.", peg_causal) + x
        x = attention(x, sd, lp + "1.", heads=heads, causal=causal, attn_bias=attn_bias,
                      mask=self_attn_mask) + x
        if lp + "2.to_q.weight" in sd and context is not None:
            x = attention(x, sd, lp + "2.", heads=heads, num_null_kv=attn_num_null_kv,
                          context=context, mask=cross_attn_context_mask) + x
        x = feed_forward(x, sd, lp + "3.") + x
    return layer_norm(x, sd[p + "norm_out.gamma"], sd[p + "norm_out.beta"])


# --------------------------------------------------------------------------------------
# C-ViViT (cvivit.py)
# --------------------------------------------------------------------------------------


def cvivit_geometry(sd, image_size, patch_size):
    """Derives (dim, heads, temporal_patch_size, channels) from state-dict shapes."""
    ph, pw = patch_size
    dim = sd["to_patch_emb.2.weight"].shape[0]
    k_first = sd["to_patch_emb_first_frame.2.weight"].shape[1]
    k_rest = sd["to_patch_emb.2.weight"].shape[1]
    channels = k_first // (ph * pw)
    pt = k_rest // k_first
    heads = sd["enc_spatial_transformer.layers.0.1.null_kv"].shape[0]
    return dim, heads, pt, channels


def cvivit_patch_embed(video, sd, patch_size, pt):
    """cvivit.py:273-285, 542-549.  Feature order inside a patch is (c, pt, p1, p2)."""
    ph, pw = patch_size
    b, c, f, H, W = video.shape
    hh, ww = H // ph, W // pw

    def embed(frames, p, tpatch):
        t = frames.shape[2] // tpatch
        x = frames.reshape(b, c, t, tpatch, hh, ph, ww, pw).permute(0, 2, 4, 6, 1, 3, 5, 7)
        x = x.reshape(b, t, hh, ww, c * tpatch * ph * pw)
        x = layer_norm(x, sd[p + "1.weight"], sd[p + "1.bias"])
        x = F.linear(x, sd[p + "2.weight"], sd[p + "2.bias"])
        return layer_norm(x, sd[p + "3.weight"], sd[p + "3.bias"])

    first = embed(video[:, :, :1], "to_patch_emb_first_frame.", 1)
    if f == 1:
        return first
    rest = embed(video[:, :, 1:], "to_patch_emb.", pt)
    return torch.cat((first, rest), dim=1)


def cvivit_encode_tokens(tokens, sd, heads):
    """cvivit.py:449-474 (encode)."""
    b, t, h, w, d = tokens.shape
    video_shape = (b, t, h, w)
    x = tokens.reshape(b * t, h * w, d)
    bias = continuous_position_bias(sd, "spatial_rel_pos_bias.", (h, w))
    x = transformer(x, sd, "enc_spatial_transformer.", heads=heads, attn_bias=bias,
                    video_shape=video_shape, attn_num_null_kv=2)
    x = x.reshape(b, t, h, w, d).permute(0, 2, 3, 1, 4).reshape(b * h * w, t, d)
    x = transformer(x, sd, "enc_temporal_transformer.", heads=heads, causal=True, peg_causal=True,
                    video_shape=video_shape)
    return x.reshape(b, h, w, t, d).permute(0, 3, 1, 2, 4)


def lfq_project(x, sd):
    """oracle/lfq.py (upstream LFQ.project_in); returns the pre-sign values."""
    return F.linear(x, sd["vq.project_in.weight"], sd["vq.project_in.bias"])


def lfq_indices_from_projection(proj, sd):
    return ((proj > 0).int() * sd["vq.mask"].int()).sum(dim=-1)


def cvivit_codebook_ids(video, sd, image_size, patch_size, return_margin=False):
    """cvivit.py:518-574 with return_only_codebook_ids=True -> int64 (b, T', H', W')."""
    if video.ndim == 4:
        video = video.unsqueeze(2)
    dim, heads, pt, _ = cvivit_geometry(sd, image_size, patch_size)
    tokens = cvivit_patch_embed(video, sd, patch_size, pt)
    tokens = cvivit_encode_tokens(tokens, sd, heads)
    b, t, h, w, d = tokens.shape
    if "vq._codebook.embed" in sd:  # lookup_free_quantization=False: cosine-sim codebook (cvivit.py:321, oracle/lfq.py)
        dist = F.normalize(tokens.reshape(b, t * h * w, d), dim=-1) @ sd["vq._codebook.embed"][0].t()
        ids = dist.argmax(dim=-1).reshape(b, t, h, w)
        return (ids, dist.reshape(b, t, h, w, -1)) if return_margin else ids
    proj = lfq_project(tokens.reshape(b, t * h * w, d), sd)
    ids = lfq_indices_from_projection(proj, sd).reshape(b, t, h, w)
    if return_margin:
        return ids, proj.reshape(b, t, h, w, -1)
    return ids


def lfq_indices_to_codes(ids, sd):
    """cvivit.py:437-439 -> oracle/lfq.py indices_to_codes."""
    bits = (ids[..., None].int() & sd["vq.mask"].int()) != 0
    codes = torch.where(bits, 1.0, -1.0).float()
    return F.linear(codes, sd["vq.project_out.weight"], sd["vq.project_out.bias"])


def cvivit_decode(tokens, sd, patch_size, pt, heads, channels):
    """cvivit.py:476-516 (decode): temporal -> spatial transformers -> to_pixels un-patchify."""
    b, t, h, w, d = tokens.shape
    ph, pw = patch_size
    video_shape = (b, t, h, w)
    x = tokens.permute(0, 2, 3, 1, 4).reshape(b * h * w, t, d)
    x = transformer(x, sd, "dec_temporal_transformer.", heads=heads, causal=True, peg_causal=True,
                    video_shape=video_shape)
    x = x.reshape(b, h, w, t, d).permute(0, 3, 1, 2, 4).reshape(b * t, h * w, d)
    bias = continuous_position_bias(sd, "spatial_rel_pos_bias.", (h, w))
    x = transformer(x, sd, "dec_spatial_transformer.", heads=heads, attn_bias=bias,
                    video_shape=video_shape)
    x = x.reshape(b, t, h, w, d)
    first = F.linear(x[:, :1], sd["to_pixels_first_frame.0.weight"], sd["to_pixels_first_frame.0.bias"])
    first = first.reshape(b, 1, h, w, channels, ph, pw).permute(0, 4, 1, 2, 5, 3, 6)
    first = first.reshape(b, channels, 1, h * ph, w * pw)
    if t == 1:
        return first
    rest = F.linear(x[:, 1:], sd["to_pixels.0.weight"], sd["to_pixels.0.bias"])
    rest = rest.reshape(b, t - 1, h, w, channels, pt, ph, pw).permute(0, 4, 1, 5, 2, 6, 3, 7)
    rest = rest.reshape(b, channels, (t - 1) * pt, h * ph, w * pw)
    return torch.cat((first, rest), dim=2)


def cvivit_decode_from_ids(ids, sd, image_size, patch_size):
    """cvivit.py:437-443.  ids (b, n) or (b, t, h, w)."""
    dim, heads, pt, channels = cvivit_geometry(sd, image_size, patch_size)
    h, w = image_size[0] // patch_size[0], image_size[1] // patch_size[1]
    b = ids.shape[0]
    if "vq._codebook.embed" in sd:  # codes = vq.codebook[indices] (cvivit.py:441)
        codes = sd["vq._codebook.embed"][0][ids.reshape(b, -1)].reshape(b, -1, h, w, dim)
    else:
        codes = lfq_indices_to_codes(ids.reshape(b, -1), sd).reshape(b, -1, h, w, dim)
    return cvivit_decode(codes, sd, patch_size, pt, heads, channels)


# --------------------------------------------------------------------------------------
# MaskGit / TokenCritic (phenaki_pytorch.py)
# --------------------------------------------------------------------------------------


def _token_embed(ids, sd, p):
    n = ids.shape[1]
    return sd[p + "pos_emb.weight"][:n] + sd[p + "token_emb.weight"][ids]


def maskgit_forward(ids, sd, *, video_patch_shape, heads=8, context=None, text_mask=None,
                    video_mask=None, cond_drop=False, gradient_shrink_alpha=0.1,
                    return_embeds=False, p=""):
    """phenaki_pytorch.py:163-213.  ``cond_drop`` = cond_drop_prob==1 (keep-mask all False, :188-190;
    probabilities 0 and 1 consume no RNG, :73-77)."""
    if ids.ndim == 4:
        video_patch_shape = tuple(ids.shape[1:])
        ids = ids.reshape(ids.shape[0], -1)
    b, n = ids.shape
    if text_mask is None:
        text_mask = torch.ones((b, n), dtype=torch.bool, device=ids.device)
    bias = continuous_position_bias(sd, p + "continuous_pos_bias.", video_patch_shape)
    if cond_drop:
        text_mask = torch.zeros_like(text_mask)
    x = _token_embed(ids, sd, p)
    a = gradient_shrink_alpha
    x = x * a + x.detach() * (1 - a)  # the gradient-shrink trick (:199): same forward value, gradient scaled by a
    x = transformer(x, sd, p + "transformer.", heads=heads, video_shape=(b, *video_patch_shape),
                    attn_bias=bias, context=context, self_attn_mask=video_mask,
                    cross_attn_context_mask=text_mask, attn_num_null_kv=2)
    if return_embeds:
        return x
    return F.linear(x, sd[p + "to_logits.weight"], sd[p + "to_logits.bias"])


def critic_forward(ids, sd, *, video_patch_shape, heads=8, context=None, text_mask=None,
                   video_mask=None, cond_drop=False, p=""):
    """phenaki_pytorch.py:265-302 (TokenCritic): no rel-pos bias; Linear(dim,1) head."""
    b = ids.shape[0]
    ids = ids.reshape(b, -1)
    n = ids.shape[1]
    if text_mask is None:
        text_mask = torch.ones((b, n), dtype=torch.bool, device=ids.device)
    if context is not None and cond_drop:
        text_mask = torch.zeros_like(text_mask)
    x = _token_embed(ids, sd, p)
    x = transformer(x, sd, p + "transformer.", heads=heads, video_shape=(b, *video_patch_shape),
                    context=context, self_attn_mask=video_mask, cross_attn_context_mask=text_mask)
    return F.linear(x, sd[p + "to_logits.0.weight"], sd[p + "to_logits.0.bias"]).squeeze(-1)


def with_cond_scale(fn, cond_scale):
    """phenaki_pytorch.py:149-161 / :251-263."""
    out = fn(cond_drop=False)
    if cond_scale == 1:
        return out
    null = fn(cond_drop=True)
    return null + (out - null) * cond_scale


# --------------------------------------------------------------------------------------
# sampling (phenaki_pytorch.py:83-93, 418-560)
# --------------------------------------------------------------------------------------


def _log(t, eps=1e-10):
    return torch.log(t + eps)


def gumbel_sample(logits, temperature, u):
    """phenaki_pytorch.py:88-93 with the uniform draw ``u`` made explicit."""
    return ((logits / max(temperature, 1e-10)) + (-_log(-_log(u)))).argmax(dim=-1)


def torch_noise(shape, tag):
    """Default noise source = exactly the reference's draw (global CPU generator)."""
    return torch.zeros(shape).float().uniform_(0, 1)


def demask_schedule(num_tokens, steps):
    """phenaki_pytorch.py:485-486: k_s for s = 1..steps-1 (fp32 cos, round-half-even, clamp>=1)."""
    ks = []
    for step in range(1, steps):
        t = torch.full((1,), step / steps)
        ks.append(int((num_tokens * torch.cos(t * math.pi * 0.5)).round().long().clamp(min=1).item()))
    return ks


def sample_token_ids(maskgit_sd, *, num_tokens, patch_shape, batch, steps=18, heads=8,
                     text_embeds=None, text_mask=None, prime_ids=None, cond_scale=3.0,
                     starting_temperature=0.9, noise_K=1.0, critic_sd=None,
                     critic_has_cross_attn=True, critic_noise_anneal="decay",
                     noise_fn=torch_noise, mask_id=None, trace=None, self_critic=None):
    """The demasking loop, phenaki_pytorch.py:473-550 (everything between text encoding and the
    final C-ViViT decode).  ``noise_fn(shape, tag)`` supplies every uniform draw in reference
    order: tag 'gumbel{step}' (b, n, V) then 'critic{step}' (b, n).
    ``self_critic`` = (to_pred.weight, to_pred.bias): SelfCritic (phenaki_pytorch.py:307-336), Linear(dim, 1) on the
    MaskGit embeddings of the sampled ids, scored like a TokenCritic.
    Returns final ids (b, num_tokens) int64 (without the prime prefix)."""
    if mask_id is None:
        mask_id = maskgit_sd["to_logits.weight"].shape[0]
    if text_embeds is not None and text_mask is None:
        text_mask = torch.any(text_embeds != 0, dim=-1)
    dev = maskgit_sd["to_logits.weight"].device
    shape = (batch, num_tokens)
    ids = torch.full(shape, mask_id, dtype=torch.long, device=dev)
    mask = torch.ones(shape, dtype=torch.bool, device=dev)
    scores = None
    has_prime = prime_ids is not None
    plen = prime_ids.shape[-1] if has_prime else 0
    for step in range(steps):
        last = step == steps - 1
        til_x0 = steps - (step + 1)
        if step > 0 and scores is not None:
            t = torch.full((1,), step / steps)
            k = (num_tokens * torch.cos(t * math.pi * 0.5)).round().long().clamp(min=1)
            _, idx = scores.topk(k.item(), dim=-1)
            mask = torch.zeros(shape, device=dev).scatter(1, idx, 1).bool()
        ids = torch.where(mask, mask_id, ids)
        inp = ids if not has_prime else torch.cat((prime_ids, ids), dim=-1)
        logits = with_cond_scale(
            lambda cond_drop: maskgit_forward(inp, maskgit_sd, video_patch_shape=patch_shape,
                                              heads=heads, context=text_embeds, text_mask=text_mask,
                                              cond_drop=cond_drop), cond_scale)
        if has_prime:
            logits = logits[:, plen:]
        temperature = starting_temperature * (til_x0 / steps)
        u = noise_fn(tuple(logits.shape), f"gumbel{step}")
        pred = gumbel_sample(logits, temperature, u)
        ids = torch.where(mask, pred, ids)
        if trace is not None:
            trace.append(dict(step=step, mask=mask.clone(), pred=pred.clone(), ids=ids.clone()))
        if not last:
            if critic_sd is not None or self_critic is not None:
                cin = ids if not has_prime else torch.cat((prime_ids, ids), dim=-1)
                ctx = text_embeds if critic_has_cross_attn else None
                if self_critic is not None:  # SelfCritic.forward (:334-336) under forward_with_cond_scale (:320-332)
                    scores = with_cond_scale(
                        lambda cond_drop: F.linear(
                            maskgit_forward(cin, maskgit_sd, video_patch_shape=patch_shape, heads=heads,
                                            context=text_embeds, text_mask=text_mask, cond_drop=cond_drop,
                                            return_embeds=True), self_critic[0], self_critic[1]).squeeze(-1),
                        cond_scale)
                else:
                    scores = with_cond_scale(
                        lambda cond_drop: critic_forward(cin, critic_sd, video_patch_shape=patch_shape,
                                                         heads=heads, context=ctx, text_mask=text_mask,
                                                         cond_drop=cond_drop), cond_scale)
                if has_prime:
                    scores = scores[:, plen:]
                mult = {"fixed": 1.0, "decay": til_x0 / steps, "increase": (step + 1) / steps}[critic_noise_anneal]
                scores = scores + noise_K * (noise_fn(tuple(scores.shape), f"critic{step}") - 0.5) * mult
            else:
                probs = logits.softmax(dim=-1)
                sc = probs.gather(2, pred[..., None]).squeeze(-1)
                scores = torch.where(mask, 1 - sc, -1e4)
            if trace is not None:
                trace[-1]["scores"] = scores.clone()
    return ids


# --------------------------------------------------------------------------------------
# training loss (phenaki_pytorch.py:562-687); differentiable through torch autograd when the
# state-dict tensors require grad -- the gradient oracle of the training-step kernels (SURVEY 8f-2)
# --------------------------------------------------------------------------------------


def mask_subset_with_prob(mask, prob, u):
    """phenaki_pytorch.py:43-55 (get_mask_subset_with_prob) with the uniform draw ``u`` (b, n) made explicit.
    Kept as is: the subset is chosen by RANK of the draw, the padding only shifts the ranks."""
    b, n = mask.shape
    num_tokens = mask.sum(dim=-1)
    num_pads = n - num_tokens
    num_masked = (prob * num_tokens).round().clamp(min=1)
    ranks = u.argsort(dim=-1)
    ranks = ranks - num_pads[:, None]
    ranks = ranks.masked_fill(ranks < 0, n)
    return ranks < num_masked[:, None]


def train_draws(batch, seq, steps):
    """The draws of one Phenaki.forward in reference order, from the global CPU generator:
    ``rand_step`` (:614) then the uniform behind the random permutation (:48)."""
    rand_step = torch.randint(0, steps, (batch,))
    u = torch.rand((batch, seq))
    return rand_step, u


def train_token_mask(rand_step, u, steps, video_mask=None):
    """phenaki_pytorch.py:614-620: cosine schedule -> which tokens are replaced by the mask id."""
    b, n = u.shape
    prob = torch.cos(rand_step * math.pi * 0.5 / steps)
    if video_mask is None:
        video_mask = torch.ones((b, n), dtype=torch.bool)
    return mask_subset_with_prob(video_mask, prob, u)


def maskgit_train_loss(ids, sd, token_mask, *, video_patch_shape, heads=8, context=None, text_mask=None,
                       video_mask=None, mask_id=None, return_logits=False, p=""):
    """phenaki_pytorch.py:620-640: masked input -> MaskGit logits -> cross entropy at the masked positions.
    ``cond_drop_prob`` is 0 in the reference's training forward (it overwrites the argument at :594, SURVEY defects),
    so no text dropout and no RNG.  ids (b, n) int64, token_mask (b, n) bool."""
    if mask_id is None:
        mask_id = sd[p + "to_logits.weight"].shape[0]
    b, n = ids.shape
    if video_mask is None:
        video_mask = torch.ones((b, n), dtype=torch.bool)  # :617-618
    masked = torch.where(token_mask, mask_id, ids)
    logits = maskgit_forward(masked, sd, video_patch_shape=video_patch_shape, heads=heads, context=context,
                             text_mask=text_mask, video_mask=video_mask, p=p)
    loss = F.cross_entropy(logits[token_mask], ids[token_mask])
    return (loss, logits) if return_logits else loss


def critic_train_loss(ids, pred_ids, token_mask, critic_sd, *, video_patch_shape, heads=8, context=None,
                      text_mask=None, video_mask=None, p=""):
    """phenaki_pytorch.py:652-680: critic input = predictions at the masked positions, labels = "was changed";
    binary cross entropy with logits over ALL positions."""
    b, n = ids.shape
    if video_mask is None:
        video_mask = torch.ones((b, n), dtype=torch.bool)
    critic_input = torch.where(token_mask, pred_ids, ids)
    scores = critic_forward(critic_input, critic_sd, video_patch_shape=video_patch_shape, heads=heads,
                            context=context, text_mask=text_mask, video_mask=video_mask, p=p)
    labels = (ids != pred_ids).to(scores.dtype)
    return F.binary_cross_entropy_with_logits(scores, labels)


def self_critic_train_loss(ids, pred_ids, token_mask, maskgit_sd, to_pred_w, to_pred_b, *, video_patch_shape, heads=8,
                           context=None, text_mask=None, video_mask=None):
    """Same with a SelfCritic (phenaki_pytorch.py:307-336): Linear(dim, 1) on the MaskGit embeddings
    (``return_embeds=True``), so this loss also differentiates MaskGit."""
    b, n = ids.shape
    if video_mask is None:
        video_mask = torch.ones((b, n), dtype=torch.bool)
    critic_input = torch.where(token_mask, pred_ids, ids)
    emb = maskgit_forward(critic_input, maskgit_sd, video_patch_shape=video_patch_shape, heads=heads, context=context,
                          text_mask=text_mask, video_mask=video_mask, return_embeds=True)
    scores = F.linear(emb, to_pred_w, to_pred_b).squeeze(-1)
    return F.binary_cross_entropy_with_logits(scores, (ids != pred_ids).to(scores.dtype))
