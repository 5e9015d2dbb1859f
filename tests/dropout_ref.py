"""Reference side of the training step's dropout (include/phk.h, phk_dropout_t), for the tests.

1. The masks, rebuilt in numpy from the counter contract with the independent Philox4x32-7 of tests/noise_ref.py: element
   e of a site is kept iff u(base + e / 4, word e % 4) >= p (p as fp32), u = (2 (draw >> 9) + 1) / 2^24.  The site
   layout is restated here from the contract, not read from the library, so that the tests can check the library's
   counter count against it.
2. A dropout-aware restatement of the training losses: the functions of oracle/phenaki_oracle.py with the reference's
   nn.Dropout (attention.py:51, 177, training mode) applied as a multiplication by given per-site masks.  The oracle's
   own primitives (LayerNorm, PEG, position bias, embeddings) are reused; with every mask None the losses equal the
   oracle's.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import phenaki_oracle as O
from tests import noise_ref as N


# ---- masks --------------------------------------------------------------------------------------------------------
def layout(module, b, n, L):
    """[(layer, site, shape, base)] of one step, bases relative to the step's offset; site 'self' | 'cross' | 'ff'.
    ``module``: the MaskGit / TokenCritic; L = 0 when the step has no context.  Returns (sites, total counters)."""
    tf = module.transformer
    sites, base = [], 0
    for li, layer in enumerate(tf.layers):
        cross = layer[2] is not None and L > 0
        inner = layer[3][1].weight.shape[0] // 2
        for name, shape in (("self", (b, tf.heads, n, n)),
                            ("cross", (b, tf.heads, n, layer[2].num_null_kv + L) if cross else None),
                            ("ff", (b * n, inner))):
            count = int(np.prod(shape)) if shape is not None else 0
            if shape is not None:
                sites.append((li, name, shape, base))
            base += (count + 3) // 4
    return sites, base


def keep(seed, base, count, p):
    """bool [count]: the keep decisions of elements 0 .. count-1 of a site whose first counter is ``base``."""
    seed %= 2 ** 64
    nb = (count + 3) // 4
    with np.errstate(over="ignore"):
        c = np.uint64(base % 2 ** 64) + np.arange(nb, dtype=np.uint64)
    words = N.philox4x32((c & N.LO32, c >> N.S32, 0, 0), (seed & 0xFFFFFFFF, seed >> 32))
    draws = np.stack(words, axis=-1).reshape(-1)[:count]
    u = (2.0 * (draws >> np.uint64(9)).astype(np.float64) + 1.0) / 2.0 ** 24  # exact, as in fp32
    return u >= float(np.float32(p))


def multiplier(kept, p, dtype):
    """M / (1 - p) as a tensor: 0 where dropped, 1 / (1 - p) (p as fp32) where kept; p = 1 gives zeros."""
    p32 = float(np.float32(p))
    scale = 0.0 if p32 >= 1.0 else 1.0 / (1.0 - p32)
    return torch.from_numpy(kept.astype(np.float64) * scale).to(dtype)


def step_masks(module, b, n, L, seed, offset, attn_p, ff_p, dtype=torch.float64):
    """Per layer {'self': [b, H, n, n] | None, 'cross': [b, H, n, nnull + L] | None, 'ff': [b, n, inner] | None}: the
    multipliers the step with (seed, offset) applies (None where that probability is 0)."""
    sites, _ = layout(module, b, n, L)
    out = [dict(self=None, cross=None, ff=None) for _ in module.transformer.layers]
    for li, name, shape, base in sites:
        p = ff_p if name == "ff" else attn_p
        if p <= 0:
            continue
        m = multiplier(keep(seed, offset + base, int(np.prod(shape)), p), p, dtype)
        out[li][name] = m.reshape(b, n, -1) if name == "ff" else m.reshape(shape)
    return out


# ---- losses with masks (oracle/phenaki_oracle.py + dropout) -------------------------------------------------------
def feed_forward(x, sd, p, drop=None):
    """attention.py:45-53: Sequential index 3 (nn.Dropout) between GEGLU and the second Linear."""
    h = O.layer_norm(x, sd[p + "0.weight"], sd[p + "0.bias"])
    h = F.linear(h, sd[p + "1.weight"])
    val, gate = h.chunk(2, dim=-1)
    h = F.gelu(gate) * val
    if drop is not None:
        h = h * drop
    return F.linear(h, sd[p + "4.weight"])


def attention(x, sd, p, *, heads, num_null_kv=0, mask=None, context=None, attn_bias=None, drop=None):
    """O.attention (attention.py:128-182) with the dropout of the probabilities before attn @ v (:177)."""
    b = x.shape[0]
    if context is not None:
        context = O.layer_norm(context, sd[p + "context_norm.gamma"], sd[p + "context_norm.beta"])
    kv_input = context if context is not None else x
    xn = O.layer_norm(x, sd[p + "norm.gamma"], sd[p + "norm.beta"])
    q = F.linear(xn, sd[p + "to_q.weight"])
    k, v = F.linear(kv_input, sd[p + "to_kv.weight"]).chunk(2, dim=-1)

    def split(t):
        return t.reshape(t.shape[0], t.shape[1], heads, -1).permute(0, 2, 1, 3)

    q, k, v = split(q), split(k), split(v)
    null_kv = sd[p + "null_kv"]
    k = torch.cat((null_kv[:, 0::2].unsqueeze(0).expand(b, -1, -1, -1), k), dim=-2)
    v = torch.cat((null_kv[:, 1::2].unsqueeze(0).expand(b, -1, -1, -1), v), dim=-2)
    q = F.normalize(q, dim=-1) * sd[p + "q_scale"]
    k = F.normalize(k, dim=-1) * sd[p + "k_scale"]
    sim = torch.einsum("bhid,bhjd->bhij", q, k) * 8
    if attn_bias is not None:
        sim = sim + F.pad(attn_bias, (num_null_kv, 0), value=0.0)
    if mask is not None:
        m = F.pad(mask, (num_null_kv, 0), value=True)
        sim = sim.masked_fill(~m[:, None, None, :], -torch.finfo(sim.dtype).max)
    attn = sim.softmax(dim=-1)
    if drop is not None:
        attn = attn * drop
    out = torch.einsum("bhij,bhjd->bhid", attn, v)
    out = out.permute(0, 2, 1, 3).reshape(b, out.shape[-2], -1)
    return F.linear(out, sd[p + "to_out.weight"])


def transformer(x, sd, p, *, heads, video_shape, attn_bias=None, context=None, self_attn_mask=None,
                cross_attn_context_mask=None, masks=None):
    """O.transformer for the MaskGit / TokenCritic (non-causal, PEG, 2 null keys in the cross-attention)."""
    depth = 1 + max(int(k[len(p):].split(".")[1]) for k in sd if k.startswith(p + "layers."))
    for i in range(depth):
        lp = f"{p}layers.{i}."
        dm = masks[i] if masks is not None else dict(self=None, cross=None, ff=None)
        if lp + "0.dsconv.weight" in sd:
            x = O.peg(x, video_shape, sd, lp + "0.", False) + x
        x = attention(x, sd, lp + "1.", heads=heads, attn_bias=attn_bias, mask=self_attn_mask, drop=dm["self"]) + x
        if lp + "2.to_q.weight" in sd and context is not None:
            x = attention(x, sd, lp + "2.", heads=heads, num_null_kv=2, context=context, mask=cross_attn_context_mask,
                          drop=dm["cross"]) + x
        x = feed_forward(x, sd, lp + "3.", drop=dm["ff"]) + x
    return O.layer_norm(x, sd[p + "norm_out.gamma"], sd[p + "norm_out.beta"])


def _maskgit_embeds(ids, sd, *, video_patch_shape, heads, context, text_mask, video_mask, masks):
    b, n = ids.shape
    bias = O.continuous_position_bias(sd, "continuous_pos_bias.", video_patch_shape)
    x = O._token_embed(ids, sd, "")
    x = x * 0.1 + x.detach() * 0.9  # gradient shrink (phenaki_pytorch.py:199), alpha 0.1
    return transformer(x, sd, "transformer.", heads=heads, video_shape=(b, *video_patch_shape), attn_bias=bias,
                       context=context, self_attn_mask=video_mask, cross_attn_context_mask=text_mask, masks=masks)


def _defaults(ids, video_mask):
    b, n = ids.shape
    return torch.ones((b, n), dtype=torch.bool) if video_mask is None else video_mask


def maskgit_train_loss(ids, sd, token_mask, *, video_patch_shape, heads=8, context=None, text_mask=None,
                       video_mask=None, masks=None):
    """O.maskgit_train_loss with the dropout masks of one step."""
    video_mask = _defaults(ids, video_mask)
    masked = torch.where(token_mask, sd["to_logits.weight"].shape[0], ids)
    emb = _maskgit_embeds(masked, sd, video_patch_shape=video_patch_shape, heads=heads, context=context,
                          text_mask=text_mask, video_mask=video_mask, masks=masks)
    logits = F.linear(emb, sd["to_logits.weight"], sd["to_logits.bias"])
    return F.cross_entropy(logits[token_mask], ids[token_mask])


def critic_train_loss(ids, pred_ids, token_mask, sd, *, video_patch_shape, heads=8, context=None, text_mask=None,
                      video_mask=None, masks=None):
    """O.critic_train_loss (TokenCritic: no position bias, no gradient shrink) with the masks of one step."""
    b, n = ids.shape
    video_mask = _defaults(ids, video_mask)
    x = O._token_embed(torch.where(token_mask, pred_ids, ids), sd, "")
    x = transformer(x, sd, "transformer.", heads=heads, video_shape=(b, *video_patch_shape), context=context,
                    self_attn_mask=video_mask, cross_attn_context_mask=text_mask, masks=masks)
    scores = F.linear(x, sd["to_logits.0.weight"], sd["to_logits.0.bias"]).squeeze(-1)
    return F.binary_cross_entropy_with_logits(scores, (ids != pred_ids).to(scores.dtype))


def self_critic_train_loss(ids, pred_ids, token_mask, maskgit_sd, to_pred_w, to_pred_b, *, video_patch_shape, heads=8,
                           context=None, text_mask=None, video_mask=None, masks=None):
    """O.self_critic_train_loss with the masks of the BCE step (its own, fresh ones)."""
    video_mask = _defaults(ids, video_mask)
    emb = _maskgit_embeds(torch.where(token_mask, pred_ids, ids), maskgit_sd, video_patch_shape=video_patch_shape,
                          heads=heads, context=context, text_mask=text_mask, video_mask=video_mask, masks=masks)
    scores = F.linear(emb, to_pred_w, to_pred_b).squeeze(-1)
    return F.binary_cross_entropy_with_logits(scores, (ids != pred_ids).to(scores.dtype))
