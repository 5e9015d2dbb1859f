"""Float64 references and error bars for the training step's products (tests/train_products_cases.py).

Every reference is computed from values the kernel itself consumed: the inputs a test hands in, or intermediates read
back from the kernel's own scratch after the call.  A bf16 product is referenced by rounding exactly those fp32
operands to bf16 (round to nearest even, as __float2bfloat16_rn) and multiplying the rounded values in float64.

Bars, per output element (u = 2^-23, the fp32 unit roundoff):
  bf16 products:  2^-16 * (|A^|.|B^|)  +  u * prefill_adds * |prefill|
      A^, B^ are the bf16 operands; bf16 x bf16 products are exact in fp32, so the only error left is the fp32
      accumulation.  With random-sign data its partial sums stay near sqrt(K) * rms, far below (|A^|.|B^|) (which
      grows like K), so at K <= 6144 the accumulation error sits orders of magnitude under the bar.  The bar is 2^7
      below what rounding a single operand differently does (2^-9 relative per product), so a wrong rounding mode,
      unrounded operands or one product too many or too few each break it.  It is TIGHTER than the worst-case
      accumulation bound for arbitrary inputs (about (K / 16) * 2u * (|A^|.|B^|) for a tensor core that truncates
      within each k16 step); it holds for the random-sign operands these tests use, not for adversarial ones.
  fp32 products:  (K + adds) * u * (|A|.|B| + |prefill|)   -- the recursive-summation bound of K fused multiply-adds
      plus the `adds` fp32 additions that combine partial sums and the prefill (split-K atomics, bias, residual).
      It holds for any summation order, so it cannot be flaky.
"""
import torch

U = 2.0 ** -23
BF16_REL = 2.0 ** -16


def rne(x):
    """fp32 -> bf16, round to nearest even (torch's conversion = __float2bfloat16_rn), as float64."""
    return x.float().bfloat16().double()


def rtz(x):
    """fp32 -> bf16 rounded toward zero (the low 16 bits dropped), as float64: the wrong rounding the bar must catch."""
    bits = x.float().contiguous().view(torch.int32) & -65536
    return bits.view(torch.float32).double()


def exact(x):
    """unrounded fp32 operand as float64: the missing rounding the bar must catch."""
    return x.double()


def bf16_bar(a_hat, b_hat, prefill=None, prefill_adds=1):
    bar = BF16_REL * (a_hat.abs() @ b_hat.abs())
    if prefill is not None:
        bar = bar + U * prefill_adds * prefill.double().abs()
    return bar


def f32_bar(a, b, k, prefill=None, adds=1):
    mag = a.double().abs() @ b.double().abs()
    if prefill is not None:
        mag = mag + prefill.double().abs()
    return (k + adds) * U * mag


def worst(got, ref, bar):
    """max over elements of |got - ref| / bar (0 / 0 counts as 0, a NaN in got as infinity)."""
    err = (got.double() - ref).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bar)
    ratio = torch.where(torch.isnan(got.double()), torch.full_like(ratio, float("inf")), ratio)
    return float(ratio.max()) if ratio.numel() else 0.0


def assert_within(name, got, ref, bar, alternatives=None):
    """got within bar of ref everywhere; prints the margin.  alternatives: {label: reference from wrongly rounded
    operands}, each of which must break the same bar on some element (the bar can tell the rounding apart)."""
    w = worst(got, ref, bar)
    print(f"[train-products] {name}: worst err/bar {w:.3g}")
    assert w <= 1.0, f"{name}: error {w:.3g} x the bar"
    for label, alt in (alternatives or {}).items():
        wa = worst(alt, ref, bar)
        assert wa > 1.0, f"{name}: the {label} reference stays within the bar ({wa:.3g}): the bar cannot see it"


def assert_close_norms(name, got, ref, max_rel=1e-4, frob_rel=2e-5):
    """fp32 grade: max |got - ref| <= max_rel * max |ref| and ||got - ref||_F <= frob_rel * ||ref||_F."""
    d = got.double() - ref
    scale = float(ref.abs().max())
    e_max = float(d.abs().max())
    e_f = float(d.norm()) / max(float(ref.norm()), 1e-300)
    print(f"[train-products] {name}: max err / max|ref| {e_max / max(scale, 1e-300):.3g} (bar {max_rel:g}), "
          f"rel Frobenius {e_f:.3g} (bar {frob_rel:g})")
    assert not torch.isnan(got).any(), f"{name}: NaN"
    assert e_max <= max_rel * scale, f"{name}: max error {e_max:.3g} > {max_rel:g} * {scale:.3g}"
    assert e_f <= frob_rel, f"{name}: relative Frobenius error {e_f:.3g} > {frob_rel:g}"


def assert_step_grade(name, got, ref):
    """the training step's bf16 closeness bar: within 5 % of the largest entry, cosine >= 0.995."""
    g, r = got.double().flatten(), ref.flatten()
    scale = float(r.abs().max())
    e = float((g - r).abs().max())
    cos = float(g @ r) / max(float(g.norm() * r.norm()), 1e-300)
    assert e <= 0.05 * scale and cos >= 0.995, f"{name}: max err {e:.3g} of {scale:.3g}, cosine {cos:.5f}"


def l2norm_scale_bwd(raw, scale, dhat):
    """float64 backward of hat = raw / max(|raw|, 1e-12) * scale over the last dim: (d raw, per-row d scale)."""
    raw = raw.double()
    r = raw.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    u = raw / r
    g = dhat * scale.double()
    draw = (g - u * (u * g).sum(-1, keepdim=True)) / r
    return draw, dhat * u
