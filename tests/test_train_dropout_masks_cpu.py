"""CPU: the dropout mask contract of the training step (include/phk.h, phk_dropout_t) on the independent Philox4x32-7 of
tests/noise_ref.py: the kept fraction is binomial, and the sites of a step, its layers and successive steps draw from
disjoint counters."""
import math

import numpy as np
import pytest

from tests import dropout_ref as DR
from tests import train_at_size_cases as T
from tests import train_dropout_cases as TD


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_kept_fraction_is_binomial(p):
    count = 1 << 20
    for seed, base in ((0, 0), (2 ** 63 + 12345, 2 ** 64 - 1000)):  # the 64-bit counter wraps in the second
        kept = int(DR.keep(seed, base, count, p).sum())
        mean, sd = count * (1 - p), math.sqrt(count * p * (1 - p))
        assert abs(kept - mean) < 5 * sd, (seed, base, kept, mean, sd)


def test_element_uses_word_e_mod_4_of_counter_base_plus_e_div_4():
    from tests import noise_ref as N
    seed, base = 987654321987, 77
    kept = DR.keep(seed, base, 10, 0.5)
    u = N.uniforms(seed, base, [0], 12)[0][:10]  # one row of 12 draws = counters base .. base + 2
    assert np.array_equal(kept, u >= 0.5)


def test_extreme_probabilities():
    assert DR.keep(1, 0, 4096, 0.0).all()
    assert not DR.keep(1, 0, 4096, 1.0).any()
    assert DR.multiplier(DR.keep(1, 0, 16, 1.0), 1.0, None).abs().sum() == 0


@pytest.mark.parametrize("name", ["tiny", "ragged_ce", "prod_critic", "emu_critic_split_head"])
def test_sites_layers_and_steps_use_disjoint_counters(name):
    c = TD.case(name)
    module = T.build_module(c)
    n = math.prod(c["patch_shape"])
    sites, total = DR.layout(module, c["batch"], n, c["ctx_len"])
    spans = sorted((base, base + (math.prod(shape) + 3) // 4) for _, _, shape, base in sites)
    assert spans[0][0] == 0 and spans[-1][1] == total
    for (_, hi), (lo, _) in zip(spans, spans[1:]):
        assert hi == lo  # back to back: no gap, no overlap
    depth = len(module.transformer.layers)
    per_layer = 3 if c["ctx_len"] and module.transformer.layers[0][2] is not None else 2
    assert len(sites) == depth * per_layer
    # successive steps: the next one starts round_up(total, 4) further on (the generator's granularity), past this one
    first, second = DR.keep(5, 0, 4 * total, 0.5), DR.keep(5, (total + 3) // 4 * 4, 4 * total, 0.5)
    assert not np.array_equal(first, second)
