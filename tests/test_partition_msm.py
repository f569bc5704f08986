"""Fixed-base MSMs answered from a partition table on the handle (partition_msm.cuh), with the
product's kernel bodies run as serial host loops (tests/emul): every result equals the oracle's
(oracle/port.fixed_msm) after normalisation, over table widths 1..16, the three scalar layouts,
degenerate generators, edge-case scalars and the three routing policies."""
import numpy as np
import pytest

from tests import common
from tests import partition_msm_emul as pm
from tests import partition_tables as pt

CURVES = [0, 1, 2, 3]
# packed widths 1..256, many of them 1 bit
WIDTHS = [1, 1, 1, 5, 1, 64, 256, 1, 13, 8, 1, 2]


def _vlen_lengths(n, w):
    lens = [0, 1, max(w - 1, 0), w, w + 1, n, 2, n - 1, w, 3, n, n]
    return sorted(min(v, n) for v in lens)


def _check(emul, port, curve, gens, w, policy, num_outputs, n, sc, chunk_groups=0, **kw):
    want = port.normalize(curve, port.fixed_msm(curve, gens, num_outputs, n, sc, **kw))
    got = pm.fixed_msm(emul, curve, gens, w, policy, num_outputs, n, sc, chunk_groups=chunk_groups,
                       **kw)
    assert common.same(curve, port.normalize(curve, got), want), (curve, w, policy, kw)


@pytest.mark.parametrize("curve", CURVES)
@pytest.mark.parametrize("w", [1, 3, 8, 16])
def test_layouts_and_widths(emul, port, curve, w):
    """Modes 0, 1 and 2 from the table alone (policy 1), n not a multiple of w; vlen lengths 0, 1,
    w - 1, w, w + 1 and n."""
    n = 20 if w == 16 else 2 * w + 7
    _, gens = common.generators_for(port, curve, n, seed=5 + w)
    rng = np.random.default_rng(100 * curve + w)
    sc = rng.integers(0, 256, (n, 3 * 2), dtype=np.uint8)
    _check(emul, port, curve, gens, w, pm.POLICY_TABLE, 3, n, sc, element_num_bytes=2)
    row = (sum(WIDTHS) + 7) // 8
    psc = rng.integers(0, 256, (n, row), dtype=np.uint8)
    if w != 16:
        _check(emul, port, curve, gens, w, pm.POLICY_TABLE, len(WIDTHS), n, psc,
               output_bit_table=WIDTHS)
    _check(emul, port, curve, gens, w, pm.POLICY_TABLE, len(WIDTHS), n, psc,
           output_bit_table=WIDTHS, output_lengths=_vlen_lengths(n, w))


@pytest.mark.parametrize("curve", CURVES)
@pytest.mark.parametrize("w", [3, 6])
def test_degenerate_generators_and_scalars(emul, port, curve, w):
    """Duplicates, G / -G pairs and identity generators (zero sums inside the table), with random,
    all-zero and all-ones scalars; the table built in one chunk and in chunks of two groups."""
    n = 29
    _, gens = common.generators_for(port, curve, n, seed=44)
    gens = pt.edit_generators(curve, np.array(gens, copy=True))
    row = (sum(WIDTHS) + 7) // 8
    rng = np.random.default_rng(curve + w)
    for fill in ("random", 0x00, 0xFF):
        if fill == "random":
            psc = rng.integers(0, 256, (n, row), dtype=np.uint8)
        else:
            psc = np.full((n, row), fill, dtype=np.uint8)
        _check(emul, port, curve, gens, w, pm.POLICY_TABLE, len(WIDTHS), n, psc,
               chunk_groups=2 if fill == 0xFF else 0, output_bit_table=WIDTHS,
               output_lengths=_vlen_lengths(n, w))


@pytest.mark.parametrize("curve", CURVES)
@pytest.mark.parametrize("policy", [pm.POLICY_MODEL, pm.POLICY_TABLE, pm.POLICY_ENGINE])
def test_policies(emul, port, curve, policy):
    n = 50
    _, gens = common.generators_for(port, curve, n, seed=9)
    rng = np.random.default_rng(7 * curve + policy)
    psc = rng.integers(0, 256, (n, (sum(WIDTHS) + 7) // 8), dtype=np.uint8)
    _check(emul, port, curve, gens, 4, policy, len(WIDTHS), n, psc, output_bit_table=WIDTHS)
    _check(emul, port, curve, gens, 4, policy, len(WIDTHS), n, psc, output_bit_table=WIDTHS,
           output_lengths=_vlen_lengths(n, 4))


def test_engine_policy_is_the_engine(emul, port):
    """Policy 2 and a handle without a table give the same bytes (the engine's own results)."""
    n = 40
    _, gens = common.generators_for(port, 2, n, seed=2)
    psc = np.random.default_rng(3).integers(0, 256, (n, (sum(WIDTHS) + 7) // 8), dtype=np.uint8)
    a = pm.fixed_msm(emul, 2, gens, 0, pm.POLICY_MODEL, len(WIDTHS), n, psc, output_bit_table=WIDTHS)
    b = pm.fixed_msm(emul, 2, gens, 3, pm.POLICY_ENGINE, len(WIDTHS), n, psc,
                     output_bit_table=WIDTHS)
    assert np.array_equal(a, b)
    assert pm.route(emul, 2, n, 3, pm.POLICY_ENGINE, WIDTHS, [n] * len(WIDTHS)) == []
    assert pm.route(emul, 2, n, 3, pm.POLICY_TABLE, WIDTHS, [n] * len(WIDTHS)) == \
        list(range(len(WIDTHS)))
    # empty outputs stay with the engine under every policy
    assert 0 not in pm.route(emul, 2, n, 3, pm.POLICY_TABLE, WIDTHS, [0] + [n] * (len(WIDTHS) - 1))


# 1-bit outputs are cheaper from a width-3 table, 256-bit ones from the engine
SPLIT_WIDTHS = [1, 256, 1, 1, 256, 8, 1]


@pytest.mark.parametrize("curve", CURVES)
def test_cost_model_splits_outputs(emul, port, curve):
    n = 2000
    routed = pm.route(emul, curve, n, 3, pm.POLICY_MODEL, SPLIT_WIDTHS, [n] * len(SPLIT_WIDTHS))
    assert 0 < len(routed) < len(SPLIT_WIDTHS), routed
    assert 0 in routed and 1 not in routed
    _, gens = common.generators_for(port, curve, n, seed=12)
    psc = np.random.default_rng(curve).integers(0, 256, (n, (sum(SPLIT_WIDTHS) + 7) // 8),
                                                dtype=np.uint8)
    _check(emul, port, curve, gens, 3, pm.POLICY_MODEL, len(SPLIT_WIDTHS), n, psc,
           output_bit_table=SPLIT_WIDTHS)
