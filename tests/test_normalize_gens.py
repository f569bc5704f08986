"""Normalising ingestion of ed25519 caller generators (msm.cuh ingest_normalized) through the CPU
emulation of the kernel bodies: generators given in scaled projective representations, with
duplicated, negated and identity generators, must give the oracle's commitments with the
normalisation on and byte-equal ones with it off, in one and in several generator ranges, through the
device call and the offsets call. A Z = 0 generator (not a point) must leave the results exactly as
they are without the normalisation."""
import numpy as np
import pytest

from tests import common
from tests import normalize_emul as ne
from tests.emul import harness

N = 300
SHAPES = [(0, 32, 0), (-100, 16, 1), (0, 1, 0), (-250, 8, 0)]
SPECIAL = dict(identity=(5, 77), negated=(9, 150), duplicated=(10, 11, 151))


def _gens(port, n, seed, **kw):
    return ne.scaled_generators(port.ristretto_generators(n), seed, **kw)


def test_ingestion_writes_unit_z(port):
    gens = _gens(port, 50, 1, **SPECIAL)
    dev, flag = harness.ingest_generators(gens)
    assert flag == 0
    for row in dev:
        ypx, ymx, z2, t2d = ne.decode_device_gen(row)
        assert z2 == 2 and max(ypx, ymx, t2d) < ne.P  # Z = 1, every field canonical
    # Z = 0 anywhere: the generators are written exactly as without the normalisation
    bad = _gens(port, 50, 2, zero_z=(17,), **SPECIAL)
    dev, flag = harness.ingest_generators(bad)
    assert flag == 1
    with harness.options(normalize=0):
        assert np.array_equal(dev, harness.ingest_generators(bad)[0])


@pytest.mark.parametrize("ranges", [1, 3])
def test_device_call(port, ranges):
    cols = common.random_columns(np.random.default_rng(10 + ranges), N, SHAPES)
    gens = _gens(port, N, 20 + ranges, **SPECIAL)
    # the oracle sees the same points in their plain representation
    plain = ne.scaled_generators(port.ristretto_generators(N), 0, scale=False, **SPECIAL)
    want = port.commit(0, cols, plain)
    with harness.options(ranges=ranges, normalize=1):
        on = harness.commit(0, cols, gens)
    with harness.options(ranges=ranges, normalize=0):
        off = harness.commit(0, cols, gens)
    assert np.array_equal(on, want)
    assert np.array_equal(off, want)


@pytest.mark.parametrize("ranges", [1, 3])
@pytest.mark.parametrize("zero_at", [3, 280])  # in the first and in the last range
def test_zero_z_keeps_todays_bytes(port, ranges, zero_at):
    cols = common.random_columns(np.random.default_rng(30 + ranges), N, SHAPES)
    gens = _gens(port, N, 40 + zero_at, zero_z=(zero_at,), **SPECIAL)
    with harness.options(ranges=ranges, normalize=1):
        on = harness.commit(0, cols, gens)
    with harness.options(ranges=ranges, normalize=0):
        off = harness.commit(0, cols, gens)
    assert np.array_equal(on, off)


@pytest.mark.parametrize("ranges", [1, 3])
def test_offsets_call(port, ranges):
    cols = common.random_columns(np.random.default_rng(50 + ranges), N, SHAPES)
    offsets = [0, 400, 120, 37]
    total = max(o + N for o in offsets)
    gens = _gens(port, total, 60 + ranges, **SPECIAL)
    with harness.options(ranges=ranges, normalize=0):
        want = harness.commit_offsets(0, cols, offsets, gens)
    with harness.options(ranges=ranges, normalize=1):
        got = harness.commit_offsets(0, cols, offsets, gens)
    assert np.array_equal(got, want)
    # every column equals the device call over its own generators
    for j, off in enumerate(offsets):
        with harness.options(normalize=0):
            one = harness.commit(0, [cols[j]], np.ascontiguousarray(gens[off:off + N]))
        assert np.array_equal(got[j:j + 1], one), j
    bad = _gens(port, total, 70 + ranges, zero_z=(405,), **SPECIAL)
    with harness.options(ranges=ranges, normalize=1):
        bad_on = harness.commit_offsets(0, cols, offsets, bad)
    with harness.options(ranges=ranges, normalize=0):
        bad_off = harness.commit_offsets(0, cols, offsets, bad)
    assert np.array_equal(bad_on, bad_off)
