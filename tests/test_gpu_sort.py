"""Binned bucket sort of the (term, window) entries (blitzar_b200/csrc/msm.cuh, BinSortBody and the
kernels before it) against the atomic count + scan + scatter, on the device.

b200_selftest_sort runs both sorts over the same device columns and counts the buckets whose end
offset or entry multiset differ. The commitment tests run whole MSMs with the sort forced to each path
(BLITZAR_B200_SORT, read on every call) and compare them with the C oracle port."""
import numpy as np
import pytest

from tests import common

pytestmark = pytest.mark.gpu
CAP = 8192  # kBinCap: entries of a bin sorted in shared memory


def _selftest(bb, columns, window_bits=0):
    bufs = [bb.DeviceBuffer(host=np.ascontiguousarray(a)) for a, _ in columns]
    shapes = [(a.shape[0], a.shape[1], s) for a, s in columns]
    try:
        return bb.selftest_sort(shapes, [b.ptr for b in bufs], window_bits)
    finally:
        for b in bufs:
            b.free()


def _u16(values):
    return np.ascontiguousarray(np.asarray(values, dtype="<u2").view(np.uint8).reshape(-1, 2))


def _shapes():
    rng = np.random.default_rng(5)
    n = 1 << 20
    c2 = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    c2[:, 31] &= 0x0F  # 252-bit: the top window is 8x denser than the others
    one_hot = []
    for j in range(8):
        a = np.zeros((4096, 32), dtype=np.uint8)
        a[rng.integers(0, 4096), rng.integers(0, 32)] = 1 << j
        one_hot.append((a, 0))
    # window 0 of c = 16: bucket 999 holds exactly CAP entries and bucket 1999 CAP + 1, so that one
    # micro-bin is sorted in shared memory at the limit and one out of global memory just above it
    vals = rng.integers(1, 1 << 15, 1 << 17)
    vals[((vals >= 993) & (vals <= 1004)) | ((vals >= 1993) & (vals <= 2004))] = 5  # rest of the micro-bins
    vals[:CAP] = 1000
    vals[CAP:2 * CAP + 1] = 2000
    rng.shuffle(vals)
    return {
        "c2_252bit": ([(c2, 0)], 0),
        "all_zero": ([(np.zeros((1 << 16, 32), dtype=np.uint8), 0)], 0),
        "boolean": ([(rng.integers(0, 2, (n, 1), dtype=np.uint8), 0)], 0),
        "one_hot": (one_hot, 0),
        "below_2_16": ([(rng.integers(0, 256, (1 << 18, 2), dtype=np.uint8), 0)], 0),
        "signed": ([(rng.integers(0, 256, (1 << 16, 8), dtype=np.uint8), 1),
                    (rng.integers(0, 256, (1 << 16, 32), dtype=np.uint8), 1)], 0),
        "cap_and_cap_plus_1": ([(_u16(vals), 0)], 16),
        "columns_64": ([(rng.integers(0, 256, (1 << 14, 32), dtype=np.uint8), 0) for _ in range(64)], 0),
        "window_20": ([(rng.integers(0, 256, (1 << 16, 32), dtype=np.uint8), 0)], 20),
    }


@pytest.mark.parametrize("name", list(_shapes()))
def test_binned_sort_matches_atomic_sort(bb, name):
    columns, c = _shapes()[name]
    assert _selftest(bb, columns, c) == 0


@pytest.mark.parametrize("path", ["0", "2"])
def test_commitments_on_both_sort_paths(bb, port, monkeypatch, path):
    """Whole MSMs per sort path against the oracle: random, signed and narrow columns, a boolean column,
    built-in generators (the fixed-base table of sxt_init), and a 4-piece host call."""
    monkeypatch.setenv("BLITZAR_B200_SORT", path)
    rng = np.random.default_rng(11)
    n = 1500
    cols = [(rng.integers(0, 256, (n, 32), dtype=np.uint8), 0),
            (rng.integers(0, 256, (n - 7, 8), dtype=np.uint8), 1),
            (rng.integers(0, 2, (n, 1), dtype=np.uint8), 0),
            (np.zeros((n, 4), dtype=np.uint8), 0)]
    for curve in (0, 1, 2):
        gens, _ = common.generators_for(port, curve, n)
        want = port.commit(curve, cols, gens)
        assert common.same(curve, bb.compute_pedersen_commitments(curve, cols, gens), want), curve
    assert np.array_equal(bb.compute_pedersen_commitments(0, cols[:2], None, 3)[:, :32],
                          port.commit(0, cols[:2], None, 3)[:, :32])
    monkeypatch.setenv("BLITZAR_B200_RANGES", "4")
    gens, _ = common.generators_for(port, 0, n)
    assert common.same(0, bb.compute_pedersen_commitments(0, cols, gens), port.commit(0, cols, gens))


@pytest.mark.parametrize("levels", ["0", "1", "3", "6"])
def test_weierstrass_pair_levels_on_binned_path(bb, port, monkeypatch, levels):
    """The binned sort serves the unpadded layout (no pair level); padded passes keep the atomic sort.
    Both must give the oracle's commitments when the binned path is requested."""
    monkeypatch.setenv("BLITZAR_B200_SORT", "2")
    monkeypatch.setenv("BLITZAR_B200_PAIR_LEVELS", levels)
    rng = np.random.default_rng(12)
    n = 1500
    cols = [(rng.integers(0, 256, (n, 32), dtype=np.uint8), 0)]
    for curve in (1, 2):
        gens, _ = common.generators_for(port, curve, n)
        assert common.same(curve, bb.compute_pedersen_commitments(curve, cols, gens),
                           port.commit(curve, cols, gens)), curve
