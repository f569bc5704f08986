"""Per-column generator offsets (b200_compute_pedersen_commitments_with_offsets and
b200_commit_device_with_offsets) through the CPU emulation of the kernel bodies: every column must
equal the oracle's commitment of that column alone, at its offset."""
import numpy as np
import pytest

from tests import common
from tests import commit_offsets_emul as eo

N = 120
# ragged unsigned / signed columns, one of them empty
SHAPES = [(0, 32, 0), (-37, 16, 1), (0, 8, 1), (-119, 5, 0), (-N, 4, 0), (-50, 1, 0)]


def lengths(shapes=SHAPES, n=N):
    return [max(0, n + d) for d, _, _ in shapes]


def offset_patterns(lens):
    adjacent = np.concatenate([[0], np.cumsum(lens)[:-1]]).tolist()
    return {
        "equal": [9] * len(lens),
        "overlapping": [0, 30, 60, 15, 100, 45][:len(lens)],
        "adjacent": adjacent,                               # every interval touches the next
        "disjoint": [0, 500, 200, 900, 1300, 700][:len(lens)],
    }


FAR = [1 << 33, 3, (1 << 33) + 50, 7, 1000, (1 << 33) - 60]  # built-in generators only


def oracle(port, curve, cols, offsets, gens):
    """k single-column commitments of the existing entry point, one per offset."""
    rows = []
    for col, off in zip(cols, offsets):
        if gens is None:
            rows.append(port.commit(0, [col], None, int(off)))
        else:
            rows.append(port.commit(curve, [col], gens[int(off):int(off) + col[0].shape[0]]))
    return np.concatenate(rows)


def columns(seed, shapes=SHAPES, n=N):
    return common.random_columns(np.random.default_rng(seed), n, shapes)


@pytest.fixture(autouse=True)
def default_options():
    eo.configure()
    yield
    eo.configure()


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
@pytest.mark.parametrize("pattern", ["equal", "overlapping", "adjacent", "disjoint"])
def test_explicit_generators(port, curve, pattern):
    cols = columns(10 * curve + len(pattern))
    offsets = offset_patterns(lengths())[pattern]
    gens, _ = common.generators_for(port, curve, max(o + n for o, n in zip(offsets, lengths())))
    got = eo.commit_offsets(curve, cols, offsets, gens)
    assert common.same(curve, got, oracle(port, curve, cols, offsets, gens))


@pytest.mark.parametrize("pattern", ["equal", "overlapping", "adjacent", "disjoint", "far"])
def test_builtin_generators(port, pattern):
    cols = columns(len(pattern))
    offsets = FAR if pattern == "far" else offset_patterns(lengths())[pattern]
    got = eo.commit_offsets(0, cols, offsets)
    assert np.array_equal(got, oracle(port, 0, cols, offsets, None))


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
def test_no_offsets_and_equal_offsets_match_the_existing_call(emul, port, curve):
    cols = columns(50 + curve)
    gens, _ = common.generators_for(port, curve, N + 40)
    assert np.array_equal(eo.commit_offsets(curve, cols, None, gens), emul.commit(curve, cols, gens))
    assert np.array_equal(eo.commit_offsets(curve, cols, [0] * len(cols), gens),
                          emul.commit(curve, cols, gens))
    assert np.array_equal(eo.commit_offsets(curve, cols, [40] * len(cols), gens),
                          emul.commit(curve, cols, gens[40:]))
    if curve == 0:
        assert np.array_equal(eo.commit_offsets(0, cols, None), emul.commit(0, cols))
        for off in (0, 17, 1 << 33):
            assert np.array_equal(eo.commit_offsets(0, cols, [off] * len(cols)),
                                  emul.commit(0, cols, None, off)), off


def test_only_empty_columns(port):
    cols = [(np.zeros((0, 4), np.uint8), 0), (np.zeros((0, 16), np.uint8), 1)]
    for curve in range(4):
        gens, _ = common.generators_for(port, curve, 1)
        got = eo.commit_offsets(curve, cols, [5, 1 << 40], gens if curve else None)
        assert common.same(curve, got, oracle(port, curve, cols, [5, 1 << 40], gens if curve else None))


@pytest.mark.parametrize("curve", [0, 2])
@pytest.mark.parametrize("ranges", [1, 2, 3, 4])
def test_upload_pieces(port, curve, ranges):
    """Each generator range ingests (or generates) only the packed positions its rows use."""
    cols = columns(70 + ranges)
    eo.configure(ranges=ranges)
    for pattern, offsets in offset_patterns(lengths()).items():
        gens, _ = common.generators_for(port, curve, max(o + n for o, n in zip(offsets, lengths())))
        got = eo.commit_offsets(curve, cols, offsets, gens)
        assert common.same(curve, got, oracle(port, curve, cols, offsets, gens)), pattern
    if curve == 0:
        got = eo.commit_offsets(0, cols, FAR)
        assert np.array_equal(got, oracle(port, 0, cols, FAR, None))


@pytest.mark.parametrize("curve", [0, 1])
def test_sort_passes_and_column_groups(port, curve):
    cols = columns(80 + curve)
    offsets = offset_patterns(lengths())["overlapping"]
    gens, _ = common.generators_for(port, curve, 300)
    want = oracle(port, curve, cols, offsets, gens)
    for range_entries, group_entries in ((300, 0), (0, 400), (500, 700)):
        eo.configure(range_entries=range_entries, group_entries=group_entries)
        got = eo.commit_offsets(curve, cols, offsets, gens)
        assert common.same(curve, got, want), (range_entries, group_entries)
        if curve == 0:
            got = eo.commit_offsets(0, cols, FAR)
            assert np.array_equal(got, oracle(port, 0, cols, FAR, None)), (range_entries, group_entries)


@pytest.mark.parametrize("policy", [1, 2, 0])
def test_builtin_table(port, policy):
    """Built-in intervals inside, straddling and beyond the precomputed range, table mode forced on,
    forced off and under the cost model."""
    cols = columns(90 + policy)
    for offsets in ([0, 30, 60, 15, 100, 45],   # inside
                    [0, 300, 60, 15, 100, 45],  # straddling (300 + 120 > 400)
                    [400, 500, 1000, 401, 2000, 450],  # beyond
                    FAR):
        eo.configure(table_policy=policy, num_builtin=400, window_bits=8)
        assert np.array_equal(eo.commit_offsets(0, cols, offsets),
                              oracle(port, 0, cols, offsets, None)), offsets
        eo.configure(ranges=3, table_policy=policy, num_builtin=400, window_bits=8)
        assert np.array_equal(eo.commit_offsets(0, cols, offsets),
                              oracle(port, 0, cols, offsets, None)), offsets


@pytest.mark.parametrize("curve", [1, 2, 3])
@pytest.mark.parametrize("levels", [0, 1, 3])
def test_pair_levels(port, curve, levels):
    eo.configure(pair_levels=levels)
    cols = columns(100 + curve, [(0, 32, 0), (-20, 16, 1), (0, 1, 0), (-N, 8, 0)])
    lens = lengths([(0, 32, 0), (-20, 16, 1), (0, 1, 0), (-N, 8, 0)])
    for offsets in ([0, 30, 60, 15], [0, 500, 200, 900]):
        gens, _ = common.generators_for(port, curve, max(o + n for o, n in zip(offsets, lens)) + 1)
        got = eo.commit_offsets(curve, cols, offsets, gens)
        assert common.same(curve, got, oracle(port, curve, cols, offsets, gens)), offsets
