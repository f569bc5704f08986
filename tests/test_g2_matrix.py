"""The G1 matrices' edge cases on the two G2 curves (4 bls12-381 G2, 5 bn254 G2), as check_*(entry,
curve) functions: this file runs the small cases under the CPU emulation of the kernel bodies, and
tests/test_gpu_g2_matrix.py runs every case through the C ABI on the GPU. Each docstring names the G1
test the case ports. Results are checked against closed forms over synthetic generators
G_i = k_i G: sum_i s_i G_i = (sum_i s_i k_i mod r) G, one oracle scalar multiplication per output
(tests/g2_reference.py, tests/bn254_g2_reference.py, behind the one interface of Oracle)."""
import contextlib

import numpy as np
import pytest

from tests import bn254_g2_reference, common
from tests import g2_reference
from tests.emul import harness
from tests.test_commit_offsets import columns, lengths, offset_patterns

CURVES = (4, 5)
# the set_tuning triples (window bits, level-1 chunk, later chunks) of test_skewed_digits_and_tuning
TUNINGS = [(2, 32, 8), (5, 7, 5), (8, 64, 4), (11, 16, 16), (13, 32, 8), (16, 32, 8), (19, 0, 8)]
# test_gpu_partition_msm's output widths and vlen lengths
WIDTHS = [1, 1, 1, 5, 1, 64, 256, 1, 13, 8, 1, 2]


def partition_lengths(n, w):
    return sorted(min(v, n) for v in [0, 1, max(w - 1, 0), w, w + 1, n, 2, n - 1, w, 3, n, n])


# ---- one interface over the two oracles ------------------------------------------------------------
class Oracle:
    """The G2 oracle of one curve id: closed forms, row edits, ABI structs and the compact
    (partition-table) entry, with the same names on both curves."""

    def __init__(self, curve):
        self.curve = curve
        if curve == 4:
            m = g2_reference
            self.commitment = m.compress
            self.edits = m.Edits
            self.W = 48  # bytes of one Fp component
        elif curve == 5:
            m = bn254_g2_reference.BN
            self.commitment = m.commitment
            self.edits = m.edits
            self.W = m.W
        else:
            raise ValueError(curve)
        self.R = m.R_ORDER
        self.scalar_mul, self.point_neg, self.closed_form = m.scalar_mul, m.point_neg, m.closed_form
        self.proj_struct, self.from_proj_struct = m.proj_struct, m.from_proj_struct
        self.fp2_to_mont_bytes = m.fp2_to_mont_bytes
        self.COMPACT = 4 * self.W

    def point(self, e):
        """(e mod r) G."""
        return self.scalar_mul(e % self.R)

    def compact(self, pt):
        """One compact partition-table entry {X, Y} (affine Montgomery limbs); the identity is
        X = 0 with its top 64 bits all ones, Y = 1 (compact_element::identity())."""
        if pt is None:
            return bytes(2 * self.W - 8) + b"\xff" * 8 + self.fp2_to_mont_bytes((1, 0))
        return self.fp2_to_mont_bytes(pt[0]) + self.fp2_to_mont_bytes(pt[1])

    def points(self, res):
        return [self.from_proj_struct(r) for r in res]


def logs(n, first=0):
    """The discrete logs k_i of synthetic generators first .. first + n - 1, as Python integers."""
    return [int.from_bytes(r.tobytes(), "little") for r in common.synth_scalars_k(n, first)]


def k_array(ints):
    """Python integers -> the uint64 [n, 4] logs the oracles' closed_form takes."""
    raw = b"".join(v.to_bytes(32, "little") for v in ints)
    return np.frombuffer(raw, dtype=np.uint64).reshape(len(ints), 4).copy()


def output_values(call):
    """The integer scalars of each output of a fixed-base call (the emulation's fixed_msm keywords:
    num_outputs, n, scalars and element_num_bytes, or output_bit_table [and output_lengths])."""
    m, n, sc = call["num_outputs"], call["n"], np.asarray(call["scalars"], dtype=np.uint8)
    rows = sc.reshape(n, -1)
    if call.get("output_bit_table") is None:
        b = call["element_num_bytes"]
        return [[int.from_bytes(r[j * b:(j + 1) * b].tobytes(), "little") for r in rows]
                for j in range(m)]
    whole = [int.from_bytes(r.tobytes(), "little") for r in rows]
    out, off = [], 0
    lens = call.get("output_lengths") or [n] * m
    for w, length in zip(call["output_bit_table"], lens):
        out.append([(v >> off) & ((1 << w) - 1) for v in whole[:length]])
        off += w
    return out


def expected_outputs(o, call, k):
    """The oracle's point of each output of a fixed-base call over generators with logs k."""
    return [o.point(sum(s * ki for s, ki in zip(vals, k))) for vals in output_values(call)]


def fixed_calls(rng, n, lens_max=None):
    """A fixed call (2 outputs x 32 bytes) and a vlen call over test_gpu_parity's bit table."""
    sc = rng.integers(0, 256, (n, 2 * 32), dtype=np.uint8)
    bt = [3, 1, 14, 64, 5, 200]
    psc = rng.integers(0, 256, (n, (sum(bt) + 7) // 8), dtype=np.uint8)
    lens = [1, 2, 17, min(40, n), min(50, n), n]
    return [dict(num_outputs=2, n=n, scalars=sc, element_num_bytes=32),
            dict(num_outputs=len(bt), n=n, scalars=psc, output_bit_table=bt, output_lengths=lens)]


def partition_calls(rng, n, w):
    """test_gpu_partition_msm's three calls: 2-byte fixed, packed and vlen over WIDTHS."""
    sc = rng.integers(0, 256, (n, 3 * 2), dtype=np.uint8)
    psc = rng.integers(0, 256, (n, (sum(WIDTHS) + 7) // 8), dtype=np.uint8)
    return [dict(num_outputs=3, n=n, scalars=sc, element_num_bytes=2),
            dict(num_outputs=len(WIDTHS), n=n, scalars=psc, output_bit_table=WIDTHS),
            dict(num_outputs=len(WIDTHS), n=n, scalars=psc, output_bit_table=WIDTHS,
                 output_lengths=partition_lengths(n, w))]


def assert_columns(o, got, cols, k):
    want = o.closed_form(cols, k)
    assert got.shape == want.shape, (got.shape, want.shape)
    bad = [j for j in range(len(cols)) if not np.array_equal(got[j], want[j])]
    assert not bad, f"columns {bad} differ from the closed form"


def assert_offset_columns(o, got, cols, offsets):
    """Column j against the closed form of that column alone, logs shifted by its offset."""
    for j, (col, off) in enumerate(zip(cols, offsets)):
        want = o.closed_form([col], common.synth_scalars_k(col[0].shape[0], int(off)))
        assert np.array_equal(got[j:j + 1], want), (j, off)


# ---- the emulation as an entry -----------------------------------------------------------------------
class EmulEntry:
    """The CPU emulation behind the names the checks use. options() takes the checks' vocabulary:
    ranges, window_bits, chunk1, chunkn, pair_levels (None: automatic), sort (the device's
    BLITZAR_B200_SORT; the emulation has one sort, so it takes only None), table_policy, table_window
    (None: no table), partition_policy."""
    SORTS = (None,)

    synth = staticmethod(harness.synth_generators)
    commit = staticmethod(harness.commit)
    commit_offsets = staticmethod(harness.commit_offsets)

    @staticmethod
    @contextlib.contextmanager
    def options(sort=None, pair_levels=None, table_window=None, **opts):
        assert sort is None, "the emulation has one sort"
        with harness.options(pair_levels=-1 if pair_levels is None else pair_levels,
                             table_window=table_window or 0, **opts):
            yield

    @staticmethod
    def fixed(curve, gens_p, call, partition_window=0):
        return harness.fixed_msm(curve, gens_p, partition_window=partition_window, **call)

    @staticmethod
    def partition_table(curve, gens_p, w, chunk_groups=0):
        return harness.partition_table(curve, gens_p, w, chunk_groups)


# ---- commitments ---------------------------------------------------------------------------------------
def check_edge_cases(entry, curve):
    """test_gpu_parity::test_edge_cases: common.edge_case_columns() (n = 1, signed extremes,
    2^256 - 1, an empty column, one loaded bucket) over 40 generators."""
    o = Oracle(curve)
    gens = entry.synth(curve, 40)
    cols = common.edge_case_columns()
    assert_columns(o, entry.commit(curve, cols, gens), cols, common.synth_scalars_k(40))


def check_random_sweep(entry, curve, n):
    """test_gpu_parity::test_random_sweep: the sweep's seven column shapes at n."""
    o = Oracle(curve)
    rng = np.random.default_rng(1000 * curve + n)
    gens = entry.synth(curve, n)
    cols = common.random_columns(rng, n, [(0, 32, 0), (-n // 3, 16, 1), (0, 8, 1), (0, 5, 0),
                                          (-(n - 1), 32, 0), (-n, 2, 0), (0, 1, 0)])
    assert_columns(o, entry.commit(curve, cols, gens), cols, common.synth_scalars_k(n))


def check_skewed_digits_and_tuning(entry, curve, n, tunings=TUNINGS):
    """test_gpu_parity::test_skewed_digits_and_tuning: a column of ones (every term in one bucket)
    and random columns under each window width and chunk shape."""
    o = Oracle(curve)
    rng = np.random.default_rng(8 + curve)
    gens = entry.synth(curve, n)
    ones = np.zeros((n, 2), dtype=np.uint8)
    ones[:, 0] = 1
    cols = [(ones, 0)] + common.random_columns(rng, n, [(0, 32, 0), (0, 4, 1)])
    want = o.closed_form(cols, common.synth_scalars_k(n))
    for c, k1, kn in tunings:
        with entry.options(window_bits=c, chunk1=k1, chunkn=kn):
            assert np.array_equal(entry.commit(curve, cols, gens), want), (c, k1, kn)


# ---- per-column offsets ----------------------------------------------------------------------------------
def check_offset_patterns(entry, curve):
    """test_gpu_commit_offsets::test_matrix: overlapping, touching, equal and disjoint offsets."""
    o = Oracle(curve)
    cols = columns(200 + curve)
    for pattern, offsets in offset_patterns(lengths()).items():
        gens = entry.synth(curve, max(off + m for off, m in zip(offsets, lengths())) + 1)
        got = entry.commit_offsets(curve, cols, offsets, gens)
        assert_offset_columns(o, got, cols, offsets)


def check_offset_sort_and_ranges(entry, curve, n):
    """test_gpu_commit_offsets::test_sort_paths_and_upload_pieces: each sort x 1 and 4 generator
    ranges (upload pieces), with intervals far apart, touching and nested."""
    o = Oracle(curve)
    shapes = [(0, 32, 0), (-n // 3, 16, 1), (0, 8, 1), (-(n - 1), 5, 0), (-n, 4, 0)]
    cols = columns(220 + curve, n=n, shapes=shapes)
    offsets = [0, n // 2, 4 * n // 3, 10, 77]
    gens = entry.synth(curve, max(off + m for off, m in zip(offsets, lengths(shapes, n))) + 1)
    for sort in entry.SORTS:
        for ranges in (1, 4):
            with entry.options(sort=sort, ranges=ranges):
                got = entry.commit_offsets(curve, cols, offsets, gens)
            assert_offset_columns(o, got, cols, offsets)


def check_offset_pair_levels(entry, curve, n):
    """test_gpu_commit_offsets::test_forced_pair_levels: pair levels 0, 1 and 3."""
    o = Oracle(curve)
    cols = columns(230 + curve, n=n, shapes=[(0, 32, 0), (-n // 4, 16, 1), (0, 1, 0)])
    offsets = [0, n // 3, 13 * n // 10]
    gens = entry.synth(curve, offsets[2] + n + 1)
    for levels in (0, 1, 3):
        with entry.options(pair_levels=levels):
            got = entry.commit_offsets(curve, cols, offsets, gens)
        assert_offset_columns(o, got, cols, offsets)


# ---- identity generators and cross-window collisions -------------------------------------------------------
def check_identity_generators(entry, curve, levels, n):
    """test_gpu_batch_affine::test_identity_generators: affine generators flagged infinity next to
    real points in the pair levels; then a handle whose projective generators have Z = 0, both as
    {0, 1, 0} and as the (X, Y, 0) an MSM writes for a cancelled sum, under table policy 1, 2, 0."""
    o = Oracle(curve)
    rng = np.random.default_rng(80 + curve)
    gens = entry.synth(curve, n).copy()
    ed = o.edits(gens)
    ident = [0, 7, 19, n - 1] + list(range(100, n, 13))
    ed.identity(ident)
    cols = common.random_columns(rng, n, [(0, 32, 0), (0, 2, 0), (-7, 16, 1)])
    cols.append((np.ones((n, 1), dtype=np.uint8), 0))
    with entry.options(pair_levels=levels):
        assert_columns(o, entry.commit(curve, cols, gens), cols, ed.k)
    gens_p = entry.synth(curve, n, 0, True).copy()
    k = logs(n)
    for j, i in enumerate(ident):
        if j % 2:
            gens_p[i, 4 * o.W:] = 0  # keep X and Y, Z = 0
        else:
            gens_p[i] = o.proj_struct(None)
        k[i] = 0
    sc = rng.integers(0, 256, (n, 2, 32), dtype=np.uint8)
    sc[:, 1] = 0
    sc[:, 1, 0] = 1
    call = dict(num_outputs=2, n=n, scalars=sc.reshape(n, 64), element_num_bytes=32)
    want = expected_outputs(o, call, k)
    for policy in (1, 2, 0):
        with entry.options(pair_levels=levels, table_policy=policy, table_window=10):
            assert o.points(entry.fixed(curve, gens_p, call)) == want, policy


def cross_window_generators(o, entry, curve, c, m=40):
    """common.cross_window_handle over G2: projective generators with G_1 = 2^c G_0, G_2 = -2^c G_0,
    G_4 = -2^c G_3, G_5 = 2^c G_3 (built by the oracle), and a call whose output 0 puts window 1 of
    G_0 (G_3) and window 0 of the other two in one bucket. Returns (generators, logs, call)."""
    gens_p = entry.synth(curve, m, 0, True).copy()
    k = logs(m)
    for i, plus, minus in ((0, 1, 2), (3, 5, 4)):
        for row, e in ((plus, k[i] << c), (minus, -(k[i] << c))):
            k[row] = e % o.R
            gens_p[row] = o.proj_struct(o.point(e))
    rng = np.random.default_rng(c + 10 * curve)
    sc = rng.integers(0, 256, (m, 2, 32), dtype=np.uint8)
    sc[:, 0] = 0

    def s32(v):
        return np.frombuffer(v.to_bytes(32, "little"), dtype=np.uint8)
    for rows, digit in (((0, 1, 2), 5), ((3, 4, 5), 9)):
        sc[rows[0], 0] = s32(digit << c)
        sc[rows[1], 0] = sc[rows[2], 0] = s32(digit)
    return gens_p, k, dict(num_outputs=2, n=m, scalars=sc.reshape(m, 64), element_num_bytes=32)


def check_cross_window_collisions(entry, curve, c):
    """test_gpu_batch_affine::test_table_cross_window_collisions: G_j = +-2^c G_i share a bucket of
    the table's one bucket set (a doubling and a cancellation), table forced on, at each pair-level
    count."""
    o = Oracle(curve)
    gens_p, k, call = cross_window_generators(o, entry, curve, c)
    want = expected_outputs(o, call, k)
    assert want[0] == o.point((5 * k[0] + 9 * k[3]) << c)  # G_1 and G_2 cancel, so do G_4 and G_5
    for levels in (None, 1, 2, 3):
        with entry.options(table_window=c, table_policy=1, pair_levels=levels):
            assert o.points(entry.fixed(curve, gens_p, call)) == want, levels


# ---- fixed-base tables and partition MSMs -----------------------------------------------------------------
def check_table_policies(entry, curve, m, windows=(10, 16, 20, None)):
    """test_gpu_parity::test_fixed_base_table_policies_agree: fixed and vlen calls with the table
    forced on, forced off and under the cost model, at each table window."""
    o = Oracle(curve)
    gens_p = entry.synth(curve, m, 0, True)
    k = logs(m)
    calls = fixed_calls(np.random.default_rng(90 + curve), m)
    wants = [expected_outputs(o, call, k) for call in calls]
    for window in windows:
        for policy in (1, 2, 0):
            with entry.options(table_window=window, table_policy=policy):
                for call, want in zip(calls, wants):
                    assert o.points(entry.fixed(curve, gens_p, call)) == want, (window, policy)


def check_partition_widths_and_policies(entry, curve, n=301, widths=(1, 3, 8, 16)):
    """test_gpu_partition_msm::test_widths_and_policies: fixed, packed and vlen calls answered with
    a partition table of each width, under each partition policy."""
    o = Oracle(curve)
    gens_p = entry.synth(curve, n, 0, True)
    k = logs(n)
    rng = np.random.default_rng(curve)
    for w in widths:
        calls = partition_calls(rng, n, w)
        wants = [expected_outputs(o, call, k) for call in calls]
        for policy in (0, 1, 2):
            with entry.options(partition_policy=policy):
                for call, want in zip(calls, wants):
                    assert o.points(entry.fixed(curve, gens_p, call, w)) == want, (w, policy)


def edited_generators(o, entry, curve, n=29):
    """partition_tables.edit_generators over G2: duplicates, G / -G pairs and identity rows, so that
    zero sums and identity sums fall in the middle of a w = 6 table. Returns (generators, logs)."""
    gens = entry.synth(curve, n, 0, True).copy()
    k = logs(n)

    def dup(dst, src):
        gens[dst], k[dst] = gens[src], k[src]

    def neg(i):
        gens[i] = o.proj_struct(o.point_neg(o.from_proj_struct(gens[i])))
        k[i] = (o.R - k[i]) % o.R

    def identity(rows):
        for i in rows:
            gens[i], k[i] = o.proj_struct(None), 0
    dup(1, 0)
    dup(3, 2)
    neg(3)
    identity([4])
    dup(7, 6)
    neg(7)
    dup(9, 8)
    identity([10, 11])
    identity(range(12, 18))
    for i in (19, 20, 21):
        dup(i, 18)
    neg(19)
    neg(21)
    dup(23, 5)
    return gens, k


def check_partition_degenerate(entry, curve):
    """test_gpu_partition_msm::test_degenerate_generators_and_scalars: duplicated, negated and
    identity generators; random, all-zero and all-ones scalars; widths 3 and 6, table forced."""
    o = Oracle(curve)
    n = 29
    gens_p, k = edited_generators(o, entry, curve, n)
    row = (sum(WIDTHS) + 7) // 8
    for w in (3, 6):
        for psc in (np.random.default_rng(w).integers(0, 256, (n, row), dtype=np.uint8),
                    np.zeros((n, row), np.uint8), np.full((n, row), 0xFF, np.uint8)):
            call = dict(num_outputs=len(WIDTHS), n=n, scalars=psc, output_bit_table=WIDTHS,
                        output_lengths=partition_lengths(n, w))
            with entry.options(partition_policy=1):
                got = entry.fixed(curve, gens_p, call, w)
            assert o.points(got) == expected_outputs(o, call, k), w


# ---- partition tables ------------------------------------------------------------------------------------
def check_partition_table_entries(entry, curve, n, w, samples=16):
    """test_gpu_partition_table (device table): sampled entries of the table of n projective
    generators (one of them the identity, one the negation of its neighbour) against the oracle's
    subset sums, byte for byte; k = 0, sums that cancel and groups padded past n hold the identity
    marker."""
    o = Oracle(curve)
    gens_p = entry.synth(curve, n, 0, True).copy()
    k = logs(n)
    gens_p[1], k[1] = o.proj_struct(None), 0
    gens_p[3] = o.proj_struct(o.point_neg(o.from_proj_struct(gens_p[2])))
    k[3] = (o.R - k[2]) % o.R
    table = entry.partition_table(curve, gens_p, w)
    groups = -(-n // w)
    assert table.size == groups * (o.COMPACT << w)
    table = table.reshape(-1, o.COMPACT)
    k += [0] * (groups * w - n)
    rng = np.random.default_rng(n + w)
    picks = [(0, 0), (0, (1 << w) - 1), (groups - 1, (1 << w) - 1)]
    picks += [(int(g), int(e)) for g, e in zip(rng.integers(0, groups, samples),
                                               rng.integers(0, 1 << w, samples))]
    pad = groups * w - n
    if pad:  # only padded rows of the last group: the identity
        picks.append((groups - 1, ((1 << pad) - 1) << (w - pad)))
    if w >= 4:  # G_2 + G_3 = O inside group 0
        picks.append((0, 0b1100))
    for g, e in picks:
        want = o.point(sum(k[g * w + j] for j in range(w) if e >> j & 1))
        assert table[(g << w) + e].tobytes() == o.compact(want), (g, e)


def check_partition_table_chunks(entry, curve, n=301, w=7):
    """test_gpu_partition_table::test_many_chunks_give_the_same_file: 1, 3 and 5 groups per chunk
    build the one-chunk table."""
    gens_p = entry.synth(curve, n, 0, True)
    one = entry.partition_table(curve, gens_p, w)
    for groups in (1, 3, 5):
        assert np.array_equal(entry.partition_table(curve, gens_p, w, groups), one), groups


# ---- under the emulation -----------------------------------------------------------------------------
@pytest.fixture
def entry():
    with harness.options():
        yield EmulEntry


def test_oracle_adapter_encodings():
    """Both oracles behind Oracle: the compact identity marker and entry width, the projective
    identity, and the closed form of one column."""
    for curve, compact in ((4, 192), (5, 128)):
        o = Oracle(curve)
        assert o.COMPACT == compact == len(o.compact(o.point(3))) == len(o.compact(None))
        assert o.compact(None)[o.COMPACT // 2 - 8:o.COMPACT // 2] == b"\xff" * 8
        assert o.from_proj_struct(o.proj_struct(None)) is None
        assert o.points([o.proj_struct(o.point(5), (3, 4))]) == [o.point(5)]
        col = (np.array([[2], [3]], dtype=np.uint8), 0)
        k = k_array([7, o.R - 1])
        assert bytes(o.closed_form([col], k)[0]) == bytes(o.commitment(o.point(14 - 3)))


@pytest.mark.parametrize("curve", CURVES)
def test_commitments(entry, curve):
    check_edge_cases(entry, curve)
    for n in (1, 31, 257):
        check_random_sweep(entry, curve, n)
    check_skewed_digits_and_tuning(entry, curve, 300, TUNINGS[:4])


@pytest.mark.parametrize("curve", CURVES)
def test_offsets(entry, curve):
    check_offset_patterns(entry, curve)
    check_offset_sort_and_ranges(entry, curve, 300)
    check_offset_pair_levels(entry, curve, 200)


@pytest.mark.parametrize("curve", CURVES)
def test_identity_generators_and_cross_window_collisions(entry, curve):
    check_identity_generators(entry, curve, 3, 300)
    check_cross_window_collisions(entry, curve, 10)


@pytest.mark.parametrize("curve", CURVES)
def test_table_policies_and_partition_msms(entry, curve):
    check_table_policies(entry, curve, 120, windows=(10, None))
    check_partition_widths_and_policies(entry, curve, 61, (1, 3, 8))
    check_partition_degenerate(entry, curve)


@pytest.mark.parametrize("curve", CURVES)
def test_partition_tables(entry, curve):
    for n in (37, 301):
        for w in (1, 3, 7):
            check_partition_table_entries(entry, curve, n, w)
    check_partition_table_chunks(entry, curve)
