"""Pipeline logic on CPU: the product's kernel bodies run as serial host loops (tests/emul) and
must agree bit-for-bit with the oracle. Mirrors the reference's shared conformance suite
(sxt/multiexp/test/multiexponentiation.cc:42-451) and ABI tests (cbindings/pedersen.t.cc:243-612,
cbindings/fixed_pedersen.t.cc:45-200)."""
import numpy as np
import pytest

from tests import common


def test_golden_commitments(emul):
    assert emul.commit(0, common.golden_columns()).tolist() == common.GOLDEN_COMMITMENTS


def test_builtin_generators(emul, port):
    g = emul.get_generators(9, 123)
    assert np.array_equal(port.normalize(0, g), port.normalize(0, port.ristretto_generators(9, 123)))


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
def test_edge_cases_all_curves(emul, port, curve):
    gens, _ = common.generators_for(port, curve, 40)
    cols = common.edge_case_columns()
    assert common.same(curve, emul.commit(curve, cols, gens), port.commit(curve, cols, gens))


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
def test_random_ragged_signed_columns(emul, port, curve):
    rng = np.random.default_rng(100 + curve)
    n = 700
    gens, _ = common.generators_for(port, curve, n)
    cols = common.random_columns(rng, n, [(0, 32, 0), (-13, 16, 1), (0, 8, 1), (-1, 5, 0),
                                          (-699, 32, 0), (-700, 2, 0), (0, 1, 0)])
    assert common.same(curve, emul.commit(curve, cols, gens), port.commit(curve, cols, gens))


@pytest.mark.parametrize("window_bits", [2, 3, 5, 7, 8, 11, 13, 16, 18, 20])
def test_every_window_width(emul, port, window_bits):
    rng = np.random.default_rng(window_bits)
    n = 300
    gens, _ = common.generators_for(port, 0, n)
    cols = common.random_columns(rng, n, [(0, 32, 0), (-3, 4, 1), (0, 7, 0)])
    with emul.options(window_bits=window_bits):
        got = emul.commit(0, cols, gens)
    assert common.same(0, got, port.commit(0, cols, gens))


@pytest.mark.parametrize("chunks", [(4, 4), (5, 4), (7, 5), (32, 8), (64, 16)])
def test_cascade_chunk_shapes_and_skew(emul, port, chunks):
    """Heavily skewed digits (all terms in one bucket) drive the multi-level cascade."""
    rng = np.random.default_rng(5)
    n = 900
    gens, _ = common.generators_for(port, 0, n)
    skew = np.full((n, 2), 0, dtype=np.uint8)
    skew[:, 0] = 1
    two = np.zeros((n, 4), dtype=np.uint8)
    two[:, 0] = rng.integers(1, 3, n)
    cols = [(skew, 0), (two, 0)] + common.random_columns(rng, n, [(0, 32, 0)])
    with emul.options(chunk1=chunks[0], chunkn=chunks[1]):
        got = emul.commit(0, cols, gens)
    assert common.same(0, got, port.commit(0, cols, gens))


def test_homomorphism(emul, port):
    """cbindings/pedersen.t.cc:287-316: commit(a) + commit(b) == commit(a + b)."""
    rng = np.random.default_rng(9)
    n = 64
    a = rng.integers(0, 2**31, n, dtype=np.uint64)
    b = rng.integers(0, 2**31, n, dtype=np.uint64)
    cols = [(x.astype("<u8").view(np.uint8).reshape(n, 8), 0) for x in (a, b, a + b)]
    gens, _ = common.generators_for(port, 0, n)
    parts = emul.commit_partial(0, cols[:2], gens)
    summed = emul.combine_partials(0, parts.reshape(2, -1), 2, 1)
    assert np.array_equal(summed[0], emul.commit(0, cols[2:], gens)[0])


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
def test_fixed_packed_vlen(emul, port, curve):
    rng = np.random.default_rng(40 + curve)
    m = 50
    _, gens_p = common.generators_for(port, curve, m)
    sc = rng.integers(0, 256, (m, 3 * 6), dtype=np.uint8)
    a = emul.fixed_msm(curve, gens_p, 3, m, sc, element_num_bytes=6)
    b = port.fixed_msm(curve, gens_p, 3, m, sc, element_num_bytes=6)
    assert common.same(curve, port.normalize(curve, a), port.normalize(curve, b))
    bt = [3, 1, 14, 9, 64, 5]
    row = (sum(bt) + 7) // 8
    psc = rng.integers(0, 256, (m, row), dtype=np.uint8)
    a = emul.fixed_msm(curve, gens_p, len(bt), m, psc, output_bit_table=bt)
    b = port.fixed_msm(curve, gens_p, len(bt), m, psc, output_bit_table=bt)
    assert common.same(curve, port.normalize(curve, a), port.normalize(curve, b))
    lens = [1, 2, 17, 17, 40, 50]
    a = emul.fixed_msm(curve, gens_p, len(bt), m, psc, output_bit_table=bt, output_lengths=lens)
    b = port.fixed_msm(curve, gens_p, len(bt), m, psc, output_bit_table=bt, output_lengths=lens)
    assert common.same(curve, port.normalize(curve, a), port.normalize(curve, b))


def test_reference_fixed_pedersen_vectors(emul, port):
    """cbindings/fixed_pedersen.t.cc:121-135: packed {0b1010, 0b0101}, table {3,1}."""
    g = port.ristretto_generators(2, 0)
    res = emul.fixed_msm(0, g, 2, 2, np.array([0b1010, 0b0101], dtype=np.uint8),
                         output_bit_table=[3, 1])
    want = port.commit(0, [(np.array([[2], [5]], dtype=np.uint8), 0),
                           (np.array([[1], [0]], dtype=np.uint8), 0)], g)
    assert np.array_equal(port.normalize(0, res), want)


def test_identity_generators_weierstrass(emul, port):
    """Affine inputs flagged `infinity` are the group identity (element_affine::identity())."""
    rng = np.random.default_rng(3)
    for curve in (1, 2, 3):
        gens, _ = common.generators_for(port, curve, 20)
        gens = gens.copy()
        stride = gens.shape[1]
        flag = {1: 96, 2: 64, 3: 64}[curve]
        for i in (0, 7, 19):
            gens[i, :] = 0
            gens[i, flag] = 1
        cols = common.random_columns(rng, 20, [(0, 32, 0), (0, 2, 0)])
        assert stride in (72, 104)
        assert common.same(curve, emul.commit(curve, cols, gens), port.commit(curve, cols, gens))


@pytest.mark.parametrize("levels", [-1, 1, 3, 6])
def test_identity_generators_in_pair_levels(emul, port, levels):
    """Identity generators as operands of the batch-affine pair levels (a column of ones pairs them
    with real points), and projective handle generators with Z = 0, with and without the table."""
    rng = np.random.default_rng(4)
    with emul.options(pair_levels=levels):
        for curve in (1, 2, 3):
            gens, gens_p = common.generators_for(port, curve, 20)
            gens, gens_p = gens.copy(), gens_p.copy()
            common.set_identity(curve, gens, [0, 7, 19])
            cols = common.random_columns(rng, 20, [(0, 32, 0), (0, 2, 0)])
            cols.append((np.ones((20, 1), dtype=np.uint8), 0))
            assert common.same(curve, emul.commit(curve, cols, gens), port.commit(curve, cols, gens))
            common.set_identity(curve, gens_p, [0, 7, 19])
            sc = rng.integers(0, 256, (20, 2 * 32), dtype=np.uint8)
            sc[:, 32:] = 0
            sc[:, 32] = 1
            want = port.normalize(curve, port.fixed_msm(curve, gens_p, 2, 20, sc, element_num_bytes=32))
            for table in (0, 10):
                emul.configure(pair_levels=levels, table_window=table,
                               table_policy=1 if table else 0)
                got = emul.fixed_msm(curve, gens_p, 2, 20, sc, element_num_bytes=32)
                assert common.same(curve, port.normalize(curve, got), want), (curve, table)


@pytest.mark.parametrize("curve", [0, 2])
@pytest.mark.parametrize("num_ranges", [2, 3, 7])
def test_generator_ranges_share_one_bucket_array(emul, port, curve, num_ranges):
    """The copy-overlap path: the generator range is processed in pieces that add into one bucket
    array (ragged columns make some pieces empty for some columns)."""
    rng = np.random.default_rng(curve * 10 + num_ranges)
    n = 500
    gens, _ = common.generators_for(port, curve, n)
    cols = common.random_columns(rng, n, [(0, 32, 0), (-300, 16, 1), (-499, 4, 0), (0, 1, 0)])
    with emul.options(ranges=num_ranges):
        got = emul.commit(curve, cols, gens)
        got_builtin = emul.commit(0, cols[:2], None, 5) if curve == 0 else None
    assert common.same(curve, got, port.commit(curve, cols, gens))
    if got_builtin is not None:
        assert common.same(0, got_builtin, port.commit(0, cols[:2], None, 5))




def test_column_groups_with_generator_ranges(emul, port):
    """Several column groups (forced small) each make a full pass over generators that arrive in
    pieces."""
    rng = np.random.default_rng(12)
    n = 400
    gens, _ = common.generators_for(port, 0, n)
    cols = common.random_columns(rng, n, [(0, 32, 0), (-100, 16, 1), (0, 8, 0), (-399, 32, 0), (0, 4, 0)])
    with emul.options(ranges=3, group_entries=4000):
        got = emul.commit(0, cols, gens)
        got_builtin = emul.commit(0, cols, None, 9)
    assert common.same(0, got, port.commit(0, cols, gens))
    assert common.same(0, got_builtin, port.commit(0, cols, None, 9))


def test_long_columns_split_into_sort_passes(emul, port):
    """A column whose (term, window) entries exceed one sort pass is processed as several generator
    ranges automatically (limit forced small here; 2^31 in production)."""
    rng = np.random.default_rng(13)
    n = 600
    gens, _ = common.generators_for(port, 2, n)
    cols = common.random_columns(rng, n, [(0, 32, 0), (-250, 8, 1)])
    with emul.options(range_entries=3000):
        got = emul.commit(2, cols, gens)
    assert common.same(2, got, port.commit(2, cols, gens))


# ---- fixed-base tables (2^(c w) G_i, shared bucket set) ----------------------------------------------
@pytest.mark.parametrize("curve", [0, 2])
@pytest.mark.parametrize("window_bits", [10, 16, 19])
def test_fixed_base_table_mode(emul, port, curve, window_bits):
    """Replaces mtxpp2's partition table (sxt/multiexp/pippenger2/partition_table.h:36-98): every
    window's multiple of every generator is tabulated, all windows share one bucket set. Same results
    as the oracle for fixed-width, packed and variable-length calls."""
    rng = np.random.default_rng(40 + curve + window_bits)
    m = 400
    _, gens_p = common.generators_for(port, curve, m)
    with emul.options(table_window=window_bits, table_policy=1):
        sc = rng.integers(0, 256, (m, 2 * 32), dtype=np.uint8)
        a = emul.fixed_msm(curve, gens_p, 2, m, sc, element_num_bytes=32)
        b = port.fixed_msm(curve, gens_p, 2, m, sc, element_num_bytes=32)
        assert common.same(curve, port.normalize(curve, a), port.normalize(curve, b))
        bt = [3, 1, 14, 9, 64, 5, 200]
        psc = rng.integers(0, 256, (m, (sum(bt) + 7) // 8), dtype=np.uint8)
        lens = [1, 2, 17, 17, 40, 50, 400]
        a = emul.fixed_msm(curve, gens_p, len(bt), m, psc, output_bit_table=bt, output_lengths=lens)
        b = port.fixed_msm(curve, gens_p, len(bt), m, psc, output_bit_table=bt, output_lengths=lens)
        assert common.same(curve, port.normalize(curve, a), port.normalize(curve, b))
        # cost model: short columns fall back to the variable-base run
        emul.configure(table_window=window_bits, table_policy=0)
        a = emul.fixed_msm(curve, gens_p, len(bt), m, psc, output_bit_table=bt)
        b = port.fixed_msm(curve, gens_p, len(bt), m, psc, output_bit_table=bt)
        assert common.same(curve, port.normalize(curve, a), port.normalize(curve, b))


def test_builtin_generator_table(emul, port):
    """sxt_config::num_precomputed_generators with the fixed-base table: commitments over the built-in
    generators inside, straddling and beyond the table."""
    rng = np.random.default_rng(77)
    cols = common.random_columns(rng, 300, [(0, 32, 0), (-100, 16, 1), (0, 1, 0), (-299, 8, 0)])
    for c in (0, 12):
        with emul.options(num_builtin=400, builtin_window=c, table_policy=1 if c else 0):
            for off in (0, 37, 100, 250):
                assert np.array_equal(emul.commit(0, cols, None, off), port.commit(0, cols, None, off))


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
def test_generators_from_reference_partition_table_file(emul, port, curve):
    """tests/golden/ref_table_curve{c}_w3.bin was written by the reference's own code (oracle/_ref,
    tests/golden/make_table_files.py) for 7 generators; the reader recovers them (padded with
    identities to a multiple of the window width)."""
    import os
    here = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    want = np.load(os.path.join(here, f"fixed_curve{curve}.npz"))["generators_p"][:7]
    got = emul.generators_from_reference_table(curve, os.path.join(here, f"ref_table_curve{curve}_w3.bin"))
    assert got.shape[0] == 9
    assert common.same(curve, port.normalize(curve, got[:7]), port.normalize(curve, want))
    ident = port.normalize(curve, got[7:])
    zero = port.commit(curve, [(np.zeros((0, 4), dtype=np.uint8), 0)] * 2,
                       common.generators_for(port, curve, 1)[0])
    assert common.same(curve, ident, zero)


def test_window_major_scatter_option(emul, port):
    """The (measured-slower, off by default) window-major scatter sorts the same entries."""
    rng = np.random.default_rng(15)
    n = 500
    gens, _ = common.generators_for(port, 0, n)
    cols = common.random_columns(rng, n, [(0, 32, 0), (-13, 16, 1), (0, 8, 1), (-499, 32, 0), (0, 1, 0)])
    with emul.options(scatter_window_major=1):
        assert common.same(0, emul.commit(0, cols, gens), port.commit(0, cols, gens))


@pytest.mark.parametrize("curve", [1, 2, 3])
def test_batch_affine_pair_levels(emul, port, curve):
    """Weierstrass accumulation through L batch-affine pair levels (padded buckets, fused passes, the
    inversion tree with its Euclid top) for several window widths / levels / batch sizes, on generators
    with duplicates and negations (doublings, cancellations, identity operands inside the pair levels)."""
    rng = np.random.default_rng(50 + curve)
    n = 600
    gens, _ = common.generators_for(port, curve, n)
    gens[1::7] = gens[0]
    cols = common.random_columns(rng, n, [(0, 32, 0), (-13, 16, 1), (0, 2, 0)])
    ones = np.full((n, 1), 3, dtype=np.uint8)
    sg = np.zeros((n, 1), dtype=np.uint8)
    sg[::2], sg[1::2] = 1, 0xFF  # +1 / -1 alternating: P + (-P) on the duplicated generators
    cols += [(ones, 0), (sg, 1)]
    want = port.commit(curve, cols, gens)
    for c, levels, batch in ((4, 1, 4), (4, 3, 5), (6, 2, 32), (3, 5, 0), (2, 6, 64), (0, 6, 1)):
        with emul.options(window_bits=c, pair_levels=levels, pair_batch=batch):
            assert common.same(curve, emul.commit(curve, cols, gens), want), (c, levels, batch)
    # later ranges: scratch buckets + merge with padded layouts
    with emul.options(ranges=3, window_bits=4, pair_levels=2, pair_batch=8):
        assert common.same(curve, emul.commit(curve, cols, gens), want)


@pytest.mark.parametrize("curve", [1, 2, 3])
def test_degenerate_pair_level_buckets(emul, port, curve):
    """Buckets of nothing but copies of +-P, identities and (bls12-381) the x = 0 points (0, +-2)
    through every number of pair levels: doublings, cancellations and identity operands at every
    level, in the fused next-level classification and in the rare-path gather of pass 1."""
    gens, cols, equal = common.degenerate_buckets(port, curve)
    want = port.commit(curve, cols, gens)
    for j, m in equal:
        assert common.same(curve, want[j:j + 1],
                           port.commit(curve, [(np.array([[m]], dtype=np.uint8), 0)], gens[:1])), m
    for levels in (-1, 1, 2, 3, 4, 5, 6):
        with emul.options(pair_levels=levels):
            assert common.same(curve, emul.commit(curve, cols, gens), want), levels


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
@pytest.mark.parametrize("window_bits", [10, 16])
def test_fixed_base_table_cross_window_collisions(emul, port, curve, window_bits):
    """Table mode shares one bucket set over all windows, so with G_j = +-2^c G_i window 1 of i and
    window 0 of j meet in one bucket with equal x: doublings and cancellations inside the pair levels
    (ristretto255, with complete formulas and no pair levels, is the control)."""
    gens_p, sc = common.cross_window_handle(port, curve, window_bits)
    m = gens_p.shape[0]
    want = port.normalize(curve, port.fixed_msm(curve, gens_p, 2, m, sc, element_num_bytes=32))
    for levels in (-1, 1, 2, 3):
        with emul.options(table_window=window_bits, table_policy=1, pair_levels=levels):
            got = emul.fixed_msm(curve, gens_p, 2, m, sc, element_num_bytes=32)
            assert common.same(curve, port.normalize(curve, got), want), levels


@pytest.mark.parametrize("curve", [1, 2, 3])
def test_edited_synthetic_generators_keep_the_closed_form(emul, port, curve):
    """Duplicated, negated and identity rows of synthetic generators, with their discrete logs kept
    in step (the bookkeeping of the full-size device test), still give the closed form."""
    n = 400
    gens = emul.synth_generators(curve, n)
    ed = common.GeneratorEdits(curve, gens)
    rng = np.random.default_rng(curve)
    s = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    rows = np.arange(16, n, 16)
    ed.duplicate(rows, rows - 1)
    s[rows] = s[rows - 1]
    ed.duplicate(rows[:-1] + 1, rows[:-1])
    ed.negate(rows[:-1] + 1)
    s[rows[:-1] + 1] = s[rows[:-1]]
    ed.duplicate(slice(200, 264), 200)
    s[200:264] = 0
    s[200:264, 0] = 1
    ed.identity(slice(5, n, 31))
    want = port.commit(curve, [(s, 0)], gens)
    assert common.same(curve, common.closed_form_commitment(port, curve, s, k=ed.k), want)
    with emul.options(pair_levels=2):
        assert common.same(curve, emul.commit(curve, [(s, 0)], gens), want)
