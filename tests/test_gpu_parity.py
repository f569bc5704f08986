"""Parity tests proper: the CUDA path, called through the C ABI (ctypes mirror in
blitzar_b200/api.py), against the oracle on the same seeded inputs. Bit-exact: every output of
this path is integer / byte data. Modelled on cbindings/pedersen.t.cc:243-612,
cbindings/fixed_pedersen.t.cc:45-200, get_generators.t.cc, get_one_commit.t.cc and the shared
conformance suite sxt/multiexp/test/multiexponentiation.cc:42-451."""
import os
import tempfile

import numpy as np
import pytest

from tests import common, test_gpu_commit_offsets

pytestmark = pytest.mark.gpu


def test_native_library_is_loaded(bb):
    import blitzar_b200.api as api
    maps = open("/proc/self/maps").read()
    assert "libblitzar_b200.so" in maps
    assert api.launch_count() > 0  # sxt_init precomputed generators with our kernel


def test_reference_golden_commitments(bb):
    out = bb.compute_pedersen_commitments(0, common.golden_columns())
    assert out.tolist() == common.GOLDEN_COMMITMENTS


def test_committed_reference_fixtures(bb, port):
    for curve in range(4):
        z = np.load(os.path.join(common.GOLDEN, f"commit_curve{curve}.npz"))
        cols = [(z[f"col{j}"], int(z["signed"][j])) for j in range(len(z["signed"]))]
        out = bb.compute_pedersen_commitments(curve, cols, z["generators"])
        assert common.same(curve, out, z["commitments"]), curve
        f = np.load(os.path.join(common.GOLDEN, f"fixed_curve{curve}.npz"))
        h = bb.MultiexpHandle(curve, f["generators_p"])
        res = h.fixed_multiexponentiation(int(f["element_num_bytes"]), int(f["num_outputs"]),
                                          int(f["n"]), f["scalars"])
        assert common.same(curve, port.normalize(curve, res), f["normalized"]), curve
        res = h.fixed_packed_multiexponentiation(f["bit_table"].tolist(), int(f["n"]),
                                                 f["packed_scalars"])
        assert common.same(curve, port.normalize(curve, res), f["packed_normalized"]), curve
        h.free()


def test_num_sequences_zero_is_a_noop(bb):
    out = bb.compute_pedersen_commitments(0, [])
    assert out.shape[0] == 0


def test_get_generators_and_one_commit(bb, port):
    g = bb.get_generators(70, 60)  # straddles the 64 precomputed generators
    assert np.array_equal(port.normalize(0, g), port.normalize(0, port.ristretto_generators(70, 60)))
    for n in (0, 1, 5, 200):
        one = bb.get_one_commit(n)
        ones = np.ones((n, 1), dtype=np.uint8)
        want = port.commit(0, [(ones, 0)], None, 0)
        assert np.array_equal(port.normalize(0, one), want), n


def test_generator_offset(bb, port):
    rng = np.random.default_rng(4)
    cols = common.random_columns(rng, 90, [(0, 8, 0), (-3, 32, 0)])
    for offset in (0, 17, 1 << 33):
        got = bb.compute_pedersen_commitments(0, cols, None, offset)
        assert np.array_equal(got, port.commit(0, cols, None, offset)), offset


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
def test_edge_cases(bb, port, curve):
    gens, _ = common.generators_for(port, curve, 40)
    cols = common.edge_case_columns()
    assert common.same(curve, bb.compute_pedersen_commitments(curve, cols, gens),
                       port.commit(curve, cols, gens))


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
@pytest.mark.parametrize("n", [1, 31, 257, 4099, 20000])
def test_random_sweep(bb, port, curve, n):
    rng = np.random.default_rng(1000 * curve + n)
    gens, _ = common.generators_for(port, curve, n)
    cols = common.random_columns(rng, n, [(0, 32, 0), (-n // 3, 16, 1), (0, 8, 1), (0, 5, 0),
                                          (-(n - 1), 32, 0), (-n, 2, 0), (0, 1, 0)])
    assert common.same(curve, bb.compute_pedersen_commitments(curve, cols, gens),
                       port.commit(curve, cols, gens))


def test_skewed_digits_and_tuning(bb, port):
    """All terms in one bucket; every window width; odd chunk shapes (cascade depth)."""
    rng = np.random.default_rng(8)
    n = 6000
    gens, _ = common.generators_for(port, 0, n)
    ones = np.zeros((n, 2), dtype=np.uint8)
    ones[:, 0] = 1
    cols = [(ones, 0)] + common.random_columns(rng, n, [(0, 32, 0), (0, 4, 1)])
    want = port.commit(0, cols, gens)
    try:
        for c, k1, kn in [(2, 32, 8), (5, 7, 5), (8, 64, 4), (11, 16, 16), (13, 32, 8), (16, 32, 8), (19, 0, 8)]:
            bb.set_tuning(c, k1, kn)
            assert np.array_equal(bb.compute_pedersen_commitments(0, cols, gens), want), (c, k1, kn)
    finally:
        bb.set_tuning()


def test_homomorphism_through_partials(bb, port):
    """cbindings/pedersen.t.cc:287-316 with the point addition done by the combine entry point."""
    rng = np.random.default_rng(9)
    n = 3000
    a = rng.integers(0, 2**62, n, dtype=np.uint64)
    b = rng.integers(0, 2**62, n, dtype=np.uint64)
    cols = [(x.astype("<u8").view(np.uint8).reshape(n, 8), 0) for x in (a, b, a + b)]
    gens, _ = common.generators_for(port, 0, n)
    dg = bb.DeviceBuffer(host=gens)
    ds = [bb.DeviceBuffer(host=c[0]) for c in cols]
    pb = 128
    parts = bb.DeviceBuffer(2 * pb)
    bb.commit_device(0, [(n, 8, 0)] * 2, [ds[0].ptr, ds[1].ptr], dg.ptr, None, parts.ptr)
    out = bb.DeviceBuffer(32)
    bb.combine_partials_device(0, out.ptr, parts.ptr, 2, 1)
    want = bb.compute_pedersen_commitments(0, cols[2:], gens)
    assert np.array_equal(out.to_host()[:32], want[0])


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
def test_fixed_packed_vlen_and_file_roundtrip(bb, port, curve, tmp_path):
    rng = np.random.default_rng(40 + curve)
    m = 300
    _, gens_p = common.generators_for(port, curve, m)
    h = bb.MultiexpHandle(curve, gens_p)
    sc = rng.integers(0, 256, (m, 3 * 32), dtype=np.uint8)
    a = h.fixed_multiexponentiation(32, 3, m, sc)
    b = port.fixed_msm(curve, gens_p, 3, m, sc, element_num_bytes=32)
    assert common.same(curve, port.normalize(curve, a), port.normalize(curve, b))
    bt = [3, 1, 14, 9, 64, 5, 200]
    row = (sum(bt) + 7) // 8
    psc = rng.integers(0, 256, (m, row), dtype=np.uint8)
    a = h.fixed_packed_multiexponentiation(bt, m, psc)
    b = port.fixed_msm(curve, gens_p, len(bt), m, psc, output_bit_table=bt)
    assert common.same(curve, port.normalize(curve, a), port.normalize(curve, b))
    lens = [1, 2, 17, 17, 40, 50, 300]
    a = h.fixed_vlen_multiexponentiation(bt, lens, psc)
    b = port.fixed_msm(curve, gens_p, len(bt), m, psc, output_bit_table=bt, output_lengths=lens)
    assert common.same(curve, port.normalize(curve, a), port.normalize(curve, b))
    path = str(tmp_path / "handle.bin")
    h.write_to_file(path)
    h2 = bb.MultiexpHandle(curve, filename=path)
    a2 = h2.fixed_vlen_multiexponentiation(bt, lens, psc)
    assert common.same(curve, port.normalize(curve, a2), port.normalize(curve, a))
    h.free()
    h2.free()


def test_reference_fixed_pedersen_vectors(bb, port):
    g = port.ristretto_generators(2, 0)
    h = bb.MultiexpHandle(0, g)
    res = h.fixed_multiexponentiation(2, 1, 2, np.array([1, 0, 0, 2], dtype=np.uint8))
    want = port.commit(0, [(np.array([[1, 0], [0, 2]], dtype=np.uint8), 0)], g)
    assert np.array_equal(port.normalize(0, res), want)
    res = h.fixed_packed_multiexponentiation([3, 1], 2, np.array([0b1010, 0b0101], dtype=np.uint8))
    want = port.commit(0, [(np.array([[2], [5]], dtype=np.uint8), 0),
                           (np.array([[1], [0]], dtype=np.uint8), 0)], g)
    assert np.array_equal(port.normalize(0, res), want)
    h.free()


def test_full_size_properties_c2(bb, port):
    """BASELINE config 2 size (ristretto, n = 2^20, 252-bit scalars): size-independent checks.
    (1) linearity: MSM over [0,n) == sum of the MSMs over two halves (partials + combine);
    (2) a 2^16 prefix with the remaining scalars zeroed equals the oracle on that prefix."""
    n = 1 << 20
    rng = np.random.default_rng(2)
    s = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    s[:, 31] &= 0x0F
    gens = bb.get_generators(n, 0)
    full = bb.compute_pedersen_commitments(0, [(s, 0)], gens)
    dg = bb.DeviceBuffer(host=gens)
    ds = bb.DeviceBuffer(host=s)
    parts = bb.DeviceBuffer(2 * 128)
    half = n // 2
    bb.commit_device(0, [(half, 32, 0)], [ds.ptr], dg.ptr, None, parts.ptr)
    bb.commit_device(0, [(half, 32, 0)], [ds.ptr + half * 32], dg.ptr + half * 160, None,
                     parts.ptr + 128)
    out = bb.DeviceBuffer(32)
    bb.combine_partials_device(0, out.ptr, parts.ptr, 2, 1)
    assert np.array_equal(out.to_host()[:32], full[0])
    m = 1 << 14
    z = s.copy()
    z[m:] = 0
    got = bb.compute_pedersen_commitments(0, [(z, 0)], gens)
    assert np.array_equal(got, port.commit(0, [(s[:m], 0)], gens[:m]))
    for b_ in (dg, ds, parts, out):
        b_.free()


def test_upload_pieces_and_column_groups(bb, port, monkeypatch):
    """Host calls upload the generator range in pieces (copy stream) while earlier pieces are being
    accumulated; with several column groups every group must see all pieces."""
    rng = np.random.default_rng(31)
    n = 9000
    gens, _ = common.generators_for(port, 0, n)
    cols = common.random_columns(rng, n, [(0, 32, 0), (-4000, 16, 1), (0, 8, 0), (-8999, 32, 0)])
    want = port.commit(0, cols, gens)
    for ranges, group_entries in (("3", None), ("5", "50000"), ("1", "20000")):
        monkeypatch.setenv("BLITZAR_B200_RANGES", ranges)
        if group_entries:
            monkeypatch.setenv("BLITZAR_B200_GROUP_ENTRIES", group_entries)
        assert np.array_equal(bb.compute_pedersen_commitments(0, cols, gens), want), (ranges, group_entries)
        assert np.array_equal(bb.compute_pedersen_commitments(0, cols[:2], None, 7),
                              port.commit(0, cols[:2], None, 7))


@pytest.mark.parametrize("curve", [1, 2, 3])
def test_upload_pieces_weierstrass(bb, port, curve, monkeypatch):
    """Later upload pieces go through the scratch bucket array + MergeBucketsBody on every curve."""
    rng = np.random.default_rng(40 + curve)
    n = 3000
    gens, _ = common.generators_for(port, curve, n)
    cols = common.random_columns(rng, n, [(0, 32, 0), (-1000, 16, 1), (-2999, 32, 0)])
    want = port.commit(curve, cols, gens)
    for ranges in ("2", "4"):
        monkeypatch.setenv("BLITZAR_B200_RANGES", ranges)
        assert common.same(curve, bb.compute_pedersen_commitments(curve, cols, gens), want), ranges


def test_default_piece_count_large_n(bb):
    """n = 2^19 + 7 takes the default multi-piece upload (no env override): compare with the
    single-piece path on the same inputs, and with the homomorphic split of the range."""
    rng = np.random.default_rng(51)
    n = (1 << 19) + 7
    s = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    cols = [(s, 0), (s[: n - 12345, :8].copy(), 1)]
    got = bb.compute_pedersen_commitments(0, cols)
    os.environ["BLITZAR_B200_RANGES"] = "1"
    try:
        one = bb.compute_pedersen_commitments(0, cols)
    finally:
        del os.environ["BLITZAR_B200_RANGES"]
    assert np.array_equal(got, one)


def _fresh_columns_split_over_devices(bb, port):
    """By column, by generator range and sharded handles, BLITZAR_B200_DEVICES=k."""
    rng = np.random.default_rng(77)
    for curve, n, shapes in ((0, 5000, [(0, 32, 0), (-100, 16, 1), (0, 1, 0), (-4999, 8, 0), (0, 4, 1)]),
                             (1, 700, [(0, 32, 0), (0, 2, 0), (-3, 8, 1)]),
                             (2, 900, [(0, 32, 0)] * 7), (3, 300, [(0, 16, 0), (0, 16, 1)])):
        gens, _ = common.generators_for(port, curve, n)
        cols = common.random_columns(rng, n, shapes)
        got = bb.compute_pedersen_commitments(curve, cols, gens)
        assert common.same(curve, got, port.commit(curve, cols, gens)), curve
    cols = common.random_columns(rng, 3000, [(0, 8, 0)] * 9)  # built-in generators on every device
    assert np.array_equal(bb.compute_pedersen_commitments(0, cols, None, 11), port.commit(0, cols, None, 11))
    # fewer columns than devices: the generator RANGE is split, partial points gathered on device 0
    for curve, n, shapes in ((0, 5003, [(0, 32, 0)]), (1, 1300, [(0, 32, 0), (-700, 16, 1)]),
                             (2, 2100, [(-1, 32, 0)]), (3, 999, [(0, 8, 1)])):
        gens, _ = common.generators_for(port, curve, n)
        cols = common.random_columns(rng, n, shapes)
        got = bb.compute_pedersen_commitments(curve, cols, gens)
        assert common.same(curve, got, port.commit(curve, cols, gens)), ("range", curve)
    cols = common.random_columns(rng, 4000, [(0, 32, 0)])
    assert np.array_equal(bb.compute_pedersen_commitments(0, cols, None, 5), port.commit(0, cols, None, 5))
    # handles are sharded over the devices at construction; fixed / packed / vlen calls and the file
    for curve in range(4):
        m = 1100
        _, gens_p = common.generators_for(port, curve, m)
        h = bb.MultiexpHandle(curve, gens_p)
        sc = rng.integers(0, 256, (m, 2 * 32), dtype=np.uint8)
        a = h.fixed_multiexponentiation(32, 2, m, sc)
        b = port.fixed_msm(curve, gens_p, 2, m, sc, element_num_bytes=32)
        assert common.same(curve, port.normalize(curve, a), port.normalize(curve, b)), ("fixed", curve)
        a = h.fixed_multiexponentiation(32, 2, 300, sc[:300])  # fewer rows than generators
        b = port.fixed_msm(curve, gens_p, 2, 300, sc[:300], element_num_bytes=32)
        assert common.same(curve, port.normalize(curve, a), port.normalize(curve, b)), ("fixed300", curve)
        bt = [3, 1, 14, 64, 5, 200]
        psc = rng.integers(0, 256, (m, (sum(bt) + 7) // 8), dtype=np.uint8)
        lens = [1, 2, 17, 400, 900, m]
        a = h.fixed_vlen_multiexponentiation(bt, lens, psc)
        b = port.fixed_msm(curve, gens_p, len(bt), m, psc, output_bit_table=bt, output_lengths=lens)
        assert common.same(curve, port.normalize(curve, a), port.normalize(curve, b)), ("vlen", curve)
        path = os.path.join(tempfile.mkdtemp(), "h.bin")
        h.write_to_file(path)
        h2 = bb.MultiexpHandle(curve, filename=path)
        a2 = h2.fixed_vlen_multiexponentiation(bt, lens, psc)
        assert common.same(curve, port.normalize(curve, a2), port.normalize(curve, b)), ("file", curve)
        h.free(); h2.free()
        h3 = bb.MultiexpHandle(curve, filename=os.path.join(common.GOLDEN, f"ref_table_curve{curve}_w3.bin"))
        g7 = np.load(os.path.join(common.GOLDEN, f"fixed_curve{curve}.npz"))["generators_p"][:7]
        s7 = rng.integers(0, 256, (7, 32), dtype=np.uint8)
        assert common.same(curve, port.normalize(curve, h3.fixed_multiexponentiation(32, 1, 7, s7)),
                           port.normalize(curve, port.fixed_msm(curve, g7, 1, 7, s7, element_num_bytes=32)))
        h3.free()


def test_columns_split_over_devices():
    """BLITZAR_B200_DEVICES=k: independent columns run on k devices of this process (the reference
    splits by output the same way, sxt/multiexp/pippenger2/multiexponentiation.h:248-287). With one
    GPU, the test hook BLITZAR_B200_SHARED_DEVICES puts two shards on it. The same child runs the
    per-column offsets entry point (tests/test_gpu_commit_offsets.py)."""
    import torch
    env = dict(BLITZAR_B200_DEVICES=str(max(2, min(4, torch.cuda.device_count()))),
               BLITZAR_B200_SHARED_DEVICES="1" if torch.cuda.device_count() < 2 else "0",
               BLITZAR_B200_MIN_SHARD_TERMS="200")
    common.run_fresh(_fresh_columns_split_over_devices,
                     test_gpu_commit_offsets._fresh_split_over_devices, env=env)


# ---- fixed-base tables --------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", [0, 1, 2, 3])
def test_fixed_base_table_policies_agree(bb, port, curve, monkeypatch):
    """A handle holds the table 2^(c w) G_i; the same calls with the table forced on, forced off and
    under the cost model give the oracle's results (window width from the environment override)."""
    rng = np.random.default_rng(90 + curve)
    m = 3000
    _, gens_p = common.generators_for(port, curve, m)
    sc = rng.integers(0, 256, (m, 2 * 32), dtype=np.uint8)
    want = port.normalize(curve, port.fixed_msm(curve, gens_p, 2, m, sc, element_num_bytes=32))
    bt = [3, 1, 14, 64, 5, 200]
    psc = rng.integers(0, 256, (m, (sum(bt) + 7) // 8), dtype=np.uint8)
    lens = [1, 2, 17, 40, 50, m]
    wantv = port.normalize(curve, port.fixed_msm(curve, gens_p, len(bt), m, psc, output_bit_table=bt,
                                                 output_lengths=lens))
    for window in ("10", "16", "20", None):
        if window:
            monkeypatch.setenv("BLITZAR_B200_TABLE_WINDOW", window)
        else:
            monkeypatch.delenv("BLITZAR_B200_TABLE_WINDOW")
        h = bb.MultiexpHandle(curve, gens_p)
        for policy in ("1", "2", "0"):
            monkeypatch.setenv("BLITZAR_B200_TABLE_POLICY", policy)
            got = h.fixed_multiexponentiation(32, 2, m, sc)
            assert common.same(curve, port.normalize(curve, got), want), (window, policy)
            got = h.fixed_vlen_multiexponentiation(bt, lens, psc)
            assert common.same(curve, port.normalize(curve, got), wantv), (window, policy)
        h.free()
    monkeypatch.delenv("BLITZAR_B200_TABLE_POLICY")


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
def test_handle_from_reference_partition_table_file(bb, port, curve):
    """sxt_multiexp_handle_new_from_file reads the reference's own [u32 w][partition table] files
    (fixture written by the reference's code, tests/golden/make_table_files.py)."""
    gens_p = np.load(os.path.join(common.GOLDEN, f"fixed_curve{curve}.npz"))["generators_p"][:7]
    h = bb.MultiexpHandle(curve, filename=os.path.join(common.GOLDEN, f"ref_table_curve{curve}_w3.bin"))
    rng = np.random.default_rng(curve)
    sc = rng.integers(0, 256, (7, 32), dtype=np.uint8)
    got = h.fixed_multiexponentiation(32, 1, 7, sc)
    want = port.fixed_msm(curve, gens_p, 1, 7, sc, element_num_bytes=32)
    assert common.same(curve, port.normalize(curve, got), port.normalize(curve, want))
    h.free()


def _fresh_builtin_generator_table(bb, port):
    rng = np.random.default_rng(3)
    cols = common.random_columns(rng, 4000, [(0, 32, 0), (-100, 16, 1), (0, 1, 0), (-3999, 8, 0)])
    for policy in ("1", "2", "0"):
        os.environ["BLITZAR_B200_TABLE_POLICY"] = policy
        for off in (0, 37, 1000, 4000):
            assert np.array_equal(bb.compute_pedersen_commitments(0, cols, None, off),
                                  port.commit(0, cols, None, off)), (policy, off)
    g = bb.get_generators(10, 4995)
    assert np.array_equal(port.normalize(0, g), port.normalize(0, port.ristretto_generators(10, 4995)))


def test_builtin_generator_table():
    """num_precomputed_generators large enough for a fixed-base table over the built-in generators:
    commitments inside, straddling and beyond it, table forced on / off / cost model; the same child
    runs the per-column offsets entry point (tests/test_gpu_commit_offsets.py)."""
    common.run_fresh(_fresh_builtin_generator_table,
                     test_gpu_commit_offsets._fresh_builtin_generator_table,
                     init={"num_precomputed_generators": 5000})


def test_lane_sliced_field_arithmetic_selftest(bb):
    """The warp-cooperative field arithmetic of the tail kernels (10 lanes per element in radix 2^25.5,
    carries across lanes by shuffle) against the per-thread schedules, on random and edge-case
    operands."""
    for seed in (1, 2, 3):
        assert bb.selftest_lane_arithmetic(256, seed) == 0, seed


def test_lane_tail_on_off_agree(bb, port, monkeypatch):
    rng = np.random.default_rng(123)
    n = 3000
    cols = common.random_columns(rng, n, [(0, 32, 0), (-100, 16, 1), (0, 1, 0), (-2999, 8, 0), (0, 5, 0)])
    want = port.commit(0, cols, None, 9)
    for flag in ("0", "1"):
        monkeypatch.setenv("BLITZAR_B200_LANE_TAIL", flag)
        assert np.array_equal(bb.compute_pedersen_commitments(0, cols, None, 9), want), flag
