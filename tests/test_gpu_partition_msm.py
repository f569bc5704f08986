"""Fixed-base MSMs answered from a partition table on the handle (b200_multiexp_handle_add_partition_table,
partition_msm.cuh) through the C ABI: the oracle's results for every layout, table width, policy and
degenerate input; the device entry with results and with partial points; handles read from the
reference's files and from files this library wrote; tables attached at construction by
BLITZAR_B200_PARTITION_HANDLES; sharded handles; a Proof-of-SQL-like shape; and a table that does
not fit."""
import os

import numpy as np
import pytest

from tests import common
from tests import partition_tables as pt

pytestmark = pytest.mark.gpu
WIDTHS = [1, 1, 1, 5, 1, 64, 256, 1, 13, 8, 1, 2]


def _lengths(n, w):
    return sorted(min(v, n) for v in [0, 1, max(w - 1, 0), w, w + 1, n, 2, n - 1, w, 3, n, n])


def _host_calls(h, rng, n, w):
    """(result, oracle call) of the three sxt_fixed_* calls."""
    sc = rng.integers(0, 256, (n, 3 * 2), dtype=np.uint8)
    psc = rng.integers(0, 256, (n, (sum(WIDTHS) + 7) // 8), dtype=np.uint8)
    lens = _lengths(n, w)
    return [(h.fixed_multiexponentiation(2, 3, n, sc), (3, n, sc), dict(element_num_bytes=2)),
            (h.fixed_packed_multiexponentiation(WIDTHS, n, psc), (len(WIDTHS), n, psc),
             dict(output_bit_table=WIDTHS)),
            (h.fixed_vlen_multiexponentiation(WIDTHS, lens, psc), (len(WIDTHS), n, psc),
             dict(output_bit_table=WIDTHS, output_lengths=lens))]


def _check_calls(port, curve, gens, h, rng, n, w):
    for got, args, kw in _host_calls(h, rng, n, w):
        want = port.fixed_msm(curve, gens, *args, **kw)
        assert common.same(curve, port.normalize(curve, got), port.normalize(curve, want)), (w, kw)


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
def test_widths_and_policies(bb, port, curve, monkeypatch):
    n = 301
    _, gens = common.generators_for(port, curve, n, seed=31)
    h = bb.MultiexpHandle(curve, gens)
    assert h.partition_window == 0
    rng = np.random.default_rng(curve)
    for w in (1, 3, 8, 16):
        assert h.add_partition_table(w) == w  # a second call replaces the table
        assert h.partition_window == w
        for policy in ("0", "1", "2"):
            monkeypatch.setenv("BLITZAR_B200_PARTITION_POLICY", policy)
            _check_calls(port, curve, gens, h, rng, n, w)
    h.free()


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
def test_degenerate_generators_and_scalars(bb, port, curve, monkeypatch):
    """Duplicates, G / -G pairs and identity generators; random, all-zero and all-ones scalars."""
    n = 29
    _, gens = common.generators_for(port, curve, n, seed=44)
    gens = pt.edit_generators(curve, np.array(gens, copy=True))
    h = bb.MultiexpHandle(curve, gens)
    monkeypatch.setenv("BLITZAR_B200_PARTITION_POLICY", "1")
    row = (sum(WIDTHS) + 7) // 8
    for w in (3, 6):
        assert h.add_partition_table(w) == w
        for psc in (np.random.default_rng(w).integers(0, 256, (n, row), dtype=np.uint8),
                    np.zeros((n, row), np.uint8), np.full((n, row), 0xFF, np.uint8)):
            lens = _lengths(n, w)
            got = h.fixed_vlen_multiexponentiation(WIDTHS, lens, psc)
            want = port.fixed_msm(curve, gens, len(WIDTHS), n, psc, output_bit_table=WIDTHS,
                                  output_lengths=lens)
            assert common.same(curve, port.normalize(curve, got), port.normalize(curve, want)), w
    h.free()


@pytest.mark.parametrize("curve", [0, 2])
def test_device_entry_results_and_partials(bb, port, curve, monkeypatch):
    n, w = 777, 5
    _, gens = common.generators_for(port, curve, n, seed=8)
    h = bb.MultiexpHandle(curve, gens)
    assert h.add_partition_table(w) == w
    psc = np.random.default_rng(4).integers(0, 256, (n, (sum(WIDTHS) + 7) // 8), dtype=np.uint8)
    sc = bb.DeviceBuffer(host=np.concatenate([psc.reshape(-1), np.zeros(64, np.uint8)]))
    m, proj = len(WIDTHS), bb.CURVE_SIZES[curve][0]
    res = bb.DeviceBuffer(m * proj)
    parts = bb.DeviceBuffer(m * bb.point_bytes(curve))
    combined = bb.DeviceBuffer(m * proj)
    for policy in ("0", "1"):
        monkeypatch.setenv("BLITZAR_B200_PARTITION_POLICY", policy)
        for lens in (None, _lengths(n, w)):
            want = port.normalize(curve, port.fixed_msm(curve, gens, m, n, psc, output_bit_table=WIDTHS,
                                                        output_lengths=lens))
            bb.fixed_msm_device(h, res.ptr, None, 0, m, n, sc.ptr, bit_table=WIDTHS, lengths=lens)
            got = res.to_host().reshape(m, proj)
            assert common.same(curve, port.normalize(curve, got), want), (policy, lens)
            bb.fixed_msm_device(h, None, parts.ptr, 0, m, n, sc.ptr, bit_table=WIDTHS, lengths=lens)
            bb.combine_partials_projective_device(curve, combined.ptr, parts.ptr, 1, m)
            got = combined.to_host().reshape(m, proj)
            assert common.same(curve, port.normalize(curve, got), want), (policy, lens)
    for b in (sc, res, parts, combined):
        b.free()
    h.free()


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
def test_handles_from_files(bb, port, curve, tmp_path, monkeypatch):
    """The reference's own w = 3 file, and a w = 7 file this library wrote, read into handles that
    then carry partition tables."""
    monkeypatch.setenv("BLITZAR_B200_PARTITION_POLICY", "1")
    g7 = np.load(os.path.join(common.GOLDEN, f"fixed_curve{curve}.npz"))["generators_p"][:7]
    h = bb.MultiexpHandle(curve, filename=os.path.join(common.GOLDEN, f"ref_table_curve{curve}_w3.bin"))
    assert h.add_partition_table(3) == 3
    _check_calls(port, curve, g7, h, np.random.default_rng(1), 7, 3)
    h.free()
    n = 500
    _, gens = common.generators_for(port, curve, n, seed=6)
    h = bb.MultiexpHandle(curve, gens)
    path = str(tmp_path / "w7.bin")
    h.write_partition_table(path, 7)
    h.free()
    h = bb.MultiexpHandle(curve, filename=path)
    assert h.add_partition_table(4) == 4
    _check_calls(port, curve, gens, h, np.random.default_rng(2), n, 4)
    h.free()


def _check_handles(bb, port, check_handle):
    """Per curve, a handle over 1100 generators: check_handle(curve, h), then a vlen call whose lengths
    straddle 550 (the shard boundary of two shards) against the oracle."""
    for curve in range(4):
        n = 1100
        _, gens = common.generators_for(port, curve, n, seed=17)
        h = bb.MultiexpHandle(curve, gens)
        check_handle(curve, h)
        bt = [1, 3, 64, 256, 1, 8]
        psc = np.random.default_rng(curve).integers(0, 256, (n, (sum(bt) + 7) // 8), dtype=np.uint8)
        lens = [0, 1, 549, 550, 551, n]
        got = h.fixed_vlen_multiexponentiation(bt, lens, psc)
        want = port.fixed_msm(curve, gens, len(bt), n, psc, output_bit_table=bt, output_lengths=lens)
        assert common.same(curve, port.normalize(curve, got), port.normalize(curve, want)), curve
        h.free()


def test_tables_attached_at_construction(bb, port, tmp_path, monkeypatch):
    """BLITZAR_B200_PARTITION_HANDLES=1: sxt_multiexp_handle_new and _new_from_file (both file
    formats) attach a table at the default width (here BLITZAR_PARTITION_WINDOW_WIDTH=5)."""
    monkeypatch.setenv("BLITZAR_B200_PARTITION_HANDLES", "1")
    monkeypatch.setenv("BLITZAR_PARTITION_WINDOW_WIDTH", "5")
    monkeypatch.setenv("BLITZAR_B200_PARTITION_POLICY", "1")

    def attached_at_width_5(curve, h):
        assert h.partition_window == 5, h.partition_window
        a, b = str(tmp_path / f"{curve}.b2hd"), str(tmp_path / f"{curve}.ref")
        h.write_to_file(a)
        h.write_partition_table(b, 7)
        for path in (a, b):
            h2 = bb.MultiexpHandle(curve, filename=path)
            assert h2.partition_window == 5, (path, h2.partition_window)
            h2.free()

    _check_handles(bb, port, attached_at_width_5)


def _fresh_sharded_handles(bb, port):
    def add_width_7(curve, h):
        assert h.add_partition_table(7) == 7 and h.partition_window == 7

    _check_handles(bb, port, add_width_7)


def test_sharded_handles():
    """Two shards sharing the GPU, each with the table of its own generators: the shard boundary
    (550) is not a multiple of w = 7."""
    common.run_fresh(_fresh_sharded_handles,
                     env=dict(BLITZAR_B200_DEVICES="2", BLITZAR_B200_SHARED_DEVICES="1",
                              BLITZAR_B200_MIN_SHARD_TERMS="200", BLITZAR_B200_PARTITION_POLICY="1"))


@pytest.mark.parametrize("curve", [0, 2])
def test_proof_of_sql_shape(bb, curve, monkeypatch):
    """n = 2^12 rows, 1024 vlen outputs of mixed widths: the same results with the table (cost model
    and forced) as without it."""
    n, m = 1 << 12, 1024
    gens = bb.synthetic_generators(curve, n, projective=True)
    h = bb.MultiexpHandle(curve, gens)
    rng = np.random.default_rng(11)
    bt = [(1, 8, 16, 32, 64, 5, 12, 64)[j % 8] for j in range(m)]
    lens = sorted(int(v) for v in rng.integers(0, n + 1, m))
    psc = rng.integers(0, 256, (n, (sum(bt) + 7) // 8), dtype=np.uint8)
    monkeypatch.setenv("BLITZAR_B200_PARTITION_POLICY", "2")
    base = h.fixed_vlen_multiexponentiation(bt, lens, psc)
    assert h.add_partition_table(0) == 16
    from oracle import port
    port.build()
    want = port.normalize(curve, base)
    for policy in ("0", "1"):
        monkeypatch.setenv("BLITZAR_B200_PARTITION_POLICY", policy)
        got = h.fixed_vlen_multiexponentiation(bt, lens, psc)
        assert np.array_equal(port.normalize(curve, got), want), policy
    h.free()


def test_table_over_budget(bb, port):
    """w = 24 over 1100 bn254 generators would take 49 GB (more than 40 % of the HBM): nothing is
    attached, the call returns 0, and the handle keeps working (and takes a smaller table)."""
    curve, n = 2, 1100
    _, gens = common.generators_for(port, curve, n, seed=3)
    h = bb.MultiexpHandle(curve, gens)
    assert h.add_partition_table(4) == 4
    assert h.add_partition_table(24) == 0
    assert h.partition_window == 0
    _check_calls(port, curve, gens, h, np.random.default_rng(5), n, 4)
    assert h.add_partition_table(4) == 4
    _check_calls(port, curve, gens, h, np.random.default_rng(6), n, 4)
    h.free()
