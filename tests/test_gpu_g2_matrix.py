"""The G2 matrix on the device: every check of tests/test_g2_matrix.py for curves 4 (bls12-381 G2) and
5 (bn254 G2) through the C ABI, plus what only the device has: the device entries with partial
points, partition-table files read back into handles, and commitments and handles split over two
devices. Each test names the G1 test it ports; results are checked against the closed forms of
tests/test_g2_matrix.Oracle."""
import contextlib
import os
import tempfile

import numpy as np
import pytest

from tests import common
from tests import test_g2_matrix as mx

pytestmark = pytest.mark.gpu
CURVES = mx.CURVES
# BLITZAR_B200_* variables behind the checks' option names
_ENV = {"ranges": "RANGES", "pair_levels": "PAIR_LEVELS", "sort": "SORT", "table_policy": "TABLE_POLICY",
        "table_window": "TABLE_WINDOW", "partition_policy": "PARTITION_POLICY"}


class DeviceEntry:
    """The C ABI behind the names the checks use (see test_g2_matrix.EmulEntry). Options go to the
    environment through monkeypatch and to set_tuning; a fixed-base call builds its handle under
    them, so that BLITZAR_B200_TABLE_WINDOW applies."""
    SORTS = ("0", "2")  # the atomic sort and the binned sort

    def __init__(self, bb, monkeypatch):
        self.bb, self.mp = bb, monkeypatch

    def synth(self, curve, n, first=0, projective=False):
        return self.bb.synthetic_generators(curve, n, first, projective)

    def commit(self, curve, cols, gens):
        return self.bb.compute_pedersen_commitments(curve, cols, gens)

    def commit_offsets(self, curve, cols, offsets, gens):
        return self.bb.compute_pedersen_commitments_with_offsets(curve, cols, offsets, gens)

    @contextlib.contextmanager
    def options(self, window_bits=0, chunk1=0, chunkn=0, **opts):
        for name, value in opts.items():
            if value is not None:
                self.mp.setenv("BLITZAR_B200_" + _ENV[name], str(value))
        self.bb.set_tuning(window_bits, chunk1, chunkn)
        try:
            yield
        finally:
            self.bb.set_tuning()
            for name in opts:
                self.mp.delenv("BLITZAR_B200_" + _ENV[name], raising=False)

    def fixed(self, curve, gens_p, call, partition_window=0):
        h = self.bb.MultiexpHandle(curve, gens_p)
        try:
            if partition_window:
                assert h.add_partition_table(partition_window) == partition_window
            return run_call(h, call)
        finally:
            h.free()

    def partition_table(self, curve, gens_p, w, chunk_groups=0):
        bb = self.bb
        if chunk_groups:
            group = bb.COMPACT_BYTES[curve] << w
            self.mp.setenv("BLITZAR_B200_PTABLE_CHUNK_BYTES", str(chunk_groups * group + group // 2))
        n = gens_p.shape[0]
        g = bb.DeviceBuffer(host=np.ascontiguousarray(gens_p))
        out = bb.DeviceBuffer(bb.partition_table_bytes(curve, n, w))
        try:
            bb.partition_table_device(curve, out.ptr, g.ptr, n, w)
            return out.to_host()
        finally:
            self.mp.delenv("BLITZAR_B200_PTABLE_CHUNK_BYTES", raising=False)
            g.free()
            out.free()


def run_call(h, call):
    """One sxt_fixed_* call on a handle, from the checks' call keywords."""
    if call.get("output_lengths") is not None:
        return h.fixed_vlen_multiexponentiation(call["output_bit_table"], call["output_lengths"],
                                                call["scalars"])
    if call.get("output_bit_table") is not None:
        return h.fixed_packed_multiexponentiation(call["output_bit_table"], call["n"], call["scalars"])
    return h.fixed_multiexponentiation(call["element_num_bytes"], call["num_outputs"], call["n"],
                                       call["scalars"])


@pytest.fixture
def entry(bb, monkeypatch):
    return DeviceEntry(bb, monkeypatch)


# ---- test_gpu_parity ---------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES)
def test_edge_cases(entry, curve):
    """test_gpu_parity::test_edge_cases"""
    mx.check_edge_cases(entry, curve)


@pytest.mark.parametrize("curve", CURVES)
@pytest.mark.parametrize("n", [1, 31, 257, 4099, 20000])
def test_random_sweep(entry, curve, n):
    """test_gpu_parity::test_random_sweep"""
    mx.check_random_sweep(entry, curve, n)


@pytest.mark.parametrize("curve", CURVES)
def test_skewed_digits_and_tuning(entry, curve):
    """test_gpu_parity::test_skewed_digits_and_tuning"""
    mx.check_skewed_digits_and_tuning(entry, curve, 6000)


@pytest.mark.parametrize("curve", CURVES)
def test_fixed_base_table_policies_agree(entry, curve):
    """test_gpu_parity::test_fixed_base_table_policies_agree"""
    mx.check_table_policies(entry, curve, 3000)


# ---- test_gpu_commit_offsets -------------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES)
def test_offsets_matrix(entry, curve):
    """test_gpu_commit_offsets::test_matrix"""
    mx.check_offset_patterns(entry, curve)


@pytest.mark.parametrize("curve", CURVES)
def test_offsets_sort_paths_and_upload_pieces(entry, curve):
    """test_gpu_commit_offsets::test_sort_paths_and_upload_pieces"""
    mx.check_offset_sort_and_ranges(entry, curve, 3000)


@pytest.mark.parametrize("curve", CURVES)
def test_offsets_forced_pair_levels(entry, curve):
    """test_gpu_commit_offsets::test_forced_pair_levels"""
    mx.check_offset_pair_levels(entry, curve, 2000)


@pytest.mark.parametrize("curve", CURVES)
def test_offsets_device_entry_partials_combined(bb, curve):
    """test_gpu_commit_offsets::test_device_entry_partials_combined: rows [0, h) at the offsets and
    rows [h, n) at offsets + h as partial points, combined on the device, and the commitments of one
    device call, against the closed form of each column at its offset."""
    o = mx.Oracle(curve)
    n, h = 900, 400
    cols = mx.columns(240 + curve, n=n, shapes=[(0, 32, 0), (0, 8, 1), (-300, 16, 0)])
    lens = [n, n, n - 300]
    offsets = [0, 250, 1200]
    gens = bb.synthetic_generators(curve, max(o_ + m for o_, m in zip(offsets, lens)) + 1)
    dg = bb.DeviceBuffer(host=gens)
    ds = [bb.DeviceBuffer(host=np.ascontiguousarray(c)) for c, _ in cols]
    pb = bb.point_bytes(curve)
    stride = bb.CURVE_SIZES[curve][2]
    parts, out, outc = bb.DeviceBuffer(6 * pb), bb.DeviceBuffer(3 * stride), bb.DeviceBuffer(3 * stride)
    try:
        lo = [min(h, m) for m in lens]
        shape_a = [(lo[j], cols[j][0].shape[1], cols[j][1]) for j in range(3)]
        shape_b = [(lens[j] - lo[j], cols[j][0].shape[1], cols[j][1]) for j in range(3)]
        bb.commit_device_with_offsets(curve, shape_a, [d.ptr for d in ds], dg.ptr, offsets, None, parts.ptr)
        bb.commit_device_with_offsets(curve, shape_b,
                                      [d.ptr + lo[j] * cols[j][0].shape[1] for j, d in enumerate(ds)],
                                      dg.ptr, [a + b for a, b in zip(offsets, lo)], None, parts.ptr + 3 * pb)
        bb.combine_partials_device(curve, out.ptr, parts.ptr, 2, 3)
        mx.assert_offset_columns(o, out.to_host((3, stride)), cols, offsets)
        bb.commit_device_with_offsets(curve, [(lens[j], cols[j][0].shape[1], cols[j][1]) for j in range(3)],
                                      [d.ptr for d in ds], dg.ptr, offsets, outc.ptr, None)
        mx.assert_offset_columns(o, outc.to_host((3, stride)), cols, offsets)
    finally:
        for b in [dg, parts, out, outc] + ds:
            b.free()


# ---- test_gpu_batch_affine -----------------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES)
@pytest.mark.parametrize("levels", [None, 1, 3, 6])
def test_identity_generators(entry, curve, levels):
    """test_gpu_batch_affine::test_identity_generators"""
    mx.check_identity_generators(entry, curve, levels, 2000)


@pytest.mark.parametrize("curve", CURVES)
@pytest.mark.parametrize("window_bits", [10, 16])
def test_table_cross_window_collisions(entry, curve, window_bits):
    """test_gpu_batch_affine::test_table_cross_window_collisions"""
    mx.check_cross_window_collisions(entry, curve, window_bits)


# ---- test_gpu_partition_msm -----------------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES)
def test_partition_widths_and_policies(entry, curve):
    """test_gpu_partition_msm::test_widths_and_policies"""
    mx.check_partition_widths_and_policies(entry, curve)


@pytest.mark.parametrize("curve", CURVES)
def test_partition_degenerate_generators_and_scalars(entry, curve):
    """test_gpu_partition_msm::test_degenerate_generators_and_scalars"""
    mx.check_partition_degenerate(entry, curve)


@pytest.mark.parametrize("curve", CURVES)
def test_partition_device_entry_results_and_partials(bb, curve, monkeypatch):
    """test_gpu_partition_msm::test_device_entry_results_and_partials: b200_fixed_msm_device with a
    w = 5 table, results and partial points through combine_partials_projective_device."""
    o = mx.Oracle(curve)
    n, w = 777, 5
    gens = bb.synthetic_generators(curve, n, projective=True)
    k = mx.logs(n)
    h = bb.MultiexpHandle(curve, gens)
    assert h.add_partition_table(w) == w
    psc = np.random.default_rng(4).integers(0, 256, (n, (sum(mx.WIDTHS) + 7) // 8), dtype=np.uint8)
    m, proj = len(mx.WIDTHS), bb.CURVE_SIZES[curve][0]
    sc = bb.DeviceBuffer(host=np.concatenate([psc.reshape(-1), np.zeros(64, np.uint8)]))
    res, parts, combined = bb.DeviceBuffer(m * proj), bb.DeviceBuffer(m * bb.point_bytes(curve)), \
        bb.DeviceBuffer(m * proj)
    try:
        for lens in (None, mx.partition_lengths(n, w)):
            want = mx.expected_outputs(o, dict(num_outputs=m, n=n, scalars=psc, output_bit_table=mx.WIDTHS,
                                               output_lengths=lens), k)
            for policy in ("0", "1"):
                monkeypatch.setenv("BLITZAR_B200_PARTITION_POLICY", policy)
                bb.fixed_msm_device(h, res.ptr, None, 0, m, n, sc.ptr, bit_table=mx.WIDTHS, lengths=lens)
                assert o.points(res.to_host((m, proj))) == want, (policy, lens)
                bb.fixed_msm_device(h, None, parts.ptr, 0, m, n, sc.ptr, bit_table=mx.WIDTHS, lengths=lens)
                bb.combine_partials_projective_device(curve, combined.ptr, parts.ptr, 1, m)
                assert o.points(combined.to_host((m, proj))) == want, (policy, lens)
    finally:
        for b in (sc, res, parts, combined):
            b.free()
        h.free()


# ---- test_gpu_partition_table ------------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES)
@pytest.mark.parametrize("n", [37, 301])
@pytest.mark.parametrize("w", [1, 3, 7])
def test_partition_table_entries(entry, curve, n, w):
    """test_gpu_partition_table::test_full_size_bn254_table, at G2's 192- and 128-byte entries"""
    mx.check_partition_table_entries(entry, curve, n, w, samples=48)


@pytest.mark.parametrize("curve", CURVES)
def test_partition_table_many_chunks(entry, curve):
    """test_gpu_partition_table::test_many_chunks_give_the_same_file"""
    mx.check_partition_table_chunks(entry, curve)


@pytest.mark.parametrize("curve", CURVES)
def test_partition_table_file_round_trip(entry, bb, curve, tmp_path):
    """test_gpu_partition_table::test_round_trip_through_handle_files: the file a handle writes holds
    the device table, and reads back into a handle (padding included) that answers the fixed, packed
    and vlen calls."""
    o = mx.Oracle(curve)
    m = 301
    gens_p = bb.synthetic_generators(curve, m, projective=True)
    k = mx.logs(m)
    h = bb.MultiexpHandle(curve, gens_p)
    rng = np.random.default_rng(70 + curve)
    try:
        for w in (3, 7):
            path = str(tmp_path / f"w{w}.bin")
            h.write_partition_table(path, w)
            raw = np.fromfile(path, dtype=np.uint8)
            assert int(raw[:4].view("<u4")[0]) == w
            assert np.array_equal(raw[4:], entry.partition_table(curve, gens_p, w)), w
            back = bb.MultiexpHandle(curve, filename=path)
            try:
                for call in mx.fixed_calls(rng, m) + mx.partition_calls(rng, m, w)[1:2]:
                    assert o.points(run_call(back, call)) == mx.expected_outputs(o, call, k), w
            finally:
                back.free()
    finally:
        h.free()


# ---- split over devices --------------------------------------------------------------------------------
def _fresh_g2_shards(bb, port, curve):
    """Commitments split by column and by generator range, with and without offsets; a sharded
    handle's fixed, vlen and partition-table calls, and its two file formats read back."""
    o = mx.Oracle(curve)
    rng = np.random.default_rng(77 + curve)
    for n, shapes in ((700, [(0, 32, 0), (-100, 16, 1), (0, 1, 0), (-699, 8, 0), (0, 4, 1)]),
                      (1300, [(0, 32, 0)])):  # one column: the generator range is split
        gens = bb.synthetic_generators(curve, n + 2000)
        cols = common.random_columns(rng, n, shapes)
        mx.assert_columns(o, bb.compute_pedersen_commitments(curve, cols, gens[:n]), cols,
                          common.synth_scalars_k(n))
        offsets = [0, 900, 350, 5, 2000][:len(cols)] if len(cols) > 1 else [333]
        got = bb.compute_pedersen_commitments_with_offsets(curve, cols, offsets, gens)
        mx.assert_offset_columns(o, got, cols, offsets)
    m = 1100
    gens_p = bb.synthetic_generators(curve, m, projective=True)
    k = mx.logs(m)
    h = bb.MultiexpHandle(curve, gens_p)
    sc = rng.integers(0, 256, (m, 64), dtype=np.uint8)
    bt = [3, 1, 14, 64, 5, 200]
    psc = rng.integers(0, 256, (m, (sum(bt) + 7) // 8), dtype=np.uint8)
    calls = [dict(num_outputs=2, n=m, scalars=sc, element_num_bytes=32),
             dict(num_outputs=2, n=300, scalars=sc[:300], element_num_bytes=32),  # fewer rows
             dict(num_outputs=len(bt), n=m, scalars=psc, output_bit_table=bt,
                  output_lengths=[1, 2, 17, 549, 551, m])]  # straddling the shard boundary
    wants = [mx.expected_outputs(o, call, k) for call in calls]
    for call, want in zip(calls, wants):
        assert o.points(run_call(h, call)) == want, call["n"]
    d = tempfile.mkdtemp()
    for name, write in (("h.bin", h.write_to_file), ("t.bin", lambda p: h.write_partition_table(p, 7))):
        path = os.path.join(d, name)
        write(path)
        back = bb.MultiexpHandle(curve, filename=path)
        assert o.points(run_call(back, calls[2])) == wants[2], name
        back.free()
    assert h.add_partition_table(7) == 7
    os.environ["BLITZAR_B200_PARTITION_POLICY"] = "1"
    assert o.points(run_call(h, calls[2])) == wants[2]
    del os.environ["BLITZAR_B200_PARTITION_POLICY"]
    h.free()


def test_split_over_devices():
    """test_gpu_parity::test_columns_split_over_devices and test_gpu_partition_msm::test_sharded_handles:
    two shards sharing the GPU (BLITZAR_B200_DEVICES=2, BLITZAR_B200_SHARED_DEVICES=1)."""
    common.run_fresh(*[(_fresh_g2_shards, c) for c in CURVES],
                     env=dict(BLITZAR_B200_DEVICES="2", BLITZAR_B200_SHARED_DEVICES="1",
                              BLITZAR_B200_MIN_SHARD_TERMS="200"))
