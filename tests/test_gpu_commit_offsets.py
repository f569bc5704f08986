"""Per-column generator offsets on the GPU, through the C ABI (b200_compute_pedersen_commitments_
with_offsets, b200_commit_device_with_offsets): every column must equal the oracle's commitment of
that column alone at its offset, and, at full size, k separate calls of the existing entry points."""
import os

import numpy as np
import pytest

from tests import common
from tests.test_commit_offsets import FAR, columns, lengths, offset_patterns, oracle

pytestmark = pytest.mark.gpu


def _gens(port, curve, offsets, lens):
    return common.generators_for(port, curve, max(o + n for o, n in zip(offsets, lens)) + 1)[0]


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
def test_matrix(bb, port, curve):
    cols = columns(200 + curve)
    for pattern, offsets in offset_patterns(lengths()).items():
        gens = _gens(port, curve, offsets, lengths())
        got = bb.compute_pedersen_commitments_with_offsets(curve, cols, offsets, gens)
        assert common.same(curve, got, oracle(port, curve, cols, offsets, gens)), pattern
    if curve == 0:
        # 64 precomputed generators (conftest): intervals inside, straddling and beyond them
        for offsets in list(offset_patterns(lengths()).values()) + [FAR, [0, 1, 2, 3, 4, 5]]:
            got = bb.compute_pedersen_commitments_with_offsets(0, cols, offsets)
            assert np.array_equal(got, oracle(port, 0, cols, offsets, None)), offsets


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
def test_no_offsets_match_the_existing_calls(bb, port, curve):
    cols = columns(210 + curve)
    gens = common.generators_for(port, curve, 200)[0]
    want = bb.compute_pedersen_commitments(curve, cols, gens)
    assert np.array_equal(bb.compute_pedersen_commitments_with_offsets(curve, cols, None, gens), want)
    assert np.array_equal(bb.compute_pedersen_commitments_with_offsets(curve, cols, [0] * 6, gens), want)
    assert np.array_equal(bb.compute_pedersen_commitments_with_offsets(curve, cols, [50] * 6, gens),
                          bb.compute_pedersen_commitments(curve, cols, gens[50:]))
    if curve == 0:
        for off in (0, 17, 1 << 33):
            assert np.array_equal(bb.compute_pedersen_commitments_with_offsets(0, cols, [off] * 6),
                                  bb.compute_pedersen_commitments(0, cols, None, off)), off


@pytest.mark.parametrize("curve", [0, 2])
def test_sort_paths_and_upload_pieces(bb, port, curve, monkeypatch):
    cols = columns(220 + curve, n=3000,
                   shapes=[(0, 32, 0), (-1000, 16, 1), (0, 8, 1), (-2999, 5, 0), (-3000, 4, 0)])
    lens = lengths([(0, 32, 0), (-1000, 16, 1), (0, 8, 1), (-2999, 5, 0), (-3000, 4, 0)], 3000)
    offsets = [0, 1500, 4000, 10, 77]
    gens = _gens(port, curve, offsets, lens)
    want = oracle(port, curve, cols, offsets, gens)
    for sort in ("0", "2"):
        for ranges in ("1", "4"):
            monkeypatch.setenv("BLITZAR_B200_SORT", sort)
            monkeypatch.setenv("BLITZAR_B200_RANGES", ranges)
            got = bb.compute_pedersen_commitments_with_offsets(curve, cols, offsets, gens)
            assert common.same(curve, got, want), (sort, ranges)
            if curve == 0:
                got = bb.compute_pedersen_commitments_with_offsets(0, cols, FAR[:5])
                assert np.array_equal(got, oracle(port, 0, cols, FAR[:5], None)), (sort, ranges)


@pytest.mark.parametrize("curve", [1, 2, 3])
def test_forced_pair_levels(bb, port, curve, monkeypatch):
    cols = columns(230 + curve, n=2000, shapes=[(0, 32, 0), (-500, 16, 1), (0, 1, 0)])
    offsets = [0, 700, 2600]
    gens = _gens(port, curve, offsets, [2000, 1500, 2000])
    want = oracle(port, curve, cols, offsets, gens)
    for levels in ("0", "1", "3"):
        monkeypatch.setenv("BLITZAR_B200_PAIR_LEVELS", levels)
        got = bb.compute_pedersen_commitments_with_offsets(curve, cols, offsets, gens)
        assert common.same(curve, got, want), levels


@pytest.mark.parametrize("curve", [0, 2])
def test_device_entry_partials_combined(bb, port, curve):
    """Rows [0, h) at offsets and rows [h, n) at offsets + h, as partial points combined on the device,
    equal the one-pass commitments (the MSM is linear)."""
    n, h = 900, 400
    cols = columns(240 + curve, n=n, shapes=[(0, 32, 0), (0, 8, 1), (-300, 16, 0)])
    lens = [n, n, n - 300]
    offsets = [0, 250, 1200]
    gens = _gens(port, curve, offsets, lens)
    want = oracle(port, curve, cols, offsets, gens)
    dg = bb.DeviceBuffer(host=gens)
    ds = [bb.DeviceBuffer(host=np.ascontiguousarray(c)) for c, _ in cols]
    pb = bb.point_bytes(curve)
    parts = bb.DeviceBuffer(2 * len(cols) * pb)
    lo = [min(h, m) for m in lens]
    shape_a = [(lo[j], cols[j][0].shape[1], cols[j][1]) for j in range(3)]
    shape_b = [(lens[j] - lo[j], cols[j][0].shape[1], cols[j][1]) for j in range(3)]
    gp = dg.ptr
    bb.commit_device_with_offsets(curve, shape_a, [d.ptr for d in ds], gp, offsets, None, parts.ptr)
    bb.commit_device_with_offsets(curve, shape_b,
                                  [d.ptr + lo[j] * cols[j][0].shape[1] for j, d in enumerate(ds)], gp,
                                  [o + l for o, l in zip(offsets, lo)], None, parts.ptr + 3 * pb)
    stride = bb.CURVE_SIZES[curve][2]
    out = bb.DeviceBuffer(3 * stride)
    bb.combine_partials_device(curve, out.ptr, parts.ptr, 2, 3)
    got = out.to_host((3, stride))
    assert common.same(curve, got, want)
    # out_commitments of one device call
    outc = bb.DeviceBuffer(3 * stride)
    bb.commit_device_with_offsets(curve, [(lens[j], cols[j][0].shape[1], cols[j][1]) for j in range(3)],
                                  [d.ptr for d in ds], gp, offsets, outc.ptr, None)
    assert common.same(curve, outc.to_host((3, stride)), want)
    for b_ in [dg, parts, out, outc] + ds:
        b_.free()


# ---- fresh-process bodies, run by tests/test_gpu_parity.py next to the plain entry point's ---------
def _fresh_split_over_devices(bb, port):
    """BLITZAR_B200_DEVICES=k: by column and by generator range."""
    rng = np.random.default_rng(5)
    for curve in range(4):
        # by column (at least as many columns as devices), then by generator range (one column)
        for n, shapes, offsets in ((700, [(0, 32, 0), (-100, 16, 1), (0, 1, 0), (-699, 8, 0), (0, 4, 1)],
                                    [0, 900, 350, 5, 2000]),
                                   (1500, [(0, 32, 0)], [333])):
            cols = common.random_columns(rng, n, shapes)
            gens = common.generators_for(port, curve, max(offsets) + n)[0]
            got = bb.compute_pedersen_commitments_with_offsets(curve, cols, offsets, gens)
            assert common.same(curve, got, oracle(port, curve, cols, offsets, gens)), (curve, len(cols))
            if curve == 0:
                offs = [o + (1 << 33) for o in offsets]
                got = bb.compute_pedersen_commitments_with_offsets(0, cols, offs)
                assert np.array_equal(got, oracle(port, 0, cols, offs, None)), len(cols)


def _fresh_builtin_generator_table(bb, port):
    """num_precomputed_generators=5000: offsets inside, straddling and beyond the built-in table."""
    rng = np.random.default_rng(6)
    cols = common.random_columns(rng, 2000, [(0, 32, 0), (-100, 16, 1), (0, 1, 0), (-1999, 8, 0)])
    for policy in ("1", "2", "0"):
        os.environ["BLITZAR_B200_TABLE_POLICY"] = policy
        for offsets in ([0, 37, 1000, 2999], [0, 3500, 10, 4000], [5000, 6000, 9000, 5001]):
            got = bb.compute_pedersen_commitments_with_offsets(0, cols, offsets)
            assert np.array_equal(got, oracle(port, 0, cols, offsets, None)), (policy, offsets)


@pytest.mark.parametrize("curve", [0, 2])
def test_full_size_64_columns(bb, curve):
    """64 columns of 2^14 rows at 64 distinct offsets (2^20 terms: the binned sort runs) against 64
    separate calls of the existing entry points."""
    k, n = 64, 1 << 14
    rng = np.random.default_rng(300 + curve)
    s = rng.integers(0, 256, (k, n, 32), dtype=np.uint8)
    s[:, :, 31] &= 0x0F
    cols = [(s[j], 0) for j in range(k)]
    offsets = [int(v) for v in rng.permutation(k) * 5000]  # overlapping, distinct, in random order
    if curve == 0:
        got = bb.compute_pedersen_commitments_with_offsets(0, cols, offsets)
        want = np.concatenate([bb.compute_pedersen_commitments(0, [c], None, o)
                               for c, o in zip(cols, offsets)])
    else:
        gens = bb.synthetic_generators(curve, max(offsets) + n)
        got = bb.compute_pedersen_commitments_with_offsets(curve, cols, offsets, gens)
        want = np.concatenate([bb.compute_pedersen_commitments(curve, [c], gens[o:o + n])
                               for c, o in zip(cols, offsets)])
    assert np.array_equal(got, want)
