"""bn254 G2 (curve id 5) on the device: the cases of tests/test_bn254_g2.py through the C ABI on the
GPU, plus what only the device shows (full sizes with the automatic pair-level count, upload pieces,
partials across calls, handle files, partition tables attached to a handle, the PTX Fp2 arithmetic).
Results are checked against the closed form (sum_i s_i k_i mod r) G over synthetic generators
G_i = k_i G (tests/bn254_g2_reference.BN). Cases whose pair-level count is asserted run in a fresh
process, because the library reads BLITZAR_LOG_LEVEL once per process."""
import os

import numpy as np
import pytest

from tests import common
from tests import test_bls12_381_g2 as bls
from tests import test_bn254_g2 as cpu
from tests.test_gpu_batch_affine import _run_logged, case

pytestmark = pytest.mark.gpu
CURVE = 5
COMMIT = cpu.COMMIT
g2 = cpu.g2


def closed_form_dot(s, k):
    """Commitment of one 32-byte column s over generators with logs k (numpy dot)."""
    return np.frombuffer(g2.commitment(g2.scalar_mul(common.dot_mod(s, k, g2.R_ORDER))), np.uint8)


def test_fp2_field_op(bb):
    cpu.check_fp2(bb)


def test_synthetic_generators(bb):
    cpu.check_synthetic_generators(bb.synthetic_generators)


def test_commitments_closed_form(bb):
    """Every column shape over 2000 synthetic generators through the host commitment call, with and
    without generator offsets, and the device call on the same inputs."""
    n = 2000
    gens = bb.synthetic_generators(CURVE, n)
    cols = cpu.g2_columns(np.random.default_rng(5), n)
    k = common.synth_scalars_k(n)
    got = bb.compute_pedersen_commitments(CURVE, cols, gens)
    cpu.assert_closed_form(got, cols, k)
    offs = np.arange(len(cols), dtype=np.uint64) * 7
    wide = bb.synthetic_generators(CURVE, n + 7 * len(cols))
    off = bb.compute_pedersen_commitments_with_offsets(CURVE, cols, offs, wide)
    for j, col in enumerate(cols):
        cpu.assert_closed_form(off[j:j + 1], [col], common.synth_scalars_k(n, 7 * j))
    # the device call on device-resident copies gives the host call's bytes
    live = [(c, s) for c, s in cols if c.shape[0]]
    bufs = [bb.DeviceBuffer(host=c) for c, _ in live]
    dg = bb.DeviceBuffer(host=gens)
    out = bb.DeviceBuffer(len(live) * COMMIT)
    bb.commit_device(CURVE, [(c.shape[0], c.shape[1], s) for c, s in live], [b.ptr for b in bufs],
                     dg.ptr, out.ptr)
    assert np.array_equal(out.to_host((len(live), COMMIT)),
                          bb.compute_pedersen_commitments(CURVE, live, gens))
    for b in bufs + [dg, out]:
        b.free()


# ---- fresh processes: forced and automatic pair-level counts ---------------------------------------
def _fresh_forced_levels(bb, port, curve):
    n = 3000
    gens = bb.synthetic_generators(curve, n)
    ed = g2.edits(gens)
    ed.duplicate(slice(1, n, 7), 0)
    rng = np.random.default_rng(61)
    cols = common.random_columns(rng, n, [(0, 32, 0), (-13, 16, 1), (0, 8, 1), (-1, 5, 0),
                                          (-2999, 32, 0), (-1000, 2, 0), (0, 1, 0)])
    sg = np.zeros((n, 1), dtype=np.uint8)
    sg[::2], sg[1::2] = 1, 0xFF
    cols.append((sg, 1))
    want = g2.closed_form(cols, ed.k)
    cases = [(4, 1, 4, {}), (4, 3, 5, {}), (6, 2, 32, {}), (3, 5, 0, {}), (2, 6, 64, {}), (0, 6, 1, {}),
             (4, 2, 8, {"BLITZAR_B200_RANGES": "3"}),
             (5, 3, 16, {"BLITZAR_B200_GROUP_ENTRIES": "20000"})]
    for c, levels, batch, extra in cases:
        os.environ.update(BLITZAR_B200_PAIR_LEVELS=str(levels), BLITZAR_B200_PAIR_BATCH=str(batch), **extra)
        bb.set_tuning(window_bits=c)
        case("%d c=%d batch=%d %s" % (levels, c, batch, sorted(extra)))
        assert np.array_equal(bb.compute_pedersen_commitments(curve, cols, gens), want), (c, levels)
        for key in extra:
            del os.environ[key]
    bb.set_tuning()
    os.environ["BLITZAR_B200_PAIR_BATCH"] = "0"
    gens, ed, cols = cpu.degenerate_inputs(bb.synthetic_generators)
    want = g2.closed_form(cols, ed.k)
    for levels in range(1, 7):
        os.environ["BLITZAR_B200_PAIR_LEVELS"] = str(levels)
        case("%d degenerate" % levels)
        assert np.array_equal(bb.compute_pedersen_commitments(curve, cols, gens), want), levels


def test_forced_pair_levels_and_degenerate_buckets():
    """Window widths x forced pair levels x pairs per thread, upload pieces and column groups, then
    buckets of only +-P, identities and mixes at every level count; every range ran with the forced
    level count."""
    levels = _run_logged(_fresh_forced_levels, CURVE)
    assert len(levels) == 14, levels
    for label, used in levels.items():
        want = int(label.split()[0])
        assert used and all(v == want for v in used), (label, used)


def _fresh_full_size(bb, port, curve):
    n = 1 << 20
    gens = bb.synthetic_generators(curve, n)
    ed = g2.edits(gens)
    rng = np.random.default_rng(71)
    s = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    rows = np.arange(16, n, 16)
    ed.duplicate(rows, rows - 1)
    s[rows] = s[rows - 1]
    block = slice(1 << 19, (1 << 19) + 4096)  # one heavily loaded bucket
    ed.duplicate(block, 1 << 19)
    s[block] = 0
    s[block, 0] = 1
    ed.identity(slice(5, n, 3001))
    ed.negate(np.arange(7, n, 4099))
    want = closed_form_dot(s, ed.k)
    dg, ds, out = bb.DeviceBuffer(host=gens), bb.DeviceBuffer(host=s), bb.DeviceBuffer(COMMIT)
    case("full")
    bb.commit_device(curve, [(n, 32, 0)], [ds.ptr], dg.ptr, out.ptr)
    assert np.array_equal(out.to_host(), want)
    for b in (dg, ds, out):
        b.free()


def test_full_size_automatic_pair_levels():
    """n = 2^20 device-resident synthetic generators with duplicated, negated and identity rows and
    one bucket of 4096 equal points: the automatic level count turns on, and the commitment equals
    the closed form."""
    levels = _run_logged(_fresh_full_size, CURVE)
    print(f"bn254 G2 n = 2^20: pair levels {levels['full']}")
    assert levels["full"] and min(levels["full"]) >= 1, levels


def test_host_call_2_22_with_upload_pieces(bb):
    """One 2^22-term commitment from host memory, uploaded in pieces, against the closed form."""
    n = 1 << 22
    gens = bb.synthetic_generators(CURVE, n)
    s = np.random.default_rng(23).integers(0, 256, (n, 32), dtype=np.uint8)
    got = bb.compute_pedersen_commitments(CURVE, [(s, 0)], gens)
    assert np.array_equal(got[0], closed_form_dot(s, common.synth_scalars_k(n)))


# ---- partials ----------------------------------------------------------------------------------------
def test_partials_across_calls(bb):
    """b200_commit_device partials of two generator halves, and b200_commit_host_partials of the same
    halves, combined on the device, equal the host call over the whole range."""
    n = 1 << 14
    gens = bb.synthetic_generators(CURVE, n)
    cols = common.random_columns(np.random.default_rng(10), n, [(0, 32, 0), (0, 8, 1), (-100, 3, 0)])
    want = bb.compute_pedersen_commitments(CURVE, cols, gens)
    cpu.assert_closed_form(want, cols, common.synth_scalars_k(n))
    pb = bb.point_bytes(CURVE)
    assert pb == 192
    m, half = len(cols), n // 2
    parts, combined = bb.DeviceBuffer(2 * m * pb), bb.DeviceBuffer(m * COMMIT)
    for p, (lo, hi) in enumerate(((0, half), (half, n))):
        sub = [(c[lo:hi], s) for c, s in cols]
        bufs = [bb.DeviceBuffer(host=c) for c, _ in sub]
        dg = bb.DeviceBuffer(host=gens[lo:hi])
        bb.commit_device(CURVE, [(c.shape[0], c.shape[1], s) for c, s in sub], [b.ptr for b in bufs],
                         dg.ptr, None, parts.ptr + p * m * pb)
        bb.synchronize()
        for b in bufs + [dg]:
            b.free()
    bb.combine_partials_device(CURVE, combined.ptr, parts.ptr, 2, m)
    assert np.array_equal(combined.to_host((m, COMMIT)), want)
    for p, (lo, hi) in enumerate(((0, half), (half, n))):
        bb.commit_host_partials(CURVE, [(c[lo:hi], s) for c, s in cols], gens[lo:hi],
                                parts.ptr + p * m * pb)
    bb.combine_partials_device(CURVE, combined.ptr, parts.ptr, 2, m)
    assert np.array_equal(combined.to_host((m, COMMIT)), want)
    for b in (parts, combined):
        b.free()


# ---- handles -------------------------------------------------------------------------------------------
def test_handle_modes_file_and_partition_tables(bb, tmp_path, monkeypatch):
    """The fixed, packed and vlen calls over a handle of synthetic projective generators; the handle
    written to a file, read back and used; partition tables of widths 4 and 8 attached, giving the
    table-less results."""
    n = 4096
    gens_p = bb.synthetic_generators(CURVE, n, projective=True)
    k = common.synth_scalars_k(n)
    cases = bls.fixed_cases(np.random.default_rng(13), n)

    def run(h, kwargs):
        if "output_lengths" in kwargs:
            return h.fixed_vlen_multiexponentiation(kwargs["output_bit_table"], kwargs["output_lengths"],
                                                    kwargs["scalars"])
        if "output_bit_table" in kwargs:
            return h.fixed_packed_multiexponentiation(kwargs["output_bit_table"], n, kwargs["scalars"])
        return h.fixed_multiexponentiation(32, kwargs["num_outputs"], n, kwargs["scalars"])

    h = bb.MultiexpHandle(CURVE, gens_p)
    path = str(tmp_path / "bn254_g2.handle")
    h.write_to_file(path)
    back = bb.MultiexpHandle(CURVE, filename=path)
    try:
        for kwargs, cols in cases:
            plain = run(h, kwargs)
            cpu.check_fixed(plain, cols, k)
            assert cpu.proj_points(run(back, kwargs)) == cpu.proj_points(plain)
            for w in (4, 8):
                assert back.add_partition_table(w) == w
                for policy in ("1", "0"):
                    monkeypatch.setenv("BLITZAR_B200_PARTITION_POLICY", policy)
                    assert cpu.proj_points(run(back, kwargs)) == cpu.proj_points(plain), (w, policy)
    finally:
        h.free()
        back.free()
