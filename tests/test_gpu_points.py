"""Point validation and decoding on the device (b200_check_points[_device], b200_decode_points[_device]):
the cases of tests/test_points.py through the C ABI, 2^20 synthetic points per curve with corruptions at
known indices, the host calls against the device calls, fixed-base MSM outputs through the device check,
and commitments decoded in HBM straight into a pairing check."""
import ctypes

import numpy as np
import pytest

from tests import common
from tests import pairing_reference as pairing
from tests import points_reference as pref
from tests import test_points as cpu

pytestmark = pytest.mark.gpu


def entries(bb):
    return cpu.Entries(lambda c, p: bb.call_check_points(bb.lib().b200_check_points, c, p),
                       lambda c, e: bb.call_decode_points(bb.lib().b200_decode_points, c, e),
                       bb.compute_pedersen_commitments,
                       lambda c, n, first, projective: bb.synthetic_generators(c, n, first, projective),
                       bb.field_op)


@pytest.mark.parametrize("check,curve", cpu.CASES, ids=cpu.CASE_IDS)
def test_points(bb, check, curve):
    check(entries(bb), curve)


@pytest.mark.parametrize("field", (1, 6))
def test_sqrt(bb, field):
    cpu.check_sqrt(entries(bb), field)


def upload_at(bb, ptr, host):
    """Copies the host array to device address ptr (inside a DeviceBuffer)."""
    host = np.ascontiguousarray(host)
    bb.lib().b200_memcpy_h2d(ctypes.c_void_p(ptr), ctypes.c_void_p(host.ctypes.data),
                             ctypes.c_uint64(host.nbytes))


def set_component(rows, idx, offset, value, width):
    rows[idx, offset:offset + width] = np.frombuffer(value.to_bytes(width, "little"), np.uint8)


def corrupted(bb, curve, n):
    """2^20-scale synthetic *_p2 points with known corruptions: (rows, expected valid flags)."""
    c = pref.CURVES[curve]
    rows = bb.synthetic_generators(curve, n, 0, projective=True)
    want = np.ones(n, np.uint8)
    rng = np.random.default_rng(curve)
    idx = rng.choice(n, 5 * 64, replace=False).reshape(5, 64)
    for i in idx[0]:  # a coordinate component at p: invalid
        set_component(rows, i, int(rng.integers(0, 3 * c.PARTS)) * c.W, c.P, c.W)
    want[idx[0]] = 0
    for i in idx[1]:  # Y + 1 (mod p): off the curve
        y = int.from_bytes(bytes(rows[i, c.COORD:c.COORD + c.W]), "little")
        set_component(rows, i, c.COORD, (y + 1) % c.P, c.W)
    want[idx[1]] = 0
    for i in idx[2]:  # Z = 0 with X and Y left as they are: the identity, valid
        rows[i, 2 * c.COORD:] = 0
    for i in idx[3]:  # X = 2^(64 limbs) - 1 on an identity: the range check comes first
        rows[i, 2 * c.COORD:] = 0
        set_component(rows, i, 0, c.MONT - 1, c.W)
    want[idx[3]] = 0
    if curve in cpu.COFACTOR_CURVES:  # points outside the subgroup
        out = cpu.outside_points(curve)
        for k, i in enumerate(idx[4]):
            rows[i] = c.proj_struct(out[k % len(out)], (k + 2, k) if c.PARTS == 2 else (k + 2, 0))
        want[idx[4]] = 0
    return rows, want


def encodings(bb, curve, m):
    """m commitment encodings: the affine synthetic generators themselves (curves 2, 3 and 5, whose
    commitments are that struct) or the library's commitments to them (curves 1 and 4)."""
    gens = bb.synthetic_generators(curve, m)
    if not pref.CURVES[curve].COMPRESSED:
        return gens
    ones = [(np.ones((1, 1), np.uint8), 0)] * m
    return bb.compute_pedersen_commitments_with_offsets(curve, ones, np.arange(m), gens)


@pytest.mark.parametrize("curve", cpu.CURVES)
def test_2_20_points_with_known_corruptions(bb, curve):
    """2^20 synthetic points with corruptions at known indices return exactly that valid pattern and
    count, and the device call gives the host call's flags. Decoding 2^12 commitment encodings, every
    97th corrupted, gives the same flags and bytes on the host and on the device."""
    c = pref.CURVES[curve]
    n = 1 << 20
    rows, want = corrupted(bb, curve, n)
    valid, count = bb.call_check_points(bb.lib().b200_check_points, curve, rows)
    assert np.array_equal(valid, want) and count == int(want.sum())
    d_rows, d_valid = bb.DeviceBuffer(host=rows), bb.DeviceBuffer(n)
    bb.check_points_device(curve, d_valid.ptr, d_rows.ptr, n)
    assert np.array_equal(d_valid.to_host(), valid)
    d_rows.free()
    m = 1 << 12
    enc = encodings(bb, curve, m)
    if c.COMPRESSED:
        enc[::97, 1] ^= 0x5A  # another x: no point, or one far outside the subgroup
    else:
        enc[::97, 2 * c.COORD] = 2  # an infinity byte other than 0 and 1
    p2, hv, hcount = bb.call_decode_points(bb.lib().b200_decode_points, curve, enc)
    want = np.ones(m, np.uint8)
    want[::97] = 0
    assert np.array_equal(hv, want) and hcount == int(want.sum())
    d_enc, d_out = bb.DeviceBuffer(host=enc), bb.DeviceBuffer(m * c.PROJ_BYTES)
    bb.decode_points_device(curve, d_out.ptr, d_valid.ptr, d_enc.ptr, m)
    assert np.array_equal(d_out.to_host((m, c.PROJ_BYTES)), p2)
    assert np.array_equal(d_valid.to_host()[:m], hv)
    for b in (d_valid, d_enc, d_out):
        b.free()


@pytest.mark.parametrize("curve", cpu.CURVES)
def test_fixed_msm_outputs_pass(bb, curve):
    """Every output of b200_fixed_msm_device (including an identity from a zero scalar row) passes
    b200_check_points_device."""
    n, m = 512, 64
    gens = bb.synthetic_generators(curve, n, projective=True)
    h = bb.MultiexpHandle(curve, gens)
    s = np.random.default_rng(curve).integers(0, 256, (n, m, 32), dtype=np.uint8)
    s[:, 0] = 0
    w = bb.CURVE_SIZES[curve][0]
    ds, res, valid = bb.DeviceBuffer(host=s), bb.DeviceBuffer(m * w), bb.DeviceBuffer(m)
    try:
        bb.fixed_msm_device(h, res.ptr, None, 32, m, n, ds.ptr)
        bb.check_points_device(curve, valid.ptr, res.ptr, m)
        assert valid.to_host().tolist() == [1] * m
        assert res.to_host((m, w))[0, 2 * w // 3:].sum() == 0  # the zero row is the identity
    finally:
        h.free()
        for b in (ds, res, valid):
            b.free()


@pytest.mark.parametrize("curve", (1, 2, 4, 5))
def test_commitments_decoded_into_a_pairing(bb, curve):
    """Commitments C_j over synthetic generators with known logs (compressed for curve 1, affine for
    curve 2, G2 commitments for curves 4 and 5) go through b200_decode_points_device and then
    b200_multi_pairing_device without returning to the host: prod_j e(C_j, H_j) e(-[s_j] G, H_j) = 1
    (G1) or prod_j e(P_j, C_j) e(-[s_j] P_j, H) = 1 (G2), with s_j in closed form."""
    g1_curve = {1: 1, 2: 2, 4: 1, 5: 2}[curve]
    t = pairing.TOWERS[g1_curve]
    g2_side = curve in (4, 5)
    n, m = 256, 8
    rng = np.random.default_rng(40 + curve)
    cols = [(rng.integers(0, 256, (n, 32), dtype=np.uint8), 0) for _ in range(m)]
    com = bb.compute_pedersen_commitments(curve, cols, bb.synthetic_generators(curve, n))
    k = common.synth_scalars_k(n)
    s = [common.dot_mod(col, k, t.R) for col, _ in cols]
    w1, w2 = bb.CURVE_SIZES[g1_curve][0], bb.CURVE_SIZES[pairing.G2_CURVE[g1_curve]][0]
    tj = [int(v) for v in rng.integers(1, 1 << 62, m)]
    if g2_side:  # g1 = [P_j, -s_j P_j], g2 = [C_j (decoded), H]
        g1 = np.stack([t.g1_proj_struct(t.g1_mul(v)) for v in tj] +
                      [t.g1_proj_struct(t.g1_mul(-sj * v)) for sj, v in zip(s, tj)])
        g2_rest = np.stack([t.g2_proj_struct(t.G2.G)] * m)
        g1_buf = bb.DeviceBuffer(host=g1)
        g2_buf = bb.DeviceBuffer(2 * m * w2)
        upload_at(bb, g2_buf.ptr + m * w2, g2_rest)
        decoded_at = g2_buf.ptr
    else:  # g1 = [C_j (decoded), -s_j G], g2 = [H_j, H_j]
        g1_rest = np.stack([t.g1_proj_struct(t.g1_mul(-sj)) for sj in s])
        hs = [t.g2_proj_struct(t.g2_mul(v)) for v in tj]
        g2_buf = bb.DeviceBuffer(host=np.stack(hs + hs))
        g1_buf = bb.DeviceBuffer(2 * m * w1)
        upload_at(bb, g1_buf.ptr + m * w1, g1_rest)
        decoded_at = g1_buf.ptr
    d_com, valid, out = bb.DeviceBuffer(host=com), bb.DeviceBuffer(m), bb.DeviceBuffer(m * t.GT_BYTES)
    try:
        bb.decode_points_device(curve, decoded_at, valid.ptr, d_com.ptr, m)
        lengths = [2 * m]
        bb.multi_pairing_device(g1_curve, out.ptr, lengths, g1_buf.ptr, g2_buf.ptr)
        got = out.to_host()[:t.GT_BYTES]
        assert valid.to_host().tolist() == [1] * m
        assert got.tobytes() == t.to_bytes(t.ONE)
    finally:
        for b in (g1_buf, g2_buf, d_com, valid, out):
            b.free()
