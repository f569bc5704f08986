"""Pairing products on the device (b200_multi_pairing, b200_multi_pairing_device): the cases of
tests/test_pairing.py through the C ABI, the PTX Fp12 arithmetic, a closed form over 2^16 synthetic
pairs, the Dory commitment flow from a fixed-base MSM into a pairing without leaving HBM, batches
against separate calls, the host call against the device call, and the launch count of a batch."""
import numpy as np
import pytest

from tests import common
from tests import pairing_reference as pr
from tests import test_pairing as cpu

pytestmark = pytest.mark.gpu
G2_FIRST = 1 << 20  # synthetic G2 points start here, so that their logs differ from the G1 ones


def logs(n, first=0):
    return common.synth_scalars_k(n, first)


def gt_power(t, e):
    return t.to_bytes(t.pow(t.pairing(t.G1, t.G2.G), e % t.R))


def synth_pairs(bb, curve, n):
    g1 = bb.synthetic_generators(curve, n, projective=True)
    g2 = bb.synthetic_generators(pr.G2_CURVE[curve], n, G2_FIRST, projective=True)
    return g1, g2


def dot_logs(k1, k2, r):
    """sum_i k1_i k2_i mod r for uint64 [n, 4] logs."""
    return common.dot_mod(np.ascontiguousarray(k2).view(np.uint8).reshape(-1, 32), k1, r)


@pytest.mark.parametrize("curve", cpu.CURVES)
def test_fp12_field_ops(bb, curve):
    cpu.check_fp12_ops(bb.field_op, curve)


@pytest.mark.parametrize("check", cpu.CHECKS, ids=[c.__name__[6:] for c in cpu.CHECKS])
@pytest.mark.parametrize("curve", cpu.CURVES)
def test_multi_pairing(bb, curve, check):
    check(bb.multi_pairing, curve)


@pytest.mark.parametrize("curve", cpu.CURVES)
def test_closed_form_2_16_pairs(bb, curve):
    """prod e(G_i, H_i) over 2^16 synthetic G_i = k_i G1 and H_i = k'_i G2 is e(G1, G2)^(sum k_i k'_i)."""
    t = pr.TOWERS[curve]
    n = 1 << 16
    g1, g2 = synth_pairs(bb, curve, n)
    got = bb.multi_pairing(curve, g1, g2, [n])
    assert got[0].tobytes() == gt_power(t, dot_logs(logs(n), logs(n, G2_FIRST), t.R))


@pytest.mark.parametrize("curve", cpu.CURVES)
def test_dory_flow_in_hbm(bb, curve):
    """b200_fixed_msm_device writes row commitments V_j = sum_i s_ij G_i over a handle of synthetic
    generators, and b200_multi_pairing_device pairs them with synthetic G2 points H_j in HBM:
    prod_j e(V_j, H_j) = e(G1, G2)^(sum_j (sum_i s_ij k_i) k'_j)."""
    t = pr.TOWERS[curve]
    n, m = 1024, 16
    gens = bb.synthetic_generators(curve, n, projective=True)
    h = bb.MultiexpHandle(curve, gens)
    s = np.random.default_rng(curve).integers(0, 256, (n, m, 32), dtype=np.uint8)
    w1 = bb.CURVE_SIZES[curve][0]
    g2_bytes = bb.CURVE_SIZES[pr.G2_CURVE[curve]][0]
    ds, rows = bb.DeviceBuffer(host=s), bb.DeviceBuffer(m * w1)
    hs, out = bb.DeviceBuffer(m * g2_bytes), bb.DeviceBuffer(t.GT_BYTES)
    try:
        bb.fixed_msm_device(h, rows.ptr, None, 32, m, n, ds.ptr)
        bb.synthetic_generators_device(pr.G2_CURVE[curve], hs.ptr, m, G2_FIRST, projective=True)
        bb.multi_pairing_device(curve, out.ptr, [m], rows.ptr, hs.ptr)
        got = out.to_host()
    finally:
        h.free()
        for b in (ds, rows, hs, out):
            b.free()
    k, k2 = logs(n), logs(m, G2_FIRST)
    v = [common.dot_mod(s[:, j], k, t.R) for j in range(m)]
    e = sum(vj * int.from_bytes(k2[j].tobytes(), "little") for j, vj in enumerate(v))
    assert got.tobytes() == gt_power(t, e)


@pytest.mark.parametrize("curve", cpu.CURVES)
def test_batch_equals_separate_calls_and_host_equals_device(bb, curve):
    """Products of 0, 1, 4 and 1000 pairs in one call give the bytes of four separate calls, and the
    device call gives the host call's bytes."""
    t = pr.TOWERS[curve]
    lengths = [0, 1, 4, 1000]
    n = sum(lengths)
    g1, g2 = synth_pairs(bb, curve, n)
    batch = bb.multi_pairing(curve, g1, g2, lengths)
    start = 0
    for k, length in enumerate(lengths):
        alone = bb.multi_pairing(curve, g1[start:start + length], g2[start:start + length], [length])
        assert np.array_equal(alone[0], batch[k]), length
        start += length
    assert batch[0].tobytes() == t.to_bytes(t.ONE)
    assert batch[1].tobytes() == gt_power(t, dot_logs(logs(1), logs(1, G2_FIRST), t.R))
    d1, d2 = bb.DeviceBuffer(host=g1), bb.DeviceBuffer(host=g2)
    out = bb.DeviceBuffer(len(lengths) * t.GT_BYTES)
    bb.multi_pairing_device(curve, out.ptr, lengths, d1.ptr, d2.ptr)
    assert np.array_equal(out.to_host(batch.shape), batch)
    for b in (d1, d2, out):
        b.free()


@pytest.mark.parametrize("curve", cpu.CURVES)
def test_launch_count_independent_of_the_number_of_products(bb, curve):
    """A batch of 64 products of 4 pairs launches as many kernels as a batch of one."""
    g1, g2 = synth_pairs(bb, curve, 64 * 4)
    counts = []
    for products in (1, 64):
        before = bb.launch_count()
        bb.multi_pairing(curve, g1[:4 * products], g2[:4 * products], [4] * products)
        counts.append(bb.launch_count() - before)
    assert counts[0] == counts[1] > 0, counts
