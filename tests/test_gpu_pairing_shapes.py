"""Pairing products (b200_multi_pairing, pairing.cuh) at the shapes of the Miller loop's split, and fed
by the points the MSM calls write. multi_pairing gives each thread one pair up to kMillerThreads pairs
in a call, and above that per_thread = ceil(total / kMillerThreads) consecutive pairs of one product,
product k's length split at len * j / threads. Every product is checked against the closed form
e(G1, G2)^(sum k_i k'_i mod r) over its pairs that are not identities, with synthetic G_i = k_i G1 and
H_i = k'_i G2 (tests/test_gpu_pairing.py) and one GT power per product."""
import functools

import numpy as np
import pytest

from tests import common
from tests import pairing_reference as pr
from tests import test_g2_matrix as mx
from tests.test_gpu_pairing import G2_FIRST, synth_pairs

pytestmark = pytest.mark.gpu
CURVES = (1, 2)
K_MILLER_THREADS = 132 * 256  # pairing.cuh kMillerThreads


def per_thread(lengths):
    return max(1, -(-sum(lengths) // K_MILLER_THREADS))


@functools.lru_cache(maxsize=None)
def base(curve):
    t = pr.TOWERS[curve]
    return t.pairing(t.G1, t.G2.G)


def gt(curve, e):
    """The GT bytes of e(G1, G2)^e."""
    t = pr.TOWERS[curve]
    return t.to_bytes(t.pow(base(curve), e % t.R))


def ints(k):
    return [int.from_bytes(r.tobytes(), "little") for r in k]


class Pairs:
    """n synthetic pairs (projective structs) and the exponent k_i k'_i of each; identity() puts Z = 0
    on one side of a pair, keeping X and Y as an MSM writes a cancelled sum."""

    def __init__(self, bb, curve, n):
        self.t = pr.TOWERS[curve]
        self.curve = curve
        self.g1, self.g2 = (np.ascontiguousarray(a).copy() for a in synth_pairs(bb, curve, n))
        r = self.t.R
        self.e = [a * b % r for a, b in zip(ints(common.synth_scalars_k(n)),
                                            ints(common.synth_scalars_k(n, G2_FIRST)))]

    def identity(self, rows, side):
        w = self.t.W
        for i in rows:
            if side == 1:
                self.g1[i, 2 * w:3 * w] = 0
            else:
                self.g2[i, 4 * w:6 * w] = 0
            self.e[i] = 0

    def expected(self, lengths):
        out, i = [], 0
        for n in lengths:
            out.append(gt(self.curve, sum(self.e[i:i + n])))
            i += n
        return out

    def check(self, got, lengths, label=""):
        want = self.expected(lengths)
        bad = [k for k, (g, w) in enumerate(zip(got, want)) if g.tobytes() != w]
        assert not bad, f"{label} products {bad[:10]} (lengths {[lengths[k] for k in bad[:10]]}) differ"


def four_per_thread_lengths():
    """About 200 products of 3 * kMillerThreads + 5 pairs in all (four per thread): lengths 0, 1,
    below, at and just above four, lengths not divisible by four, and a few long products. The long
    product at index 2 has a length divisible by four, so its runs are aligned to multiples of 4."""
    total = 3 * K_MILLER_THREADS + 5
    rng = np.random.default_rng(4)
    short = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 11, 13, 0, 1, 4, 5]
    short += [int(v) for v in rng.integers(0, 40, 170)]
    lengths = [20000, 9, 24000] + short + [31001, 17]
    lengths.append(total - sum(lengths))
    assert lengths[-1] > 4000 and per_thread(lengths) == 4
    return lengths


@pytest.mark.parametrize("curve", CURVES)
def test_one_pair_per_thread(bb, curve):
    """Exactly kMillerThreads pairs: one per thread."""
    lengths = [K_MILLER_THREADS - 10, 0, 1, 2, 7]
    assert sum(lengths) == K_MILLER_THREADS and per_thread(lengths) == 1
    p = Pairs(bb, curve, sum(lengths))
    p.identity(range(5, K_MILLER_THREADS, 1001), 1)
    p.identity(range(500, K_MILLER_THREADS, 1003), 2)
    p.check(bb.multi_pairing(curve, p.g1, p.g2, lengths), lengths)


@pytest.mark.parametrize("curve", CURVES)
def test_two_pairs_per_thread(bb, curve):
    """kMillerThreads + 1 pairs: two per thread, with products of 1 and 3 pairs."""
    lengths = [K_MILLER_THREADS - 11, 1, 3, 0, 8]
    assert sum(lengths) == K_MILLER_THREADS + 1 and per_thread(lengths) == 2
    p = Pairs(bb, curve, sum(lengths))
    p.identity(range(3, K_MILLER_THREADS, 997), 2)
    p.check(bb.multi_pairing(curve, p.g1, p.g2, lengths), lengths)


@pytest.mark.parametrize("curve", CURVES)
def test_four_pairs_per_thread_with_identities(bb, curve):
    """Four pairs per thread over about 200 products, with Z = 0 on the G1 side in some rows and on
    the G2 side in others, a product made only of identities, and one aligned run of four identity
    pairs inside a long product. Five products in separate calls give the batch's bytes, and the
    device call gives the host call's."""
    lengths = four_per_thread_lengths()
    n = sum(lengths)
    starts = np.concatenate([[0], np.cumsum(lengths)[:-1]]).tolist()
    p = Pairs(bb, curve, n)
    p.identity(range(11, n, 97), 1)
    p.identity(range(40, n, 89), 2)
    p.identity(range(starts[1], starts[1] + 9), 1 + curve % 2)  # a product of identities only
    run = starts[2] + 4 * 1234  # thread 1234 of product 2 (24000 pairs, 6000 threads)
    p.identity(range(run, run + 4), 2)
    p.identity([run + 1], 1)
    batch = bb.multi_pairing(curve, p.g1, p.g2, lengths)
    p.check(batch, lengths)
    assert batch[1].tobytes() == pr.TOWERS[curve].to_bytes(pr.TOWERS[curve].ONE)
    for k in (0, 1, 5, 7, len(lengths) - 1):
        s, m = starts[k], lengths[k]
        alone = bb.multi_pairing(curve, p.g1[s:s + m], p.g2[s:s + m], [m])
        assert np.array_equal(alone[0], batch[k]), k
    d1, d2 = bb.DeviceBuffer(host=p.g1), bb.DeviceBuffer(host=p.g2)
    out = bb.DeviceBuffer(len(lengths) * p.t.GT_BYTES)
    try:
        bb.multi_pairing_device(curve, out.ptr, lengths, d1.ptr, d2.ptr)
        assert np.array_equal(out.to_host(batch.shape), batch)
    finally:
        for b in (d1, d2, out):
            b.free()


@pytest.mark.parametrize("curve", CURVES)
def test_launch_count_batch_values(bb, curve):
    """The 64 four-pair products of test_launch_count_independent_of_the_number_of_products, against
    the closed form."""
    lengths = [4] * 64
    p = Pairs(bb, curve, 256)
    p.check(bb.multi_pairing(curve, p.g1, p.g2, lengths), lengths)


def _neg_g1(t, pt):
    return None if pt is None else (pt[0], (-pt[1]) % t.P)


@pytest.mark.parametrize("curve", CURVES)
def test_kzg_dory_shape_from_msm_outputs(bb, curve):
    """V_j = b200_fixed_msm_device on the G1 curve and W_j = b200_fixed_msm_device on its G2 curve,
    both over handles of synthetic projective generators whose row 1 is the negation of row 0, paired
    by b200_multi_pairing_device without leaving HBM. V_0 and W_5 are identities by cancellation
    (s G + s (-G)), so the pairing reads the MSM's own (X, Y, 0); the last product's exponent
    sum_j v_j w_j is 0 mod r through the last W column's one non-zero scalar, so it is exactly 1."""
    t = pr.TOWERS[curve]
    o = mx.Oracle(pr.G2_CURVE[curve])
    r = t.R
    n, m = 64, 12
    lengths = [4, 3, 5]
    g1 = bb.synthetic_generators(curve, n, projective=True).copy()
    g2 = bb.synthetic_generators(o.curve, n, G2_FIRST, projective=True).copy()
    k1, k2 = ints(common.synth_scalars_k(n)), ints(common.synth_scalars_k(n, G2_FIRST))
    g1[1] = t.g1_proj_struct(_neg_g1(t, t.g1_mul(k1[0])))
    k1[1] = r - k1[0]
    g2[1] = o.proj_struct(o.point(-k2[0]))
    k2[1] = r - k2[0]
    rng = np.random.default_rng(curve)
    s1 = rng.integers(0, 256, (n, m, 32), dtype=np.uint8)
    s2 = rng.integers(0, 256, (n, m, 32), dtype=np.uint8)
    for s, j in ((s1, 0), (s2, 5)):  # one cancelled output each
        s[:, j] = 0
        s[0, j] = s[1, j] = rng.integers(1, 256, 32, dtype=np.uint8)
    s2[:, m - 1] = 0

    def values(s, k):
        return [sum(int.from_bytes(s[i, j].tobytes(), "little") * k[i] for i in range(n)) % r
                for j in range(m)]
    v, w = values(s1, k1), values(s2, k2)
    assert v[0] == 0 and w[5] == 0
    last = range(m - lengths[-1], m - 1)
    t_last = -sum(v[j] * w[j] for j in last) * pow(v[m - 1] * k2[7], -1, r) % r
    s2[7, m - 1] = np.frombuffer(t_last.to_bytes(32, "little"), np.uint8)
    w[m - 1] = t_last * k2[7] % r
    w1, w2 = bb.CURVE_SIZES[curve][0], bb.CURVE_SIZES[o.curve][0]
    h1, h2 = bb.MultiexpHandle(curve, g1), bb.MultiexpHandle(o.curve, g2)
    bufs = [bb.DeviceBuffer(host=s1), bb.DeviceBuffer(host=s2), bb.DeviceBuffer(m * w1),
            bb.DeviceBuffer(m * w2), bb.DeviceBuffer(len(lengths) * t.GT_BYTES)]
    ds1, ds2, rows1, rows2, out = bufs
    try:
        bb.fixed_msm_device(h1, rows1.ptr, None, 32, m, n, ds1.ptr)
        bb.fixed_msm_device(h2, rows2.ptr, None, 32, m, n, ds2.ptr)
        bb.multi_pairing_device(curve, out.ptr, lengths, rows1.ptr, rows2.ptr)
        got = out.to_host((len(lengths), t.GT_BYTES))
        V, W = rows1.to_host((m, w1)), rows2.to_host((m, w2))
    finally:
        h1.free()
        h2.free()
        for b in bufs:
            b.free()
    nb = w1 // 3
    assert not V[0, 2 * nb:].any() and not W[5, 4 * o.W:].any()  # the cancelled outputs have Z = 0
    e, i = [], 0
    for length in lengths:
        e.append(sum(v[j] * w[j] for j in range(i, i + length)))
        i += length
    assert e[-1] % r == 0
    assert got[-1].tobytes() == t.to_bytes(t.ONE)
    assert [g.tobytes() for g in got] == [gt(curve, x) for x in e]


@pytest.mark.parametrize("curve", CURVES)
def test_commit_partials_as_pairing_inputs(bb, curve):
    """b200_commit_device partial points of the G1 curve and of its G2 curve are the pairing's
    projective inputs as they stand: point_bytes equals the pairing's G1 / G2 stride, and
    prod_j e(P_j, Q_j) = e(G1, G2)^(sum_j (sum_i s_ij k_i)(sum_i t_ij k'_i)). Column 2 is all zero on
    both sides."""
    t = pr.TOWERS[curve]
    c2 = pr.G2_CURVE[curve]
    pb1, pb2 = bb.point_bytes(curve), bb.point_bytes(c2)
    assert pb1 == bb.CURVE_SIZES[curve][0] == t.g1_proj_struct(None).size
    assert pb2 == bb.CURVE_SIZES[c2][0] == t.g2_proj_struct(None).size
    n, m = 500, 6
    rng = np.random.default_rng(10 + curve)
    s1 = rng.integers(0, 256, (m, n, 32), dtype=np.uint8)
    s2 = rng.integers(0, 256, (m, n, 16), dtype=np.uint8)
    s1[2] = 0
    s2[2] = 0
    gens1 = bb.synthetic_generators(curve, n)
    gens2 = bb.synthetic_generators(c2, n, G2_FIRST)
    bufs = [bb.DeviceBuffer(host=gens1), bb.DeviceBuffer(host=gens2)]
    bufs += [bb.DeviceBuffer(host=s1[j]) for j in range(m)] + [bb.DeviceBuffer(host=s2[j]) for j in range(m)]
    p1, p2, out = bb.DeviceBuffer(m * pb1), bb.DeviceBuffer(m * pb2), bb.DeviceBuffer(2 * t.GT_BYTES)
    try:
        bb.commit_device(curve, [(n, 32, 0)] * m, [b.ptr for b in bufs[2:2 + m]], bufs[0].ptr, None, p1.ptr)
        bb.commit_device(c2, [(n, 16, 0)] * m, [b.ptr for b in bufs[2 + m:]], bufs[1].ptr, None, p2.ptr)
        bb.multi_pairing_device(curve, out.ptr, [4, 2], p1.ptr, p2.ptr)
        got = out.to_host((2, t.GT_BYTES))
    finally:
        for b in bufs + [p1, p2, out]:
            b.free()
    k1, k2 = common.synth_scalars_k(n), common.synth_scalars_k(n, G2_FIRST)
    v = [common.dot_mod(s1[j], k1, t.R) * common.dot_mod(s2[j], k2, t.R) for j in range(m)]
    assert [g.tobytes() for g in got] == [gt(curve, sum(v[:4])), gt(curve, sum(v[4:]))]
