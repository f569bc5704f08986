"""Pairing products (b200_multi_pairing, pairing.cuh) on the CPU emulation of the product's kernel bodies,
against the pure-Python oracle tests/pairing_reference.py: the oracle's own properties, the Fp12
arithmetic of b200_field_op fields 8 and 9, and multi-pairings of generators, random points,
identities, empty products and mixed lengths. The check_* functions take the entry under test, so
that tests/test_gpu_pairing.py runs the same cases through the C ABI."""
import random

import numpy as np
import pytest

from tests import pairing_reference as pr
from tests.emul import pairing as emul_pairing

CURVES = (1, 2)
FIELD = {1: 8, 2: 9}


def rand_fp12(t, rng):
    return tuple((rng.randrange(t.P), rng.randrange(t.P)) for _ in range(6))


def edge_fp12(t):
    """Elements whose components sit at 0, 1 and p - 1."""
    p = t.P
    return [t.ONE, tuple(((p - 1, p - 1),) * 6), tuple(((1, p - 1), (p - 1, 0)) * 3),
            tuple(((0, 1),) * 6), ((0, 0),) * 5 + ((p - 1, 1),)]


def easy_part(t, a):
    """a^((p^6 - 1)(p^2 + 1)): an element of the cyclotomic subgroup."""
    f = t.mul(t.frobenius(a, 6), t.inv(a))
    return t.mul(t.frobenius(f, 2), f)


def point_pair(t, a, b, z1=1, z2=(1, 0)):
    """(g1 struct, g2 struct, (P, Q)) for P = a G1, Q = b G2 with projective scalings z1, z2."""
    P, Q = t.g1_mul(a), t.g2_mul(b)
    return t.g1_proj_struct(P, z1), t.g2_proj_struct(Q, z2), (P, Q)


def expected(t, lengths, pts):
    """Oracle bytes of each product of consecutive pairs."""
    out, i = [], 0
    for n in lengths:
        out.append(t.to_bytes(t.pairing_product(pts[i:i + n])))
        i += n
    return out


def run(multi_pairing, curve, pairs, lengths):
    t = pr.TOWERS[curve]
    w1 = t.g1_proj_struct(None).size
    w2 = t.g2_proj_struct(None).size
    g1 = np.array([p[0] for p in pairs], np.uint8).reshape(-1, w1)
    g2 = np.array([p[1] for p in pairs], np.uint8).reshape(-1, w2)
    return multi_pairing(curve, g1, g2, lengths)


# ---- shared checks ---------------------------------------------------------------------------------
def check_fp12_ops(field_op, curve):
    """add, sub, neg, mul, sqr, invert and frobenius on random and edge elements, cyclotomic_sqr on
    cyclotomic ones, and final_exp, each against the oracle."""
    t = pr.TOWERS[curve]
    rng = random.Random(curve)
    xs = edge_fp12(t) + [rand_fp12(t, rng) for _ in range(6)]
    ys = xs[1:] + xs[:1]
    A = np.stack([t.to_limbs(x) for x in xs])
    B = np.stack([t.to_limbs(y) for y in ys])
    f = FIELD[curve]

    def got(op, a, b=None):
        return [t.from_limbs(r) for r in field_op(f, op, a, b)]
    assert got("add", A, B) == [t.add(x, y) for x, y in zip(xs, ys)]
    assert got("sub", A, B) == [t.sub(x, y) for x, y in zip(xs, ys)]
    assert got("neg", A) == [t.neg(x) for x in xs]
    assert got("mul", A, B) == [t.mul(x, y) for x, y in zip(xs, ys)]
    assert got("sqr", A) == [t.mul(x, x) for x in xs]
    assert got("invert", A) == [t.inv(x) for x in xs]
    assert got("frobenius", A) == [t.frobenius(x) for x in xs]
    cyc = [easy_part(t, x) for x in xs[-3:]]
    assert got("cyclotomic_sqr", np.stack([t.to_limbs(c) for c in cyc])) == [t.mul(c, c) for c in cyc]
    fin = xs[-2:]
    assert got("final_exp", np.stack([t.to_limbs(x) for x in fin])) == [t.final_exp(x) for x in fin]


def check_generators(multi_pairing, curve):
    """e(G1, G2) byte for byte, with the inputs scaled projectively."""
    t = pr.TOWERS[curve]
    g1, g2, pts = point_pair(t, 1, 1, 5, (3, 7))
    got = run(multi_pairing, curve, [(g1, g2)], [1])
    assert got[0].tobytes() == t.to_bytes(t.pairing(t.G1, t.G2.G))


def check_random_pairs(multi_pairing, curve):
    """Three single pairings of random multiples of the generators, in one call."""
    t = pr.TOWERS[curve]
    rng = random.Random(10 + curve)
    pairs, pts = [], []
    for _ in range(3):
        g1, g2, pq = point_pair(t, rng.randrange(1, t.R), rng.randrange(1, t.R),
                                rng.randrange(1, t.P), (rng.randrange(t.P), rng.randrange(t.P)))
        pairs.append((g1, g2))
        pts.append(pq)
    got = run(multi_pairing, curve, pairs, [1, 1, 1])
    assert [g.tobytes() for g in got] == expected(t, [1, 1, 1], pts)


def check_identities_and_empty(multi_pairing, curve):
    """A pair with the identity on either side contributes 1; an empty product is 1; a product of
    identities only is 1."""
    t = pr.TOWERS[curve]
    one = t.to_bytes(t.ONE)
    g1, g2, pq = point_pair(t, 3, 5)
    i1, i2 = t.g1_proj_struct(None), t.g2_proj_struct(None)
    pairs = [(i1, g2), (g1, i2), (i1, i2), (g1, g2), (i1, g2)]
    got = run(multi_pairing, curve, pairs, [0, 1, 1, 0, 2, 1, 0])
    e = t.to_bytes(t.pairing(*pq))
    assert [g.tobytes() for g in got] == [one, one, one, one, e, one, one]
    assert run(multi_pairing, curve, [], [0, 0]).tolist() == [list(one)] * 2
    assert run(multi_pairing, curve, [], []).shape == (0, t.GT_BYTES)


def check_mixed_lengths(multi_pairing, curve):
    """Products of 0, 1, 2 and 5 pairs in one call."""
    t = pr.TOWERS[curve]
    rng = random.Random(20 + curve)
    lengths = [0, 1, 2, 5]
    pairs, pts = [], []
    for _ in range(sum(lengths)):
        g1, g2, pq = point_pair(t, rng.randrange(1, 1 << 64), rng.randrange(1, 1 << 64))
        pairs.append((g1, g2))
        pts.append(pq)
    got = run(multi_pairing, curve, pairs, lengths)
    assert [g.tobytes() for g in got] == expected(t, lengths, pts)


def check_relation(multi_pairing, curve):
    """e(aG, bH) e(-ab G, H) = 1, the shape of a pairing check."""
    t = pr.TOWERS[curve]
    rng = random.Random(30 + curve)
    a, b = rng.randrange(1, t.R), rng.randrange(1, t.R)
    p1, q1, _ = point_pair(t, a, b, 11)
    p2, q2, _ = point_pair(t, -a * b, 1, 1, (2, 9))
    got = run(multi_pairing, curve, [(p1, q1), (p2, q2)], [2])
    assert got[0].tobytes() == t.to_bytes(t.ONE)


CHECKS = [check_generators, check_random_pairs, check_identities_and_empty, check_mixed_lengths,
          check_relation]


# ---- the oracle --------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES)
def test_oracle_nondegenerate_of_order_r_and_bilinear(curve):
    t = pr.TOWERS[curve]
    e = t.pairing(t.G1, t.G2.G)
    assert e != t.ONE and t.pow(e, t.R) == t.ONE
    rng = random.Random(curve)
    a, b = rng.randrange(1, t.R), rng.randrange(1, t.R)
    assert t.pairing(t.g1_mul(a), t.g2_mul(b)) == t.pow(e, a * b % t.R)


@pytest.mark.parametrize("curve", CURVES)
def test_hard_part_decompositions(curve):
    """lambda_0 + lambda_1 p + lambda_2 p^2 + lambda_3 p^3 = (p^4 - p^2 + 1) / r for the decompositions
    the device's final exponentiation uses."""
    t = pr.TOWERS[curve]
    p, x = t.P, t.X
    if curve == 1:
        l3 = (x - 1) ** 2 // 3
        assert (x - 1) ** 2 % 3 == 0 and l3.bit_length() == 126
        l2 = l3 * x
        l1 = l2 * x - l3
        l0 = l1 * x + 1
    else:
        l3, l2 = 1, 6 * x * x + 1
        l1 = -36 * x ** 3 - 18 * x ** 2 - 12 * x + 1
        l0 = -36 * x ** 3 - 30 * x ** 2 - 18 * x - 2
    assert (p ** 4 - p ** 2 + 1) % t.R == 0
    assert l0 + l1 * p + l2 * p ** 2 + l3 * p ** 3 == (p ** 4 - p ** 2 + 1) // t.R


# ---- the emulated kernels ---------------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES)
def test_fp12_field_ops(emul, curve):
    check_fp12_ops(emul.field_op, curve)


@pytest.mark.parametrize("check", CHECKS, ids=[c.__name__[6:] for c in CHECKS])
@pytest.mark.parametrize("curve", CURVES)
def test_multi_pairing(curve, check):
    check(emul_pairing.multi_pairing, curve)
