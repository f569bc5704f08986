"""Point validation and decoding (b200_check_points, b200_decode_points, points.cuh) on the CPU emulation
of the product's kernel bodies, against the pure-Python oracle tests/points_reference.py, whose ground
truth for the subgroup is [r] P = O. The check_* functions take the entries under test (Entries), so
that tests/test_gpu_points.py runs the same cases through the C ABI.

Covered: identities (also Z = 0 with arbitrary X and Y), generators, their negations and random
subgroup points at random projective scalings; coordinates at p, p + 1, 2^(64 limbs) - 1 and X + p in
each Fp component, and Y + 1; points of every small prime order dividing the cofactor, alone and
added to G, points of the large cofactor prime's order and uniformly random curve points; the
library's own commitments decoding byte for byte; every flag rule of both bls12-381 encodings, x = p
and x = 2^381 - 1, x with a non-square right-hand side; infinity bytes 0, 1 and 2 with garbage padding;
and the bls12-381 Fp / Fp2 square roots of b200_field_op op 27."""
import functools
import random

import numpy as np
import pytest

from blitzar_b200.api import FIELD_LIMBS
from tests import points_reference as pref
from tests import test_field_arithmetic as fa
from tests.emul import points as emul_points
from tests.test_bls12_381_g2 import fp2_operands

CURVES = (1, 2, 3, 4, 5)
COFACTOR_CURVES = (1, 4, 5)


class Entries:
    """The calls under test. check(curve, p2) -> (valid, count); decode(curve, encoded) -> (p2,
    valid, count); commit(curve, columns, generators) -> commitments; synth(curve, n, first,
    projective) -> synthetic generators; field_op as b200_field_op."""

    def __init__(self, check, decode, commit, synth, field_op):
        self.check, self.decode, self.commit, self.synth = check, decode, commit, synth
        self.field_op = field_op


def emul_entries(emul):
    return Entries(emul_points.check_points, emul_points.decode_points, emul.commit,
                   emul.synth_generators, emul.field_op)


# ---- point sets ------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def valid_points(curve):
    """The identity, G, -G and random subgroup points."""
    c = pref.CURVES[curve]
    rng = pref.rng_for(curve, 1)
    return [None, c.G, c.point_neg(c.G)] + [c.random_subgroup(rng) for _ in range(5)]


@functools.lru_cache(maxsize=None)
def outside_points(curve):
    """Points on the curve outside the order-r subgroup: of each small prime order q | h, alone and
    as G + T; of the large cofactor prime's order (G2); uniformly random curve points."""
    c = pref.CURVES[curve]
    rng = pref.rng_for(curve, 2)
    out = []
    for q in c.SMALL:
        t = c.of_order(q, rng)
        out += [t, c.point_add(c.G, t)]
    large = c.large_cofactor_prime()
    if large > 1:
        out += [c.of_order(large, rng) for _ in range(2)]
    return out + [c.random_on_curve(rng) for _ in range(4)]


def structs(c, pts, rng):
    """*_p2 structs of the points at random projective scalings."""
    return np.stack([c.proj_struct(p, c.rand_elem(rng) if p is not None else pref.ONE) for p in pts])


def run_check(e, curve, rows, want):
    valid, count = e.check(curve, rows)
    assert valid.tolist() == [int(w) for w in want]
    assert count == int(np.sum(want))


# ---- shared checks ---------------------------------------------------------------------------------
def check_valid_points(e, curve):
    """The identity (also Z = 0 with arbitrary X and Y below p), generators, negations and random
    subgroup points at random scalings all pass."""
    c = pref.CURVES[curve]
    rng = pref.rng_for(curve, 3)
    rows = [structs(c, valid_points(curve), rng)]
    rows.append(c.raw_proj_struct([c.rand_elem(rng), c.rand_elem(rng), pref.ZERO])[None])
    rows.append(c.raw_proj_struct([(c.P - 1, c.P - 1), (0, 0), pref.ZERO])[None])
    rows = np.concatenate(rows)
    run_check(e, curve, rows, [1] * len(rows))


def check_bad_coordinates(e, curve):
    """p, p + 1, 2^(64 limbs) - 1 and X + p in each component of each coordinate, of a valid point and
    of the identity (the range check comes first), and Y + 1 all fail."""
    c = pref.CURVES[curve]
    rng = pref.rng_for(curve, 4)
    good = c.proj_struct(c.random_subgroup(rng), c.rand_elem(rng))
    ident = c.proj_struct(None)
    top = c.MONT - 1
    rows = []
    for base in (good, ident):
        for coord in range(3):
            for part in range(c.PARTS):
                off = coord * c.COORD + part * c.W
                cur = int.from_bytes(bytes(base[off:off + c.W]), "little")
                for v in (c.P, c.P + 1, top, cur + c.P):
                    row = base.copy()
                    row[off:off + c.W] = np.frombuffer(v.to_bytes(c.W, "little"), np.uint8)
                    rows.append(row)
    y1 = good.copy()
    y = int.from_bytes(bytes(y1[c.COORD:c.COORD + c.W]), "little")
    y1[c.COORD:c.COORD + c.W] = np.frombuffer(((y + 1) % c.P).to_bytes(c.W, "little"), np.uint8)
    rows.append(y1)
    rows.append(good)  # the control
    run_check(e, curve, np.stack(rows), [0] * (len(rows) - 1) + [1])


def check_outside_subgroup(e, curve):
    """Points of the small orders dividing the cofactor, alone and added to G, of the large cofactor
    prime's order, and random curve points fail; the oracle agrees that none of them is in G."""
    c = pref.CURVES[curve]
    pts = outside_points(curve)
    assert all(c.on_curve(p) and not c.in_subgroup(p) for p in pts)
    rows = structs(c, pts, pref.rng_for(curve, 5))
    run_check(e, curve, rows, [0] * len(pts))


def check_prime_order_curve(e, curve):
    """On bn254 G1 and Grumpkin every curve point passes: random x with a square x^3 + b."""
    c = pref.CURVES[curve]
    rng = pref.rng_for(curve, 6)
    pts = [c.random_on_curve(rng) for _ in range(6)]
    assert all(c.in_subgroup(p) for p in pts)
    run_check(e, curve, structs(c, pts, rng), [1] * len(pts))


def run_decode(e, curve, encoded):
    """Decodes the rows and compares each output struct and flag with the oracle."""
    c = pref.CURVES[curve]
    encoded = np.stack([np.frombuffer(bytes(r), np.uint8) for r in encoded])
    p2, valid, count = e.decode(curve, encoded)
    want = [c.decode(r) for r in encoded]
    assert valid.tolist() == [int(ok) for ok, _ in want]
    assert count == sum(ok for ok, _ in want)
    for got, (_, exp) in zip(p2, want):
        assert got.tobytes() == exp.tobytes()
    return valid


def check_decode_commitments(e, curve):
    """The library's own commitments of random columns (and of a zero column) decode to the oracle's
    structs byte for byte, with Z = R, and all pass."""
    c = pref.CURVES[curve]
    n = 24
    gens = e.synth(curve, n, 0, False)
    rng = np.random.default_rng(curve)
    cols = [(rng.integers(0, 256, (n, 32), dtype=np.uint8), 0) for _ in range(5)]
    cols.append((np.zeros((n, 8), np.uint8), 0))
    com = e.commit(curve, cols, gens)
    valid = run_decode(e, curve, com)
    assert valid.tolist() == [1] * len(cols)
    p2, _, _ = e.decode(curve, com)
    one = c.coord_bytes(pref.ONE)
    assert all(row[2 * c.COORD:].tobytes() == one for row in p2[:-1])


def check_decode_compressed_flags(e, curve):
    """bls12-381 encodings: every flag rule, x = p and x = 2^381 - 1 in each half, x with a
    non-square right-hand side under both signs, and compressed points outside the subgroup."""
    c = pref.CURVES[curve]
    rng = pref.rng_for(curve, 7)
    g = bytearray(c.compress(c.G))
    rows = [bytes(g)]
    flipped = bytearray(g)
    flipped[0] ^= 0x20  # the other root: -G, valid
    rows.append(bytes(flipped))
    no_c = bytearray(g)
    no_c[0] &= 0x7F  # uncompressed forms are not accepted
    rows.append(bytes(no_c))
    ident = bytearray(c.compress(None))
    rows.append(bytes(ident))
    for flag, pos, bit in ((0x20, 0, 0), (0, c.COORD - 1, 1), (0, 0, 0x10), (0, c.COORD // 2, 4)):
        r = bytearray(ident)  # the identity with the sign flag or another bit set
        r[0] |= flag
        r[pos] |= bit
        rows.append(bytes(r))
    ident_no_c = bytearray(ident)
    ident_no_c[0] &= 0x7F
    rows.append(bytes(ident_no_c))
    halves = [0] if c.PARTS == 1 else [0, 48]  # x.c1 then x.c0
    for start in halves:
        for v in (c.P, (1 << 381) - 1):
            r = bytearray(g)
            r[start:start + 48] = v.to_bytes(48, "big")
            r[0] |= 0x80 | (g[0] & 0x20)
            rows.append(bytes(r))
    found = 0
    while found < 2:  # x without a point: x^3 + b is not a square
        x = c.rand_elem(rng)
        if c.sqrt(c.add(c.mul(c.sqr(x), x), c.B)) is None:
            for sign in (0, 0x20):
                r = bytearray(c.compress((x, pref.ONE)))
                r[0] = (r[0] & 0x9F) | sign
                rows.append(bytes(r))
            found += 1
    rows += [c.compress(p) for p in outside_points(curve)]
    rows += [c.compress(p) for p in valid_points(curve)]
    valid = run_decode(e, curve, rows)
    assert valid[:2].tolist() == [1, 1] and valid[2] == 0 and valid[3] == 1
    assert valid[4:].sum() == len(valid_points(curve))


def check_decode_affine(e, curve):
    """Affine structs: infinity 0 (a point), 1 (the identity, whatever X and Y hold) and 2, each with
    garbage padding; coordinates >= p in each component; Y + 1; for bn254 G2 points outside G."""
    c = pref.CURVES[curve]
    rng = pref.rng_for(curve, 8)
    pts = valid_points(curve)[1:4]
    rows = []
    for p in pts:
        for flag in (0, 1, 2):
            rows.append(c.affine_struct(p, flag, bytes(rng.randrange(256) for _ in range(7))))
    rows.append(c.affine_struct(None, 1, b"\xff" * 7))
    base = c.affine_struct(pts[0])
    for coord in range(2):
        for part in range(c.PARTS):
            off = coord * c.COORD + part * c.W
            cur = int.from_bytes(bytes(base[off:off + c.W]), "little")
            for v in (c.P, c.P + 1, c.MONT - 1, cur + c.P):
                r = base.copy()
                r[off:off + c.W] = np.frombuffer(v.to_bytes(c.W, "little"), np.uint8)
                rows.append(r)
    y1 = base.copy()
    y = int.from_bytes(bytes(y1[c.COORD:c.COORD + c.W]), "little")
    y1[c.COORD:c.COORD + c.W] = np.frombuffer(((y + 1) % c.P).to_bytes(c.W, "little"), np.uint8)
    rows.append(y1)
    if curve in COFACTOR_CURVES:
        rows += [c.affine_struct(p) for p in outside_points(curve)]
    valid = run_decode(e, curve, rows)
    assert valid[:9].tolist() == [1, 1, 0] * 3 and valid[9] == 1 and valid[10:].sum() == 0


def check_sqrt(e, field):
    """sqrt (op 27) on fields 1 and 6 over the edge operands: r^2 = a, and the flag is Euler's
    criterion (the root is 0 for a non-square)."""
    c = pref.CURVES[1 if field == 1 else 4]
    P, R = c.P, c.MONT
    rinv = pow(R, -1, P)
    if field == 1:
        raw = fa.variants(fa.edge_values(P, 12) | {P, P + 1, R - 1, R - P}, 12)
        elems = sorted({v % P for v in raw})
        rng = random.Random(61)
        elems += [rng.randrange(P) for _ in range(64)]
        limbs = fa.to_limbs(elems, 12)
        vals = [(v * rinv % P, 0) for v in elems]
    else:
        elems, _, _ = fp2_operands(6)
        elems = elems[:-2048] + elems[-64:]  # every edge element and 64 random ones
        limbs = np.stack([np.frombuffer(a.to_bytes(48, "little") + b.to_bytes(48, "little"),
                                        np.uint32) for a, b in elems])
        vals = [(a * rinv % P, b * rinv % P) for a, b in elems]
    out = e.field_op(field, "sqrt", limbs)
    squares = 0
    for row, a in zip(out, vals):
        raw = np.ascontiguousarray(row[:-1]).tobytes()
        r = [int.from_bytes(raw[i * 48:(i + 1) * 48], "little") * rinv % P for i in range(c.PARTS)]
        r = (r[0], r[1] if c.PARTS == 2 else 0)
        euler = a == pref.ZERO or c.pow(a, (P ** c.PARTS - 1) // 2) == pref.ONE
        assert row[-1] == int(euler), a
        assert c.sqr(r) == a if euler else r == pref.ZERO, a
        squares += euler
    assert 0 < squares < len(vals)


CHECKS = [check_valid_points, check_bad_coordinates, check_decode_commitments]
COFACTOR_CHECKS = [check_outside_subgroup]
PRIME_ORDER_CHECKS = [check_prime_order_curve]
CASES = [(ch, cv) for ch in CHECKS for cv in CURVES] + \
    [(ch, cv) for ch in COFACTOR_CHECKS for cv in COFACTOR_CURVES] + \
    [(ch, cv) for ch in PRIME_ORDER_CHECKS for cv in (2, 3)] + \
    [(check_decode_compressed_flags, cv) for cv in (1, 4)] + \
    [(check_decode_affine, cv) for cv in (2, 3, 5)]
CASE_IDS = [f"{ch.__name__[6:]}-{cv}" for ch, cv in CASES]


# ---- the oracle ------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", COFACTOR_CURVES)
def test_endomorphism_checks_agree_with_r_torsion(curve):
    """The device's endomorphism checks, written in Python, agree with [r] P = O on every point set."""
    c = pref.CURVES[curve]
    pts = [p for p in valid_points(curve) + outside_points(curve) if p is not None]
    assert all(c.endo_check(p) == c.in_subgroup(p) for p in pts)
    assert sum(c.in_subgroup(p) for p in pts) == len(valid_points(curve)) - 1


@pytest.mark.parametrize("curve", COFACTOR_CURVES)
def test_cofactors(curve):
    """h r is the group order (odd), with the small primes of the module docstring dividing h."""
    c = pref.CURVES[curve]
    rng = pref.rng_for(curve, 9)
    assert c.N % 2 == 1 and c.mul_point(c.N, c.random_on_curve(rng)) is None
    assert all(c.H % q == 0 for q in c.SMALL)
    assert (c.large_cofactor_prime() == 1) == (curve == 1)  # bls12-381 G1: h has small primes only


# ---- the emulated kernels --------------------------------------------------------------------------
@pytest.mark.parametrize("check,curve", CASES, ids=CASE_IDS)
def test_points(emul, check, curve):
    check(emul_entries(emul), curve)


@pytest.mark.parametrize("field", (1, 6))
def test_sqrt(emul, field):
    check_sqrt(emul_entries(emul), field)


def test_sqrt_not_offered_elsewhere(emul):
    """Only fields 1 and 6 offer op 27."""
    for field in (2, 3, 7):
        with pytest.raises(ValueError):
            emul.field_op(field, "sqrt", np.zeros((1, FIELD_LIMBS[field]), np.uint32))
