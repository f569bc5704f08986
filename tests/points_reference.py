"""TEST INFRASTRUCTURE — pure-Python point validation and decoding for curves 1-5, the oracle of the
point-check tests. Never imported by the product.

Every curve is y^2 = x^3 + b over Fp (curves 1-3) or Fp2 = Fp[u] / (u^2 + 1) (curves 4 and 5), its
coordinates held as pairs (c0, c1) in both cases (c1 = 0 over Fp). The ground truth of subgroup
membership is [r] P = O. The endomorphism checks the device uses are written out here as well, only so
that a test can confirm they agree with [r] P. Square roots take a different route from the device:
a^((p+1)/4) or Tonelli-Shanks in Fp, and the norm method in Fp2, each checked by squaring.

Group orders n = h r of the curves with a cofactor, with the small prime factors of h:
  bls12-381 G1: h = (x - 1)^2 / 3 = 3 * 11^2 * 10177^2 * 859267^2 * 52437899^2;
  bls12-381 G2: h = 13^2 * 23^2 * 2713 * 11953 * 262069 * (a large prime);
  bn254 G2:     h = 2p - r = 10069 * 5864401 * 1875725156269 * (a large prime)."""
import random

import numpy as np

from tests import common
from tests import g2_reference as bls_g2
from tests.bn254_g2_reference import BN as BN_G2

BLS_X = -0xd201000000010000
BN_X = 0x44e992b44a6909f1
ZERO, ONE = (0, 0), (1, 0)


class Curve:
    """One curve: id, p, r, b (pair), generator, components per coordinate (1 or 2), bytes per Fp
    component in the ABI structs, the cofactor h and the small primes dividing it."""

    def __init__(self, cid, p, r, b, g, parts, width, h, small):
        self.ID, self.P, self.R, self.B, self.G = cid, p, r, b, g
        self.PARTS, self.W, self.H, self.SMALL = parts, width, h, small
        self.MONT = 1 << (8 * width)
        self.N = h * r  # the group order
        self.COORD = parts * width  # bytes of one coordinate
        self.PROJ_BYTES = 3 * self.COORD
        self.COMPRESSED = cid in (1, 4)
        self.COMMIT_BYTES = self.COORD if self.COMPRESSED else 2 * self.COORD + 8

    # ---- Fp2 (pairs) ---------------------------------------------------------------------------------
    def add(self, a, b):
        return ((a[0] + b[0]) % self.P, (a[1] + b[1]) % self.P)

    def sub(self, a, b):
        return ((a[0] - b[0]) % self.P, (a[1] - b[1]) % self.P)

    def neg(self, a):
        return (-a[0] % self.P, -a[1] % self.P)

    def mul(self, a, b):
        P = self.P
        return ((a[0] * b[0] - a[1] * b[1]) % P, (a[0] * b[1] + a[1] * b[0]) % P)

    def sqr(self, a):
        return self.mul(a, a)

    def inv(self, a):
        n = pow((a[0] * a[0] + a[1] * a[1]) % self.P, self.P - 2, self.P)
        return (a[0] * n % self.P, -a[1] * n % self.P)

    def pow(self, a, e):
        acc = ONE
        for bit in bin(e)[2:]:
            acc = self.mul(acc, acc)
            if bit == "1":
                acc = self.mul(acc, a)
        return acc

    def conj(self, a):
        return (a[0], -a[1] % self.P)

    def rand_elem(self, rng):
        return (rng.randrange(self.P), rng.randrange(self.P) if self.PARTS == 2 else 0)

    def sqrt(self, a):
        """A square root of a, or None for a non-square."""
        P = self.P
        if self.PARTS == 1 or a[1] == 0:
            r = sqrt_fp(a[0], P)
            if r is not None:
                return (r, 0)
            if self.PARTS == 1:
                return None
            r = sqrt_fp(-a[0] % P, P)  # a0 = -(r^2) = (r u)^2
            return (0, r)
        n = sqrt_fp((a[0] * a[0] + a[1] * a[1]) % P, P)  # the norm of a root
        if n is None:
            return None
        half = pow(2, -1, P)
        for s in (n, P - n):
            x0 = sqrt_fp((a[0] + s) * half % P, P)
            if x0:
                x = (x0, a[1] * pow(2 * x0, -1, P) % P)
                if self.sqr(x) == a:
                    return x
        return None

    def lex_largest(self, a):
        half = (self.P - 1) // 2
        return a[1] > half if a[1] else a[0] > half

    # ---- points: affine pairs of elements, None the identity ----------------------------------------------
    def on_curve(self, pt):
        if pt is None:
            return True
        return self.sqr(pt[1]) == self.add(self.mul(self.sqr(pt[0]), pt[0]), self.B)

    def _jdbl(self, j):
        if j is None or j[1] == ZERO:
            return None
        add, sub, mul, sqr = self.add, self.sub, self.mul, self.sqr
        X, Y, Z = j
        A, B = sqr(X), sqr(Y)
        C = sqr(B)
        D = sub(sqr(add(X, B)), add(A, C))
        D = add(D, D)
        E = add(add(A, A), A)
        X3 = sub(sqr(E), add(D, D))
        C8 = add(C, C)
        C8 = add(C8, C8)
        C8 = add(C8, C8)
        Y3 = sub(mul(E, sub(D, X3)), C8)
        Z3 = mul(Y, Z)
        return (X3, Y3, add(Z3, Z3))

    def _jadd(self, p, q):
        if p is None or q is None:
            return q if p is None else p
        add, sub, mul, sqr = self.add, self.sub, self.mul, self.sqr
        X1, Y1, Z1 = p
        X2, Y2, Z2 = q
        z1z1, z2z2 = sqr(Z1), sqr(Z2)
        U1, U2 = mul(X1, z2z2), mul(X2, z1z1)
        S1, S2 = mul(Y1, mul(Z2, z2z2)), mul(Y2, mul(Z1, z1z1))
        if U1 == U2:
            return self._jdbl(p) if S1 == S2 else None
        H, r = sub(U2, U1), sub(S2, S1)
        HH = sqr(H)
        HHH = mul(H, HH)
        V = mul(U1, HH)
        X3 = sub(sub(sqr(r), HHH), add(V, V))
        Y3 = sub(mul(r, sub(V, X3)), mul(S1, HHH))
        return (X3, Y3, mul(mul(Z1, Z2), H))

    def _affine(self, j):
        if j is None:
            return None
        zi = self.inv(j[2])
        zi2 = self.sqr(zi)
        return (self.mul(j[0], zi2), self.mul(j[1], self.mul(zi2, zi)))

    def point_add(self, a, b):
        jac = [None if t is None else (t[0], t[1], ONE) for t in (a, b)]
        return self._affine(self._jadd(*jac))

    def point_neg(self, a):
        return None if a is None else (a[0], self.neg(a[1]))

    def mul_point(self, k, pt):
        """[k] pt for any integer k."""
        if pt is None or k == 0:
            return None
        if k < 0:
            k, pt = -k, self.point_neg(pt)
        acc, base = None, (pt[0], pt[1], ONE)
        for bit in bin(k)[2:]:
            acc = self._jdbl(acc)
            if bit == "1":
                acc = self._jadd(acc, base)
        return self._affine(acc)

    def in_subgroup(self, pt):
        """The ground truth: [r] P = O."""
        return self.mul_point(self.R, pt) is None

    def endo_check(self, pt):
        """The device's endomorphism check for a point on the curve (True for the prime-order curves)."""
        if pt is None or self.H == 1:
            return True
        x, y = pt
        if self.ID == 1:  # phi(P) = (beta x, y) = [-x^2] P
            beta = pow(2, (self.P - 1) // 3, self.P)
            return (self.mul((beta, 0), x), y) == self.mul_point(-BLS_X * BLS_X, pt)
        if self.ID == 4:  # psi(Q) = [x] Q
            cx = self.inv(self.pow((1, 1), (self.P - 1) // 3))
            cy = self.inv(self.pow((1, 1), (self.P - 1) // 2))
            return (self.mul(self.conj(x), cx), self.mul(self.conj(y), cy)) == self.mul_point(BLS_X, pt)
        gx, gy = self.pow((9, 1), (self.P - 1) // 3), self.pow((9, 1), (self.P - 1) // 2)  # ID 5
        return (self.mul(self.conj(x), gx), self.mul(self.conj(y), gy)) == \
            self.mul_point(6 * BN_X * BN_X, pt)

    def valid(self, pt):
        return self.on_curve(pt) and self.in_subgroup(pt)

    # ---- point sets ---------------------------------------------------------------------------------
    def random_on_curve(self, rng):
        """A uniformly random affine point of E (mostly outside the subgroup when h > 1)."""
        while True:
            x = self.rand_elem(rng)
            y = self.sqrt(self.add(self.mul(self.sqr(x), x), self.B))
            if y is not None:
                return (x, y if rng.random() < 0.5 else self.neg(y))

    def random_subgroup(self, rng):
        return self.mul_point(rng.randrange(1, self.R), self.G)

    def of_order(self, q, rng):
        """A point of prime order q dividing h: t = [n / q^e] T for random T (q^e the power of q in
        n), then [q] t while that is not O, until t is not O."""
        assert self.H % q == 0
        m = self.N
        while m % q == 0:
            m //= q
        while True:
            t = self.mul_point(m, self.random_on_curve(rng))
            while t is not None and self.mul_point(q, t) is not None:
                t = self.mul_point(q, t)
            if t is not None:
                return t

    def large_cofactor_prime(self):
        """h without its small primes (bls12-381 G2 and bn254 G2)."""
        h = self.H
        for q in self.SMALL:
            while h % q == 0:
                h //= q
        return h

    # ---- ABI bytes ---------------------------------------------------------------------------------------
    def coord_bytes(self, a, mont=True):
        """One coordinate's ABI bytes: each component as Montgomery limbs (mont) or as given (raw)."""
        vals = [v * self.MONT % self.P if mont else v for v in a[:self.PARTS]]
        return b"".join(v.to_bytes(self.W, "little") for v in vals)

    def proj_struct(self, pt, z=ONE):
        """The *_p2 struct of pt scaled by z; the identity is {0, 1, 0}."""
        coords = (ZERO, ONE, ZERO) if pt is None else (self.mul(pt[0], z), self.mul(pt[1], z), z)
        return np.frombuffer(b"".join(self.coord_bytes(c) for c in coords), np.uint8).copy()

    def raw_proj_struct(self, coords):
        """A *_p2 struct from three coordinates of raw Montgomery limb values (anything below
        2^(8 W), also p and above)."""
        return np.frombuffer(b"".join(self.coord_bytes(c, False) for c in coords), np.uint8).copy()

    def from_proj_struct(self, row):
        """(X, Y, Z) as plain field values of a struct's Montgomery limbs."""
        raw, w = bytes(np.asarray(row, np.uint8)), self.W
        inv_r = pow(self.MONT, -1, self.P)
        vals = [int.from_bytes(raw[w * i:w * (i + 1)], "little") * inv_r % self.P
                for i in range(3 * self.PARTS)]
        if self.PARTS == 1:
            return tuple((v, 0) for v in vals)
        return tuple((vals[2 * i], vals[2 * i + 1]) for i in range(3))

    def decoded_struct(self, pt):
        """What decoding writes for pt: {x R, y R, R}, the identity {0, R, 0}."""
        return self.proj_struct(pt)

    def compress(self, pt):
        """The zcash compressed encoding (curves 1 and 4)."""
        if pt is None:
            return bytes([0xC0]) + bytes(self.COORD - 1)
        x = pt[0]
        value = x[0] if self.PARTS == 1 else x[0] + (x[1] << 384)
        out = bytearray(value.to_bytes(self.COORD, "big"))
        out[0] |= 0x80 | (0x20 if self.lex_largest(pt[1]) else 0)
        return bytes(out)

    def affine_struct(self, pt, infinity=None, pad=b""):
        """The affine commitment struct {X, Y, u8 infinity, pad} (curves 2, 3, 5); the identity as the
        library writes it, {0, 1, 1}; pad fills the 7 bytes after the flag."""
        x, y = (ZERO, ONE) if pt is None else pt
        flag = (1 if pt is None else 0) if infinity is None else infinity
        body = self.coord_bytes(x) + self.coord_bytes(y) + bytes([flag]) + (pad + bytes(7))[:7]
        return np.frombuffer(body, np.uint8).copy()

    def encode(self, pt):
        """The commitment encoding of pt."""
        if self.COMPRESSED:
            return np.frombuffer(self.compress(pt), np.uint8).copy()
        return self.affine_struct(pt)

    def decompress(self, raw):
        """(ok, point) of a zcash compressed encoding, by the rules of b200_decode_points."""
        raw = bytes(raw)
        flags = raw[0]
        v = int.from_bytes(bytes([raw[0] & 0x1F]) + raw[1:], "big")
        if not flags & 0x80:
            return False, None
        if flags & 0x40:
            return (not flags & 0x20 and v == 0), None
        x = (v, 0) if self.PARTS == 1 else (v & ((1 << 384) - 1), v >> 384)
        if x[0] >= self.P or x[1] >= self.P:
            return False, None
        y = self.sqrt(self.add(self.mul(self.sqr(x), x), self.B))
        if y is None:
            return False, None
        if self.lex_largest(y) != bool(flags & 0x20):
            y = self.neg(y)
        pt = (x, y)
        return self.in_subgroup(pt), pt

    def decode_affine(self, raw):
        """(ok, point) of an affine struct, by the rules of b200_decode_points."""
        raw = bytes(raw)
        flag = raw[2 * self.COORD]
        if flag == 1:
            return True, None
        if flag != 0:
            return False, None
        inv_r = pow(self.MONT, -1, self.P)
        comps = [int.from_bytes(raw[self.W * i:self.W * (i + 1)], "little")
                 for i in range(2 * self.PARTS)]
        if any(c >= self.P for c in comps):
            return False, None
        vals = [c * inv_r % self.P for c in comps]
        pt = ((vals[0], 0), (vals[1], 0)) if self.PARTS == 1 else \
            ((vals[0], vals[1]), (vals[2], vals[3]))
        return self.valid(pt), pt

    def decode(self, raw):
        """(ok, expected output struct) of one commitment encoding."""
        ok, pt = self.decompress(raw) if self.COMPRESSED else self.decode_affine(raw)
        return ok, self.decoded_struct(pt if ok else None)


def sqrt_fp(a, p):
    """A square root of a in Fp, or None: a^((p+1)/4) for p = 3 mod 4 (bls12-381, bn254),
    Tonelli-Shanks otherwise (the Grumpkin field)."""
    a %= p
    if p % 4 == 3:
        r = pow(a, (p + 1) // 4, p)
    elif a == 0 or pow(a, (p - 1) // 2, p) != 1:
        r = 0
    else:
        q, e = p - 1, 0
        while q % 2 == 0:
            q, e = q // 2, e + 1
        z = 2
        while pow(z, (p - 1) // 2, p) != p - 1:
            z += 1
        c, t, r = pow(z, q, p), pow(a, q, p), pow(a, (q + 1) // 2, p)
        while t != 1:
            i, t2 = 0, t
            while t2 != 1:
                t2, i = t2 * t2 % p, i + 1
            b = pow(c, 1 << (e - i - 1), p)
            e, c, t, r = i, b * b % p, t * b * b % p, r * b % p
    return r if r * r % p == a else None


def _g1(v):
    return (v, 0)


BLS_H1 = (BLS_X - 1) ** 2 // 3
BLS_H2 = (BLS_X ** 8 - 4 * BLS_X ** 7 + 5 * BLS_X ** 6 - 4 * BLS_X ** 4 + 6 * BLS_X ** 3
          - 4 * BLS_X ** 2 - 4 * BLS_X + 13) // 9
BN_H2 = 2 * common.BN254_Q - common.BN254_R

CURVES = {
    1: Curve(1, common.BLS_Q, common.BLS_R, (4, 0), (_g1(common.BLS_GX), _g1(common.BLS_GY)), 1, 48,
             BLS_H1, (3, 11, 10177, 859267, 52437899)),
    2: Curve(2, common.BN254_Q, common.BN254_R, (3, 0), (_g1(1), _g1(2)), 1, 32, 1, ()),
    3: Curve(3, common.BN254_R, common.BN254_Q, (-17 % common.BN254_R, 0),
             (_g1(1), _g1(common.curve_params(3)[4])), 1, 32, 1, ()),
    4: Curve(4, common.BLS_Q, common.BLS_R, bls_g2.B2, bls_g2.G, 2, 48, BLS_H2,
             (13, 23, 2713, 11953, 262069)),
    5: Curve(5, BN_G2.P, BN_G2.R_ORDER, BN_G2.B2, BN_G2.G, 2, 32, BN_H2,
             (10069, 5864401, 1875725156269)),
}


def rng_for(curve, salt=0):
    return random.Random(1000 * curve + salt)
