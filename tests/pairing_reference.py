"""TEST INFRASTRUCTURE — pure-Python pairings over bls12-381 and bn254, the oracle of the pairing tests.
Never imported by the product.

Kept as plain as possible, so that it shares nothing with the device formulas: Fp12 = Fp2[w] / (w^6 - xi)
as six Fp2 coefficients of w^0 .. w^5, Q untwisted into E(Fp12) (bls12-381, M-type:
psi(x', y') = (x' w^-2, y' w^-3); bn254, D-type: psi(x', y') = (x' w^2, y' w^3)), affine
chord-and-tangent lines in Fp12 without the vertical lines (they lie in Fp6, which the final
exponentiation maps to 1), the Frobenius as pow(., p) and the final exponent (p^12 - 1) / r by one plain
pow. For bls12-381 the Miller value f_{|x|,Q}(P) is inverted rather than conjugated (x < 0): after the
final exponentiation the two agree.

The device layout c0.b0, c0.b1, c0.b2, c1.b0, c1.b1, c1.b2 (Fp12 = Fp6[w] / (w^2 - v), v = w^2) holds the
coefficients of w^0, w^2, w^4, w^1, w^3, w^5, each an Fp2 as Montgomery c0 then c1."""
import numpy as np

from tests import common
from tests import g2_reference as bls_g2
from tests.bn254_g2_reference import BN as bn_g2


class Tower:
    """One pairing: p, r, xi = xi0 + u, the G1 curve y^2 = x^3 + b1 with generator g1, the G2 oracle
    (affine points over Fp2 as (c0, c1)), and the Miller loop."""

    def __init__(self, p, r, xi0, b1, g1, g2, x, m_type, limbs):
        self.P, self.R, self.XI, self.B1, self.G1, self.G2, self.X = p, r, (xi0, 1), b1, g1, g2, x
        self.M_TYPE = m_type
        self.W = 8 * limbs  # bytes of one Fp
        self.MONT = 1 << (8 * self.W)
        self.GT_BYTES = 12 * self.W
        self.ONE = ((1, 0),) + ((0, 0),) * 5

    # ---- Fp2 -------------------------------------------------------------------------------------------
    def f2_add(self, a, b):
        return ((a[0] + b[0]) % self.P, (a[1] + b[1]) % self.P)

    def f2_sub(self, a, b):
        return ((a[0] - b[0]) % self.P, (a[1] - b[1]) % self.P)

    def f2_mul(self, a, b):
        P = self.P
        return ((a[0] * b[0] - a[1] * b[1]) % P, (a[0] * b[1] + a[1] * b[0]) % P)

    # ---- Fp12 = Fp2[w] / (w^6 - xi) -----------------------------------------------------------------------
    def add(self, a, b):
        return tuple(self.f2_add(x, y) for x, y in zip(a, b))

    def sub(self, a, b):
        return tuple(self.f2_sub(x, y) for x, y in zip(a, b))

    def neg(self, a):
        return self.sub(((0, 0),) * 6, a)

    def mul(self, a, b):
        acc = [(0, 0)] * 11
        for i, x in enumerate(a):
            if x == (0, 0):
                continue
            for j, y in enumerate(b):
                acc[i + j] = self.f2_add(acc[i + j], self.f2_mul(x, y))
        for k in range(10, 5, -1):  # w^k = xi w^(k-6)
            acc[k - 6] = self.f2_add(acc[k - 6], self.f2_mul(self.XI, acc[k]))
        return tuple(acc[:6])

    def pow(self, a, e):
        acc = self.ONE
        for bit in bin(e)[2:]:
            acc = self.mul(acc, acc)
            if bit == "1":
                acc = self.mul(acc, a)
        return acc

    def inv(self, a):
        """1 / a by Gaussian elimination of the 12 x 12 Fp matrix of multiplication by a."""
        P = self.P
        cols = []
        for i in range(6):
            for c in range(2):
                basis = [(0, 0)] * 6
                basis[i] = (1, 0) if c == 0 else (0, 1)
                cols.append([v for f2 in self.mul(a, tuple(basis)) for v in f2])
        rows = [[cols[j][i] for j in range(12)] + [1 if i == 0 else 0] for i in range(12)]
        for col in range(12):
            piv = next(r for r in range(col, 12) if rows[r][col])
            rows[col], rows[piv] = rows[piv], rows[col]
            iv = pow(rows[col][col], P - 2, P)
            rows[col] = [v * iv % P for v in rows[col]]
            for r in range(12):
                if r != col and rows[r][col]:
                    m = rows[r][col]
                    rows[r] = [(v - m * u) % P for v, u in zip(rows[r], rows[col])]
        sol = [rows[i][12] for i in range(12)]
        return tuple((sol[2 * i], sol[2 * i + 1]) for i in range(6))

    def frobenius(self, a, k=1):
        return self.pow(a, self.P ** k)

    def embed(self, x):
        """An Fp2 element as an Fp12 element."""
        return (x,) + ((0, 0),) * 5

    def w_pow(self, k):
        """w^k for k in -3 .. 3."""
        if k >= 0:
            e = [(0, 0)] * 6
            e[k] = (1, 0)
            return tuple(e)
        return self.pow(self.inv(self.w_pow(1)), -k)

    # ---- E(Fp12) ----------------------------------------------------------------------------------------
    def untwist(self, q):
        """psi(Q) for an affine G2 point Q = (x', y') over Fp2 (None = identity)."""
        if q is None:
            return None
        s = -1 if self.M_TYPE else 1
        return (self.mul(self.embed(q[0]), self.w_pow(2 * s)), self.mul(self.embed(q[1]), self.w_pow(3 * s)))

    def line(self, a, b, p):
        """The line through a and b (the tangent when a == b) of E(Fp12) at the Fp point p, and a + b."""
        if a == b:
            x2 = self.mul(a[0], a[0])
            lam = self.mul(self.add(self.add(x2, x2), x2), self.inv(self.add(a[1], a[1])))
        else:
            lam = self.mul(self.sub(b[1], a[1]), self.inv(self.sub(b[0], a[0])))
        x3 = self.sub(self.sub(self.mul(lam, lam), a[0]), b[0])
        y3 = self.sub(self.mul(lam, self.sub(a[0], x3)), a[1])
        px, py = self.embed((p[0], 0)), self.embed((p[1], 0))
        value = self.sub(self.sub(py, a[1]), self.mul(lam, self.sub(px, a[0])))
        return value, (x3, y3)

    def miller(self, p, q):
        """The Miller value whose final exponentiation is e(p, q); p affine over Fp, q affine over Fp2."""
        Q = self.untwist(q)
        loop = abs(self.X) if self.X < 0 else 6 * self.X + 2
        f, T = self.ONE, Q
        for bit in bin(loop)[3:]:
            v, T = self.line(T, T, p)
            f = self.mul(self.mul(f, f), v)
            if bit == "1":
                v, T = self.line(T, Q, p)
                f = self.mul(f, v)
        if self.X < 0:
            return self.inv(f)
        q1 = (self.frobenius(Q[0]), self.frobenius(Q[1]))
        q2 = (self.frobenius(Q[0], 2), self.neg(self.frobenius(Q[1], 2)))
        v, T = self.line(T, q1, p)
        f = self.mul(f, v)
        v, _ = self.line(T, q2, p)
        return self.mul(f, v)

    def final_exp(self, f):
        return self.pow(f, (self.P ** 12 - 1) // self.R)

    def pairing_product(self, pairs):
        """prod e(p_i, q_i) over (p, q) pairs of affine points (None = identity)."""
        f = self.ONE
        for p, q in pairs:
            if p is not None and q is not None:
                f = self.mul(f, self.miller(p, q))
        return self.final_exp(f)

    def pairing(self, p, q):
        return self.pairing_product([(p, q)])

    # ---- G1 (affine over Fp, None = identity) -------------------------------------------------------------
    def g1_add(self, a, b):
        P = self.P
        if a is None:
            return b
        if b is None:
            return a
        if a[0] == b[0]:
            if (a[1] + b[1]) % P == 0:
                return None
            lam = 3 * a[0] * a[0] * pow(2 * a[1], P - 2, P) % P
        else:
            lam = (b[1] - a[1]) * pow(b[0] - a[0], P - 2, P) % P
        x3 = (lam * lam - a[0] - b[0]) % P
        return (x3, (lam * (a[0] - x3) - a[1]) % P)

    def g1_mul(self, k, pt=None):
        pt = self.G1 if pt is None else pt
        k %= self.R
        acc = None
        for bit in bin(k)[2:] if k else "":
            acc = self.g1_add(acc, acc)
            if bit == "1":
                acc = self.g1_add(acc, pt)
        return acc

    def g2_mul(self, k, pt=None):
        return self.G2.scalar_mul(k % self.R, self.G2.G if pt is None else pt)

    # ---- ABI layouts ----------------------------------------------------------------------------------
    def _mont(self, v):
        return (v * self.MONT % self.P).to_bytes(self.W, "little")

    def g1_proj_struct(self, pt, z=1):
        """One sxt_*_g1_p2 struct of the affine point scaled by z; the identity is {0, 1, 0}."""
        x, y, z = (0, 1, 0) if pt is None else (pt[0] * z % self.P, pt[1] * z % self.P, z)
        return np.frombuffer(self._mont(x) + self._mont(y) + self._mont(z), np.uint8).copy()

    def g2_proj_struct(self, pt, z=(1, 0)):
        return self.G2.proj_struct(pt, z)

    def to_bytes(self, a):
        """The GT ABI bytes of an Fp12 element: c0.b0 .. c0.b2 = w^0, w^2, w^4, c1.b0 .. c1.b2 = w^1, w^3,
        w^5."""
        order = (0, 2, 4, 1, 3, 5)
        return b"".join(self._mont(a[i][0]) + self._mont(a[i][1]) for i in order)

    def from_bytes(self, raw):
        raw = bytes(raw)
        inv_r = pow(self.MONT, -1, self.P)
        vals = [int.from_bytes(raw[self.W * i:self.W * (i + 1)], "little") * inv_r % self.P
                for i in range(12)]
        out = [None] * 6
        for slot, i in enumerate((0, 2, 4, 1, 3, 5)):
            out[i] = (vals[2 * slot], vals[2 * slot + 1])
        return tuple(out)

    def to_limbs(self, a):
        """uint32 limbs of the GT ABI layout (b200_field_op fields 8 and 9)."""
        return np.frombuffer(self.to_bytes(a), np.uint32).copy()

    def from_limbs(self, limbs):
        return self.from_bytes(np.asarray(limbs, np.uint32).tobytes())


class _BlsG2:
    """tests/g2_reference's module functions behind the interface of bn254_g2_reference.Fp2Curve."""
    G = bls_g2.G
    R_ORDER = bls_g2.R_ORDER

    @staticmethod
    def scalar_mul(k, pt=bls_g2.G):
        return bls_g2.scalar_mul(k, pt)

    @staticmethod
    def proj_struct(pt, z=(1, 0)):
        return bls_g2.proj_struct(pt, z)

    @staticmethod
    def point_neg(pt):
        return bls_g2.point_neg(pt)


BLS = Tower(common.BLS_Q, common.BLS_R, 1, 4, (common.BLS_GX, common.BLS_GY), _BlsG2, -0xd201000000010000,
            True, 6)
BN = Tower(common.BN254_Q, common.BN254_R, 9, 3, (1, 2), bn_g2, 0x44e992b44a6909f1, False, 4)
TOWERS = {1: BLS, 2: BN}
G2_CURVE = {1: 4, 2: 5}  # the G2 curve id of each G1 curve id


def synth_log(i, first=0):
    """k_{first + i} (top bit cleared) of synthetic generator first + i."""
    return int.from_bytes(common.synth_scalars_k(1, first + i)[0].tobytes(), "little")
