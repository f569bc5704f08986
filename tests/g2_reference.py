"""TEST INFRASTRUCTURE — a pure-Python bls12-381 G2, the oracle of the G2 tests. Never imported by the
product.

Fp2 = Fp[u] / (u^2 + 1) as pairs (c0, c1) of Python integers, G2: y^2 = x^3 + 4 (1 + u) in Jacobian
coordinates, the library's ABI layouts (Montgomery limbs, R = 2^384, c0 first) and the 96-byte zcash
compressed encoding. Synthetic generators are G_i = (k_i mod 2^255) G with the k_i of
tests/common.synth_scalars_k, so an MSM over them has the closed form (sum_i s_i k_i mod r) G."""
import numpy as np

from tests import common

P = common.BLS_Q
R_ORDER = common.BLS_R
MONT = 1 << 384
B2 = (4, 4)
GX = (0x024aa2b2f08f0a91260805272dc51051c6e47ad4fa403b02b4510b647ae3d1770bac0326a805bbefd48056c8c121bdb8,
      0x13e02b6052719f607dacd3a088274f65596bd0d09920b61ab5da61bbdc7f5049334cf11213945d57e5ac7d055d042b7e)
GY = (0x0ce5d527727d6e118cc9cdc6da2e351aadfd9baa8cbdd3a76d429a695160d12c923ac9cc3baca289e193548608b82801,
      0x0606c4a02ea734cc32acd2b02bc28b99cb3e287e85a763af267492ab572e99ab3f370d275cec1da1aaa9075ff05f79be)
COMPRESSED_G = bytes.fromhex(
    "93e02b6052719f607dacd3a088274f65596bd0d09920b61ab5da61bbdc7f5049334cf11213945d57e5ac7d055d042b7e"
    "024aa2b2f08f0a91260805272dc51051c6e47ad4fa403b02b4510b647ae3d1770bac0326a805bbefd48056c8c121bdb8")
AFFINE_BYTES, PROJ_BYTES, COMMIT_BYTES = 200, 288, 96
FLAG = 192  # byte offset of the infinity flag of an affine generator
ZERO, ONE = (0, 0), (1, 0)


# ---- Fp2 --------------------------------------------------------------------------------------------
def add(a, b):
    return ((a[0] + b[0]) % P, (a[1] + b[1]) % P)


def sub(a, b):
    return ((a[0] - b[0]) % P, (a[1] - b[1]) % P)


def neg(a):
    return (-a[0] % P, -a[1] % P)


def mul(a, b):
    return ((a[0] * b[0] - a[1] * b[1]) % P, (a[0] * b[1] + a[1] * b[0]) % P)


def sqr(a):
    return mul(a, a)


def inv(a):
    """1 / a, 0 -> 0."""
    n = pow((a[0] * a[0] + a[1] * a[1]) % P, P - 2, P)
    return (a[0] * n % P, -a[1] * n % P)


def lex_largest(a):
    """The zcash rule: c1 > (p - 1) / 2, or c1 = 0 and c0 > (p - 1) / 2."""
    half = (P - 1) // 2
    return a[1] > half if a[1] else a[0] > half


# ---- G2: Jacobian (X, Y, Z), x = X / Z^2, y = Y / Z^3; None is the identity -----------------------------
G = (GX, GY)


def on_curve(pt):
    if pt is None:
        return True
    x, y = pt
    return sqr(y) == add(mul(sqr(x), x), B2)


def _jac(pt):
    return None if pt is None else (pt[0], pt[1], ONE)


def _affine(j):
    if j is None:
        return None
    zi = inv(j[2])
    zi2 = sqr(zi)
    return (mul(j[0], zi2), mul(j[1], mul(zi2, zi)))


def _jdbl(j):
    if j is None or j[1] == ZERO:
        return None
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


def _jadd(p, q):
    if p is None:
        return q
    if q is None:
        return p
    X1, Y1, Z1 = p
    X2, Y2, Z2 = q
    z1z1, z2z2 = sqr(Z1), sqr(Z2)
    U1, U2 = mul(X1, z2z2), mul(X2, z1z1)
    S1, S2 = mul(Y1, mul(Z2, z2z2)), mul(Y2, mul(Z1, z1z1))
    if U1 == U2:
        return _jdbl(p) if S1 == S2 else None
    H, r = sub(U2, U1), sub(S2, S1)
    HH = sqr(H)
    HHH = mul(H, HH)
    V = mul(U1, HH)
    X3 = sub(sub(sqr(r), HHH), add(V, V))
    Y3 = sub(mul(r, sub(V, X3)), mul(S1, HHH))
    return (X3, Y3, mul(mul(Z1, Z2), H))


def point_add(a, b):
    return _affine(_jadd(_jac(a), _jac(b)))


def point_neg(a):
    return None if a is None else (a[0], neg(a[1]))


def scalar_mul(k, pt=G):
    """k * pt (affine, None = identity) for any integer k."""
    if pt is None or k == 0:
        return None
    if k < 0:
        k, pt = -k, point_neg(pt)
    acc, base = None, _jac(pt)
    for bit in bin(k)[2:]:
        acc = _jdbl(acc)
        if bit == "1":
            acc = _jadd(acc, base)
    return _affine(acc)


# ---- encodings --------------------------------------------------------------------------------------
def compress(pt):
    """96-byte zcash compressed encoding: x.c1 then x.c0, big-endian; 0x80 compressed, 0x40 infinity,
    0x20 lexicographically largest y."""
    if pt is None:
        return bytes([0xC0]) + bytes(95)
    out = bytearray(pt[0][1].to_bytes(48, "big") + pt[0][0].to_bytes(48, "big"))
    out[0] |= 0x80 | (0x20 if lex_largest(pt[1]) else 0)
    return bytes(out)


def fp2_to_mont_bytes(a):
    """24 Montgomery limbs (c0 then c1) as 96 little-endian bytes."""
    return (a[0] * MONT % P).to_bytes(48, "little") + (a[1] * MONT % P).to_bytes(48, "little")


def fp2_from_mont_bytes(raw):
    inv_r = pow(MONT, -1, P)
    raw = bytes(raw)
    return (int.from_bytes(raw[:48], "little") * inv_r % P,
            int.from_bytes(raw[48:96], "little") * inv_r % P)


def affine_struct(pt):
    """One b200_bls12_381_g2 (200 bytes): identity = zero coordinates with the infinity flag."""
    out = np.zeros(AFFINE_BYTES, dtype=np.uint8)
    if pt is None:
        out[FLAG] = 1
    else:
        out[:192] = np.frombuffer(fp2_to_mont_bytes(pt[0]) + fp2_to_mont_bytes(pt[1]), np.uint8)
    return out


def proj_struct(pt, z=ONE):
    """One b200_bls12_381_g2_p2 (288 bytes) of the affine point scaled by z: (x z, y z, z); the
    identity is {0, 1, 0}."""
    if pt is None:
        coords = (ZERO, ONE, ZERO)
    else:
        coords = (mul(pt[0], z), mul(pt[1], z), z)
    return np.frombuffer(b"".join(fp2_to_mont_bytes(c) for c in coords), np.uint8).copy()


def from_affine_struct(row):
    row = np.asarray(row, dtype=np.uint8)
    if row[FLAG]:
        return None
    return (fp2_from_mont_bytes(row[:96]), fp2_from_mont_bytes(row[96:192]))


def from_proj_struct(row):
    """The affine point of one projective struct (None for Z = 0)."""
    row = np.asarray(row, dtype=np.uint8)
    X, Y, Z = (fp2_from_mont_bytes(row[96 * i:96 * (i + 1)]) for i in range(3))
    if Z == ZERO:
        return None
    zi = inv(Z)
    return (mul(X, zi), mul(Y, zi))


# ---- synthetic generators and the closed form --------------------------------------------------------
def synth_log(i):
    """k_i (top bit cleared) of synthetic generator i."""
    return int.from_bytes(common.synth_scalars_k(1, i)[0].tobytes(), "little")


def scalar_values(col):
    """The integers of one column (uint8 [n, nbytes], is_signed): little-endian, two's complement
    when signed."""
    data, signed = col
    data = np.asarray(data, dtype=np.uint8)
    bits = 8 * data.shape[1]
    vals = [int.from_bytes(r.tobytes(), "little") for r in data]
    if signed:
        vals = [v - (1 << bits) if v >> (bits - 1) else v for v in vals]
    return vals


def dot_logs(col, k):
    """sum_i s_i k_i mod r for one column and discrete logs k (uint64 [n, 4])."""
    ks = [int.from_bytes(r.tobytes(), "little") for r in np.asarray(k)[:np.asarray(col[0]).shape[0]]]
    return sum(s * kk for s, kk in zip(scalar_values(col), ks)) % R_ORDER


def closed_form(columns, k):
    """Compressed commitments of columns over generators with discrete logs k."""
    out = np.zeros((len(columns), COMMIT_BYTES), dtype=np.uint8)
    for j, col in enumerate(columns):
        out[j] = np.frombuffer(compress(scalar_mul(dot_logs(col, k))), np.uint8)
    return out


class Edits:
    """Row edits of synthetic affine G2 generators that keep their discrete logs k in step (the G2
    counterpart of tests/common.GeneratorEdits): duplicates share k, negations take r - k,
    identities k = 0."""

    def __init__(self, gens, first=0):
        self.gens = gens
        self.k = common.synth_scalars_k(gens.shape[0], first)

    def _logs(self, rows):
        return np.arange(self.k.shape[0])[rows]

    def duplicate(self, dst, src):
        self.gens[dst] = self.gens[src]
        self.k[dst] = self.k[src]

    def negate(self, rows):
        for i in self._logs(rows):
            pt = from_affine_struct(self.gens[i])
            self.gens[i] = affine_struct(point_neg(pt))
            v = (R_ORDER - int.from_bytes(self.k[i].tobytes(), "little")) % R_ORDER
            self.k[i] = np.frombuffer(v.to_bytes(32, "little"), dtype=np.uint64)

    def identity(self, rows):
        for i in self._logs(rows):
            self.gens[i] = affine_struct(None)
        self.k[rows] = 0
