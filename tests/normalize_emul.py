"""Ristretto255 generators in scaled representations, and the decoding of the device generators that
the normalising ingestion writes."""
import numpy as np

P = 2 ** 255 - 19
MASK51 = (1 << 51) - 1


def _decode(row):
    """160-byte sxt_ristretto255 {X[5], Y[5], Z[5], T[5]} (radix 2^51) -> [X, Y, Z, T] mod p."""
    limbs = np.frombuffer(row.tobytes(), dtype="<u8")
    return [sum(int(limbs[5 * c + i]) << (51 * i) for i in range(5)) % P for c in range(4)]


def _encode(coords):
    out = np.zeros(20, dtype="<u8")
    for c, v in enumerate(coords):
        v %= P
        for i in range(5):
            out[5 * c + i] = (v >> (51 * i)) & MASK51
    return out.view(np.uint8)


def scaled_generators(gens, seed, identity=(), negated=(), duplicated=(), zero_z=(), scale=True):
    """Copies of the ABI generators, each with X, Y, Z, T multiplied by its own random lambda != 0 (the
    same points in other projective representations; scale=False: lambda = 1). Rows in `identity`
    become the identity, rows in `negated` the negation of the row before them, a row r in
    `duplicated` a (differently scaled) copy of row r - 1; rows in `zero_z` get Z = 0 (not a point)."""
    rng = np.random.default_rng(seed)
    out = np.array(gens, dtype=np.uint8, copy=True)
    pts = [_decode(out[i]) for i in range(out.shape[0])]
    for i in range(len(pts)):
        if i in identity:
            pts[i] = [0, 1, 1, 0]
        elif i in negated and i > 0:
            x, y, z, t = pts[i - 1]
            pts[i] = [-x % P, y, z, -t % P]
        elif i in duplicated and i > 0:
            pts[i] = list(pts[i - 1])
    for i, pt in enumerate(pts):
        lam = int.from_bytes(rng.bytes(32), "little") % (P - 1) + 1 if scale else 1
        pt = [v * lam % P for v in pt]
        if i in zero_z:
            pt[2] = 0
        out[i] = _encode(pt)
    return out


def decode_device_gen(row):
    """128-byte device generator (Y+X, Y-X, 2Z, 2dT as 8 x u32 limbs each) -> its four values."""
    limbs = np.frombuffer(row.tobytes(), dtype="<u4").astype(object)
    return [sum(int(limbs[8 * c + i]) << (32 * i) for i in range(8)) for c in range(4)]

