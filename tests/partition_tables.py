"""Partition-table fixtures shared by the tests, the fixture generator
(tests/golden/make_partition_table_files.py) and tests/partition_table_timing.py: the cases, their
input generators, and the digest rule (SHA-256 of the table bytes after the u32 window-width header;
ristretto255 tables are canonicalised first, because the reference's radix-2^51 limbs are not
guaranteed canonical, so they compare by value)."""
import ctypes as C
import hashlib

import numpy as np

from tests import common

P25519 = (1 << 255) - 19
MASK51 = (1 << 51) - 1
COMPACT_BYTES = {0: 120, 1: 96, 2: 64, 3: 64}  # c21t / cg1t / cn1t / cgkt::compact_element
# name -> (n, window width, edited generators)
CASES = {"n37_w8": (37, 8, False), "n24_w6_edited": (24, 6, True), "n16_w16": (16, 16, False)}


def _r51(limbs):
    return sum(int(v) << (51 * i) for i, v in enumerate(limbs)) % P25519


def _limbs51(v):
    return [(v >> (51 * i)) & MASK51 for i in range(5)]


def canonicalise_ristretto_table(table):
    """uint8 table of c21t::compact_element {X, Y, T} (radix-2^51) -> the same values with every
    limb set canonical (each limb < 2^51, value < p)."""
    t = np.ascontiguousarray(table).view("<u8").reshape(-1, 5)
    out = np.array([_limbs51(_r51(row)) for row in t], dtype="<u8")
    return out.view(np.uint8).reshape(-1)


def sha256(table):
    return hashlib.sha256(np.ascontiguousarray(table).tobytes()).hexdigest()


def table_digest(curve, table):
    """The fixtures' digest of a table (no header): ristretto255 tables canonicalised first."""
    return sha256(canonicalise_ristretto_table(table) if curve == 0 else table)


def edit_generators(curve, gens):
    """Projective ABI generators with duplicates, G / -G pairs and identity rows, so that Z = 0 sums
    (Weierstrass) and identity sums occur in the middle of a w = 6 table. In place."""
    def negate(i):
        if curve == 0:  # (X : Y : Z : T) -> (-X : Y : Z : -T)
            for off in (0, 120):
                v = _r51(gens[i, off:off + 40].view("<u8"))
                gens[i, off:off + 40] = np.array(_limbs51((P25519 - v) % P25519), "<u8").view(np.uint8)
        else:  # (X : Y : Z) -> (X : -Y : Z)
            p, nb = common.curve_params(curve)[0], 8 * common.curve_params(curve)[2]
            y = int.from_bytes(gens[i, nb:2 * nb].tobytes(), "little")
            gens[i, nb:2 * nb] = np.frombuffer(((p - y) % p).to_bytes(nb, "little"), dtype=np.uint8)

    def identity(rows):
        if curve == 0:  # (0 : 1 : 1 : 0)
            gens[rows] = 0
            gens[rows, 40] = 1
            gens[rows, 80] = 1
        else:
            common.set_identity(curve, gens, rows)

    gens[1] = gens[0]            # group 0: a doubling at k = 3
    gens[3] = gens[2]
    negate(3)                    # G_3 = -G_2: zero sums at k = 12, 13, ...
    identity([4])
    gens[7] = gens[6]
    negate(7)                    # group 1: G_7 = -G_6 (k = 3 is the identity)
    gens[9] = gens[8]
    identity([10, 11])
    identity(list(range(12, 18)))  # group 2: every entry is the identity
    for i in (19, 20, 21):       # group 3: G_18, -G_18, G_18, -G_18, ..., a generator of group 0
        gens[i] = gens[18]
    negate(19)
    negate(21)
    gens[23] = gens[5]
    return gens


def case_generators(port, curve, name):
    n, _, edited = CASES[name]
    _, gens_p = common.generators_for(port, curve, n, seed=40 + n)
    gens_p = np.array(gens_p, copy=True)
    return edit_generators(curve, gens_p) if edited else gens_p


def emulated_table(emul, curve_id, generators_p, window_width, chunk_groups=0):
    """The partition table (no header) of projective ABI generators, through the product's kernel
    bodies run as serial host loops (tests/emul/ptable_emul.cpp), `chunk_groups` groups per chunk
    (0 = one chunk). emul: the tests/emul/harness module."""
    generators_p = np.ascontiguousarray(generators_p, dtype=np.uint8)
    n = generators_p.shape[0]
    out = np.zeros(-(-n // window_width) * (COMPACT_BYTES[curve_id] << window_width), dtype=np.uint8)
    emul.lib().emul_partition_table(C.c_uint(curve_id), C.c_void_p(out.ctypes.data),
                                    C.c_void_p(generators_p.ctypes.data), C.c_uint64(n),
                                    C.c_uint(window_width), C.c_uint64(chunk_groups))
    return out
