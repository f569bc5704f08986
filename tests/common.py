"""Shared input builders for the parity tests (seeded, deterministic), and the runner of the cases
that need a fresh interpreter."""
import importlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

# the reference's end-to-end golden (rust/tests/src/main.rs:21-49): three u32 columns over the
# built-in generators at offset 0 and their ristretto255 commitments
GOLDEN_COLUMNS = [[2000, 7500, 5000, 1500], [5000, 0, 400000, 10], [7000, 7500, 405000, 1510]]
GOLDEN_COMMITMENTS = [
    [4, 105, 58, 131, 59, 69, 150, 106, 120, 137, 32, 225, 175, 244, 82, 115,
     216, 180, 206, 150, 21, 250, 240, 98, 251, 192, 146, 244, 54, 169, 199, 97],
    [2, 254, 178, 195, 198, 238, 44, 156, 24, 29, 88, 196, 37, 63, 157, 50,
     236, 159, 61, 49, 153, 181, 79, 126, 55, 188, 67, 1, 228, 248, 72, 51],
    [30, 237, 163, 234, 252, 111, 45, 133, 235, 227, 21, 117, 229, 188, 88, 149,
     240, 109, 205, 90, 6, 130, 199, 152, 5, 221, 57, 231, 168, 9, 141, 122],
]
CMP = {0: 32, 1: 48, 2: 65, 3: 65}  # bytes of a commitment that are specified (no struct padding)


def golden_columns():
    return [(np.array(c, dtype="<u4").view(np.uint8).reshape(4, 4), 0) for c in GOLDEN_COLUMNS]


def random_columns(rng, n, shapes):
    """shapes: list of (length delta, element_nbytes, is_signed)."""
    cols = []
    for delta, nbytes, signed in shapes:
        m = max(0, n + delta)
        cols.append((rng.integers(0, 256, (m, nbytes), dtype=np.uint8), signed))
    return cols


def generators_for(port, curve, n, seed=3):
    """(commit-API generators, projective ABI generators) for a curve."""
    if curve == 0:
        g = port.ristretto_generators(n, seed)
        return g, g
    p2, af = port.test_points(curve, n, seed)
    return af, p2


def same(curve, a, b):
    k = CMP[curve]
    return np.array_equal(np.asarray(a)[:, :k], np.asarray(b)[:, :k])


# edge-case matrix modelled on mtxtst::exercise_multiexponentiation_fn
# (sxt/multiexp/test/multiexponentiation.cc:42-451)
def edge_case_columns():
    def u(vals, nbytes):
        return np.array([[(v >> (8 * k)) & 0xFF for k in range(nbytes)] for v in vals],
                        dtype=np.uint8).reshape(len(vals), nbytes)

    def s(vals, nbytes):
        return u([v & ((1 << (8 * nbytes)) - 1) for v in vals], nbytes)

    return [
        (u([0], 1), 0), (u([1], 1), 0), (u([2], 1), 0), (u([3], 1), 0),
        (u([0xFFFFFFFFFFFFFFFF], 8), 0),
        (u([1, 2, 3], 4), 0), (u([0, 0, 0], 4), 0),
        (u([1, 0, 255, 256, 65535], 3), 0),
        (s([-1], 1), 1), (s([-1, 1, -128, 127], 1), 1), (s([-(1 << 63), (1 << 63) - 1], 8), 1),
        (s([-(1 << 127), (1 << 127) - 1, -1, 0], 16), 1),
        (u([(1 << 256) - 1, (1 << 255), (1 << 252) + 27742317777372353535851937790883648493], 32), 0),
        (u([], 4), 0),
        (u([5] * 40, 2), 0),  # one heavily loaded bucket
    ]


# ---- closed-form check for MSMs over the reference's benchmark generators --------------------------
# G_i = (k_i mod 2^255) * G with k_i the 32 bytes of fast_random_number_generator{i+1, i+2}
# (sxt/curve_g1/random/element_p2.h:38-50), so sum_i s_i G_i = (sum_i s_i k_i mod r) * G at ANY size.
BN254_Q = 21888242871839275222246405745257275088696311157297823662689037894645226208583
BN254_R = 21888242871839275222246405745257275088548364400416034343698204186575808495617
BLS_Q = 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab
BLS_R = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001
BLS_GX = 3685416753713387016781088315183077757961620795782546409894578378688607592378376318836054947676345821548104185464507
BLS_GY = 1339506544944476473020471379941921221584933875938349620426543736416511423956333506472724655353366534992391756441569


def _grumpkin_gy():
    p = BN254_R
    # the smaller square root of -16 (curve_gk/constant/generator.h:47-50)
    n, q, s = -16 % p, p - 1, 0
    while q % 2 == 0:
        q //= 2
        s += 1
    z = 2
    while pow(z, (p - 1) // 2, p) != p - 1:
        z += 1
    m, c, t, r = s, pow(z, q, p), pow(n, q, p), pow(n, (q + 1) // 2, p)
    while t != 1:  # Tonelli-Shanks
        i, t2 = 0, t
        while t2 != 1:
            t2 = t2 * t2 % p
            i += 1
        b = pow(c, 1 << (m - i - 1), p)
        m, c = i, b * b % p
        t, r = t * c % p, r * b % p
    return min(r, p - r)


# curve id -> (field modulus, group order, limbs, Gx, Gy)
def curve_params(curve):
    if curve == 1:
        return BLS_Q, BLS_R, 6, BLS_GX, BLS_GY
    if curve == 2:
        return BN254_Q, BN254_R, 4, 1, 2
    if curve == 3:
        return BN254_R, BN254_Q, 4, 1, _grumpkin_gy()
    raise ValueError(curve)


def subgroup_generator_affine(curve):
    """The curve's generator as one affine ABI struct (Montgomery limbs), uint8 [1, stride]."""
    p, _, nl, gx, gy = curve_params(curve)
    R = 1 << (64 * nl)
    stride = 104 if curve == 1 else 72
    out = np.zeros((1, stride), dtype=np.uint8)
    out[0, :8 * nl] = np.frombuffer((gx * R % p).to_bytes(8 * nl, "little"), dtype=np.uint8)
    out[0, 8 * nl:16 * nl] = np.frombuffer((gy * R % p).to_bytes(8 * nl, "little"), dtype=np.uint8)
    return out


def synth_scalars_k(n, first=0):
    """k_i for i in [first, first+n): uint64 [n, 4] little-endian words, top bit cleared
    (basn::fast_random_number_generator, sxt/base/num/fast_random_number_generator.h:27-50)."""
    i = np.arange(first, first + n, dtype=np.uint64)
    sa, sb = i + np.uint64(1), i + np.uint64(2)
    out = np.zeros((n, 4), dtype=np.uint64)
    for j in range(4):
        t, s = sa.copy(), sb
        sa = s
        t ^= t << np.uint64(23)
        t ^= t >> np.uint64(17)
        t ^= s ^ (s >> np.uint64(26))
        sb = t
        out[:, j] = t + s
    out[:, 3] &= np.uint64(0x7FFFFFFFFFFFFFFF)
    return out


def _limbs16(a_u8):
    """uint8 [n, 2m] little-endian -> uint64 [n, m] of 16-bit limbs."""
    return np.ascontiguousarray(a_u8).view("<u2").astype(np.uint64)


def dot_mod(scalars_u8, k_u64, r):
    """sum_i scalar_i * k_i mod r, exact. scalars: uint8 [n, nbytes] (even nbytes), k: uint64 [n, 4]."""
    S = _limbs16(scalars_u8)
    K = _limbs16(k_u64.view(np.uint8).reshape(k_u64.shape[0], 32))
    total = 0
    step = 1 << 16  # 2^16 terms x (2^16)^2 < 2^48 per partial sum: exact in uint64
    for b in range(0, S.shape[0], step):
        M = S[b:b + step].T @ K[b:b + step]
        for a in range(M.shape[0]):
            for c in range(M.shape[1]):
                total += int(M[a, c]) << (16 * (a + c))
    return total % r


def closed_form_commitment(refcpu, curve, scalars_u8, first=0, k=None):
    """Reference commitment bytes of sum_i scalar_i * G_{first+i} through ONE reference scalar
    multiplication of the subgroup generator. k: discrete logs of generators that were edited after
    synthesis (uint64 [n, 4], see GeneratorEdits); default the synthetic ones."""
    _, r, _, _, _ = curve_params(curve)
    if k is None:
        k = synth_scalars_k(scalars_u8.shape[0], first)
    e = dot_mod(scalars_u8, k, r)
    sc = np.frombuffer(e.to_bytes(32, "little"), dtype=np.uint8).reshape(1, 32)
    return refcpu.commit(curve, [(sc, 0)], subgroup_generator_affine(curve))


# ---- degenerate Weierstrass generators (duplicates, negations, identities) --------------------------
# byte offset of the infinity flag of an affine commitment generator {X, Y, infinity}
AFFINE_FLAG = {1: 96, 2: 64, 3: 64}


def _field_bytes(curve):
    p, _, nl, _, _ = curve_params(curve)
    return p, 8 * nl


def negate_affine(curve, gens, rows):
    """In place: y -> p - y (Montgomery form) on the given rows of an affine generator array of any
    of the three Weierstrass layouts. Rows that are the identity are left alone."""
    p, nb = _field_bytes(curve)
    for i in np.arange(gens.shape[0])[rows]:
        if gens[i, AFFINE_FLAG[curve]]:
            continue
        y = int.from_bytes(gens[i, nb:2 * nb].tobytes(), "little")
        gens[i, nb:2 * nb] = np.frombuffer(((p - y) % p).to_bytes(nb, "little"), dtype=np.uint8)
    return gens


def set_identity(curve, gens, rows):
    """In place: the group identity on the given rows. Affine arrays (stride 104 / 72) get the
    infinity flag over zero coordinates (element_affine::identity()); projective arrays (stride 144 /
    96) get {0, R, 0}, i.e. Z = 0 (element_p2::identity())."""
    p, nb = _field_bytes(curve)
    gens[rows] = 0
    if gens.shape[1] == 3 * nb:
        gens[rows, nb:2 * nb] = np.frombuffer(((1 << (8 * nb)) % p).to_bytes(nb, "little"),
                                              dtype=np.uint8)
    else:
        gens[rows, AFFINE_FLAG[curve]] = 1
    return gens


def degenerate_buckets(port, curve):
    """Affine generators and 1-byte columns whose terms all land in ONE bucket per column (scalar 1:
    window 0, digit 1) holding nothing but copies of +-P, identities or, on bls12-381, the points
    (0, +-2) of order 3 (x = 0 without being the identity). The bucket contents do not depend on the
    order the entries are scattered in, only which pairs meet does.
    Returns (gens, cols, equal): equal lists (column index, m) for buckets of m copies of P."""
    p, nb = _field_bytes(curve)
    n = 176
    base = generators_for(port, curve, 2, seed=11)[0]
    gens = np.repeat(base[:1], n, axis=0)              # rows 0..63: P
    negate_affine(curve, gens, slice(65, 128, 2))      # rows 64..127: P, -P, P, -P, ...
    set_identity(curve, gens, slice(129, 160, 2))      # rows 128..159: P, O, P, O, ...
    gens[160:] = base[1]                               # rows 160..175: another point Q
    if curve == 1:                                     # rows 160..167: (0, 2) (0, 2) (0, -2) ...
        for i, sign in zip(range(160, 168), (1, 1, -1, 1, -1, -1, 1, 1)):
            gens[i, :nb] = 0
            gens[i, nb:2 * nb] = np.frombuffer((sign * 2 * (1 << (8 * nb)) % p).to_bytes(nb, "little"),
                                               dtype=np.uint8)

    def ones(rows):
        col = np.zeros((n, 1), dtype=np.uint8)
        col[rows] = 1
        return (col, 0)

    cols, equal = [], []
    for m in (2, 4, 8, 16, 32, 64, 3, 5, 7):  # doublings at every level; real entries next to pads
        equal.append((len(cols), m))
        cols.append(ones(slice(0, m)))
    cols += [ones(slice(64, 128)),   # cancellations at level 0, identity operands above
             ones(slice(64, 69)),    # P - P + P - P + P
             ones(slice(128, 160)),  # P next to identity generators
             ones(slice(127, 162)),  # -P, then P / O, then Q (x = 0 on bls12-381)
             ones(slice(160, 168)), ones(slice(160, 162)), ones(slice(161, 163))]
    rng = np.random.default_rng(curve)
    mix = rng.choice(np.array([1, 1, 1, 2, 0xFF], dtype=np.uint8), (n, 1))  # digits +-1 and 2, signed
    cols.append((mix, 1))
    return gens, cols, equal


RISTRETTO_R = (1 << 252) + 27742317777372353535851937790883648493


def cross_window_handle(port, curve, c, m=40):
    """Projective handle generators and fixed-MSM scalars (2 outputs x 32 bytes) for a fixed-base
    table of window c, whose windows share one bucket set: G_1 = 2^c G_0, G_2 = -2^c G_0 and
    G_4 = -2^c G_3, G_5 = 2^c G_3, with scalars d 2^c, d, d (and e 2^c, e, e), so that window 1 of
    G_0 (G_3) and window 0 of the other two land in the same bucket: a doubling and a cancellation
    inside table mode. Output 1 is random over all m rows."""
    r = RISTRETTO_R if curve == 0 else curve_params(curve)[1]
    _, gens_p = generators_for(port, curve, m, seed=21)
    gens_p = gens_p.copy()

    def s32(v):
        return np.frombuffer(v.to_bytes(32, "little"), dtype=np.uint8)

    two_c = 1 << c
    mult = np.concatenate([s32(two_c), s32(r - two_c)])[None]
    for i, plus, minus in ((0, 1, 2), (3, 5, 4)):
        gens_p[[plus, minus]] = port.fixed_msm(curve, gens_p[i:i + 1], 2, 1, mult, element_num_bytes=32)
    rng = np.random.default_rng(c + 10 * curve)
    sc = rng.integers(0, 256, (m, 2, 32), dtype=np.uint8)
    sc[:, 0] = 0
    for rows, digit in (((0, 1, 2), 5), ((3, 4, 5), 9)):
        sc[rows[0], 0] = s32(digit << c)
        sc[rows[1], 0] = sc[rows[2], 0] = s32(digit)
    return gens_p, sc.reshape(m, 64)


class GeneratorEdits:
    """Row edits of synthetic affine generators G_i = k_i G (synthetic_generators) that keep the
    discrete logs k'_i in step, so that closed_form_commitment(..., k=edits.k) stays exact."""

    def __init__(self, curve, gens, first=0):
        self.curve, self.gens = curve, gens
        self.r = curve_params(curve)[1]
        self.k = synth_scalars_k(gens.shape[0], first)

    def _set_logs(self, rows, fn):
        for i in np.arange(self.k.shape[0])[rows]:
            v = fn(int.from_bytes(self.k[i].tobytes(), "little"))
            self.k[i] = np.frombuffer(v.to_bytes(32, "little"), dtype=np.uint64)

    def duplicate(self, dst, src):
        """G_dst = G_src (k'_dst = k_src)."""
        self.gens[dst] = self.gens[src]
        self.k[dst] = self.k[src]

    def negate(self, rows):
        """G_i = -G_i (k'_i = r - k_i)."""
        negate_affine(self.curve, self.gens, rows)
        self._set_logs(rows, lambda v: (self.r - v) % self.r)

    def identity(self, rows):
        """G_i = O (k'_i = 0)."""
        set_identity(self.curve, self.gens, rows)
        self.k[rows] = 0


def mt19937_bytes(seed, n, nbytes=32, top_mask=0x0F):
    """The reference benchmark's scalar bytes: std::mt19937{seed} through
    uniform_int_distribution<uint8_t> (benchmark/multi_commitment/benchmark.m.cc:141-156;
    libstdc++ scales a 32-bit draw down by 2^24, i.e. the top byte), top byte masked."""
    rs = np.random.RandomState(seed)
    out = (rs.randint(0, 2 ** 32, n * nbytes, dtype=np.uint64) >> 24).astype(np.uint8).reshape(n, nbytes)
    out[:, nbytes - 1] &= top_mask
    return out


# ---- cases that need a fresh interpreter -------------------------------------------------------------
# The library reads part of its configuration once per process: sxt_init's arguments,
# BLITZAR_B200_DEVICES / _SHARED_DEVICES, BLITZAR_B200_MIN_SHARD_TERMS and BLITZAR_LOG_LEVEL. A child
# gets none of the variables the library reads from the test process, only the ones the case sets.
_LIBRARY_ENV = ("BLITZAR_LOG_LEVEL", "BLITZAR_PARTITION_WINDOW_WIDTH", "BLITZAR_BACKEND")
_FRESH_DONE = "fresh process: every body returned"
_FRESH_CHILD = ("import sys; sys.path.insert(0, sys.argv[1]); from tests import common; "
                "common._fresh_child(sys.argv[2])")


def run_fresh(*bodies, init={"num_precomputed_generators": 64}, env=None):
    """Runs body(bb, port, *args) for each entry, in order, in one new interpreter and returns its
    CompletedProcess. An entry is a module-level function or a tuple (function, *args) with
    JSON-serialisable args; the child imports the function by module and name. init: the child's
    sxt_init arguments (None: the child leaves the library alone). env: variables set on top of this
    process's environment without the library's variables."""
    calls = []
    for entry in bodies:
        fn, *args = entry if isinstance(entry, tuple) else (entry,)
        calls.append((fn.__module__, fn.__qualname__, args))
    child_env = {k: v for k, v in os.environ.items()
                 if not (k.startswith("BLITZAR_B200_") or k in _LIBRARY_ENV)}
    child_env.update(env or {})
    r = subprocess.run([sys.executable, "-c", _FRESH_CHILD, ROOT,
                        json.dumps(dict(init=init, calls=calls))],
                       env=child_env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and _FRESH_DONE in r.stdout, r.stdout + r.stderr[-8000:]
    return r


def _fresh_child(spec):
    import blitzar_b200 as bb
    from oracle import port
    spec = json.loads(spec)
    calls = [(getattr(importlib.import_module(module), name), args)
             for module, name, args in spec["calls"]]
    port.build()
    if spec["init"] is not None:
        assert bb.sxt_init(**spec["init"]) == 0
    for fn, args in calls:
        fn(bb, port, *args)
    print(_FRESH_DONE)
