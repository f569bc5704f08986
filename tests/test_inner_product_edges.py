"""The inner-product argument at its edges, single and batched, on the CPU emulation of the kernel
bodies and on the GPU.

A  Prove parity, byte for byte against the C oracle port and the reference's CPU prover: n at and
   around powers of two, generator offsets inside, across and far beyond the precomputed table, and
   scalars that are unreduced (l, l + 1, 2^255, 2^256 - 1, random values in [l, 2^256) or near
   2^256), all zero, l - 1, or zero except in the padded upper half. n = 1 returns the caller's
   a[0] unchanged.
B  Large n on the GPU: n = 2^16 + 1 against the reference's prover, n = 2^20 proved and verified.
C  Inputs equal to an honest proof's as group elements or scalars are accepted: ap + l, product + l,
   b_i + l, a_commit with a scaled Z, with limbs of coordinate + 2p, or plus a 4-torsion point.
D  Each single tampering of an honest proof is rejected.
E  Every rejection branch of ristretto255 decoding (RFC 9496 section 4.3.1: non-canonical s,
   negative s, non-square, negative t, y = 0), hit alone at L_0, L_last, R_0 and R_last of a proof
   whose challenges are taken over those bytes and whose a_commit makes it verify with the decoded
   point, is rejected and flagged alone in a batch; a decoder without that one check accepts it.
F  A proof that is honest except that one L_j or R_j is written as p - s, s + p or s + 2^255 (each
   challenge over the emitted bytes) is accepted by the port's verifier without the canonical and
   sign checks, and rejected here.
G  The batched entry points on mixed batches of n, offsets and honest, equivalent, tampered and
   mis-encoded proofs: equal to the single calls, exact result flags.

The reference (sxt/proof/inner_product) defines A-D; it reduces every caller scalar mod l except the
n = 1 ap, which it returns as given. It does not check the status of its ristretto decoder, so for
E and F the rule is RFC 9496 section 4.3.1, which the device decoder (Ed25519::decode) and the
port's (ristretto_decode) implement. A model of the RFC over Python integers picks the encodings."""
import numpy as np
import pytest

from tests.emul import ipa_batch
from tests.test_field_arithmetic import P25519 as P, SQRT_M1, sqrt_ratio_m1
from tests.test_inner_product_batch import _prove_singly, _same_proofs, check_mixed_batch

L = 2**252 + 27742317777372353535851937790883648493
D = -121665 * pow(121666, -1, P) % P
INVSQRT_A_MINUS_D = sqrt_ratio_m1(1, -1 - D)[0]
NUM_BUILTIN = 64  # the precomputed generators of the `bb` fixture, and of the emulated cases
EMUL_MAX_N = 129  # larger shapes run on the GPU only
FAR_OFFSET = 2**33 + 5
SPECIAL = (L, L + 1, 2**255, 2**256 - 1)


# ---- engines ----------------------------------------------------------------------------------------
@pytest.fixture
def engine(request):
    if request.param == "gpu":
        yield request.getfixturevalue("bb")
        return
    emul = request.getfixturevalue("emul")
    with emul.options(num_builtin=NUM_BUILTIN):
        yield ipa_batch.Engine(NUM_BUILTIN)


def engines(max_n=EMUL_MAX_N, n=1):
    out = [pytest.param("gpu", id="gpu", marks=pytest.mark.gpu)]
    return ([pytest.param("emul", id="emul")] if n <= max_n else []) + out


# ---- scalars, points and encodings over Python integers ---------------------------------------------
def enc(values):
    raw = b"".join(int(v).to_bytes(32, "little") for v in values)
    return np.frombuffer(raw, np.uint8).reshape(-1, 32).copy()


def dec(arr):
    raw = np.ascontiguousarray(arr, np.uint8).tobytes()
    return [int.from_bytes(raw[i:i + 32], "little") for i in range(0, len(raw), 32)]


def scalar_class(name, rng, n):
    """(a, b) as Python integers of one scalar class."""
    rand = lambda lo, hi: [int(lo + int.from_bytes(rng.bytes(32), "little") % (hi - lo))
                           for _ in range(n)]
    if name == "canonical":
        return rand(0, L), rand(0, L)
    if name == "unreduced":  # the specials first, then random values in [l, 2^256), in both vectors
        a, b = rand(L, 2**256), rand(L, 2**256)
        for i, v in enumerate(SPECIAL[:n]):
            a[i] = v
            b[n - 1 - i] = v
        return a, b
    if name == "near 2^256":  # every product of round 0 near 2^256, its sums past 2^256
        return rand(2**256 - 2**250, 2**256), rand(2**256 - 2**250, 2**256)
    if name == "a zero":
        return [0] * n, rand(0, L)
    if name == "b zero":
        return rand(0, L), [0] * n
    if name == "l - 1":
        return [L - 1] * n, [L - 1] * n
    if name == "last a only":  # index n - 1 lies in the zero-padded upper half of round 0
        return [0] * (n - 1) + rand(1, L)[:1], rand(0, L)
    raise ValueError(name)


CLASSES = ("canonical", "unreduced", "near 2^256", "a zero", "b zero", "l - 1", "last a only")


def radix51(v):
    return [(v >> (51 * i)) & (2**51 - 1) for i in range(5)]


TWO_P_LIMBS = [2**52 - 38] + [2**52 - 2] * 4  # 2p with every limb near 2^52


def point_from_abi(raw):
    """sxt_ristretto255 (X, Y, Z, T, each five radix-2^51 limbs, include/blitzar_b200.h) -> ints"""
    w = np.frombuffer(np.ascontiguousarray(raw, np.uint8).tobytes(), "<u8")
    return tuple(sum(int(w[5 * c + i]) << (51 * i) for i in range(5)) % P for c in range(4))


def point_to_abi(pt, plus_two_p=False):
    limbs = []
    for c in pt:
        lc = radix51(c % P)
        limbs += [x + y for x, y in zip(lc, TWO_P_LIMBS)] if plus_two_p else lc
    assert max(limbs) < 2**54
    return np.frombuffer(np.array(limbs, "<u8").tobytes(), np.uint8).copy()


def point_add(p1, p2):
    """extended twisted Edwards addition (a = -1)"""
    x1, y1, z1, t1 = p1
    x2, y2, z2, t2 = p2
    a, b = (y1 - x1) * (y2 - x2) % P, (y1 + x1) * (y2 + x2) % P
    c, d = 2 * D * t1 * t2 % P, 2 * z1 * z2 % P
    e, f, g, h = b - a, d - c, d + c, b + a
    return e * f % P, g * h % P, f * g % P, e * h % P


def point_neg(pt):
    return (-pt[0] % P, pt[1], pt[2], -pt[3] % P)


def point_mul(k, pt):
    """k pt for an integer k >= 0 (the addition above is complete, so it doubles too)"""
    acc = (0, 1, 1, 0)
    for bit in bin(k)[2:]:
        acc = point_add(acc, acc)
        if bit == "1":
            acc = point_add(acc, pt)
    return acc


TORSION4 = [(0, P - 1, 1, 0), (SQRT_M1, 0, 1, 0), (P - SQRT_M1, 0, 1, 0)]  # E[4] minus identity


def is_negative(v):
    return (v % P) & 1


def ristretto_encode(pt):
    """RFC 9496 section 4.3.2 -> the canonical s"""
    x0, y0, z0, t0 = pt
    u1 = (z0 + y0) * (z0 - y0) % P
    u2 = x0 * y0 % P
    invsqrt = sqrt_ratio_m1(1, u1 * u2 * u2)[0]
    den1, den2 = invsqrt * u1 % P, invsqrt * u2 % P
    z_inv = den1 * den2 * t0 % P
    rotate = is_negative(t0 * z_inv)
    x, y = (y0 * SQRT_M1 % P, x0 * SQRT_M1 % P) if rotate else (x0, y0)
    den_inv = den1 * INVSQRT_A_MINUS_D % P if rotate else den2
    if is_negative(x * z_inv):
        y = P - y
    s = den_inv * (z0 - y) % P
    return P - s if is_negative(s) else s


def ristretto_decode(raw):
    """RFC 9496 section 4.3.1 on a 256-bit integer -> (the point the formulas give, the rejection
    branches hit). The field element is read as the device reads it, from the low 255 bits."""
    hits = []
    if raw >= P:
        hits.append("non-canonical")
    if raw & 1:
        hits.append("negative s")
    s = (raw % 2**255) % P
    ss = s * s % P
    u1, u2 = (1 - ss) % P, (1 + ss) % P
    u2sq = u2 * u2 % P
    v = (-D * u1 * u1 - u2sq) % P
    invsqrt, was_square, _ = sqrt_ratio_m1(1, v * u2sq)
    den_x = invsqrt * u2 % P
    den_y = invsqrt * den_x * v % P
    x = 2 * s * den_x % P
    x = P - x if is_negative(x) else x
    y = u1 * den_y % P
    t = x * y % P
    if not was_square:
        hits.append("non-square")
    if is_negative(t):
        hits.append("negative t")
    if y == 0:
        hits.append("y = 0")
    return (x, y, 1, t), hits


def branch_encodings():
    """branch -> 32-byte encodings that hit that rejection branch of the decoder alone"""
    rng = np.random.default_rng(2024)
    out = {"non-canonical": [], "non-square": [], "negative t": [], "y = 0": [P - 1]}
    for raw in range(P + 1, 2**255, 2):  # even, >= p: s = raw - p is odd and small
        if ristretto_decode(raw)[1] == ["non-canonical"]:
            out["non-canonical"].append(raw)
    while len(out["non-square"]) < 2 or len(out["negative t"]) < 2:
        raw = (int.from_bytes(rng.bytes(32), "little") % P) & ~1
        hits = ristretto_decode(raw)[1]
        if len(hits) == 1 and hits[0] in out and len(out[hits[0]]) < 2:
            out[hits[0]].append(raw)
    return out


def honest_case(port, seed, n, offset):
    """An honest proof with every verifier input: dict of t0, a, b, product, a_commit, l, r, ap."""
    rng = np.random.default_rng(seed)
    av, bv = scalar_class("canonical", rng, n)
    a, b = enc(av), enc(bv)
    t0 = port.transcript_new(b"edges %d" % seed)
    t = t0.copy()
    lv, rv, ap = port.prove_inner_product(t, a, b, offset)
    gens = port.ristretto_generators(n, offset)
    a_commit = port.fixed_msm(0, gens, 1, n, a, element_num_bytes=32)[0]
    product = enc([sum(x * y for x, y in zip(av, bv)) % L])[0]
    return dict(t0=t0, t1=t, n=n, offset=offset, a=a, b=b, av=av, bv=bv, product=product,
                a_commit=a_commit, l=lv, r=rv, ap=ap)


def verify_args(case, **changed):
    c = dict(case, **changed)
    return (c["t0"].copy(), c["b"], c["product"], c["a_commit"], c["l"], c["r"], c["ap"],
            c["offset"])


def call(verify, args, **kw):
    """verify(*args) on a copy of the transcript in args"""
    return verify(args[0].copy(), *args[1:], **kw)


def verify_all(engine, cases):
    """single and batched results of `engine` on a list of verify_args tuples; the batch's
    transcripts advance as the single calls advance them"""
    singles, t_single = [], []
    for args in cases:
        t = args[0].copy()
        singles.append(engine.verify_inner_product(t, *args[1:]))
        t_single.append(t)
    tb = np.stack([args[0] for args in cases])
    res = engine.verify_inner_products(tb, [x[1] for x in cases], np.stack([x[2] for x in cases]),
                                       np.stack([x[3] for x in cases]), [x[4] for x in cases],
                                       [x[5] for x in cases], np.stack([x[6] for x in cases]),
                                       [x[7] for x in cases])
    assert res.tolist() == singles
    assert all(np.array_equal(x, y) for x, y in zip(tb, t_single))
    return singles


# ---- the model itself ---------------------------------------------------------------------------------
def test_ristretto_model_matches_the_port(port):
    """The model decodes the port's L and R to points it re-encodes to the same bytes, and every
    chosen encoding hits its branch alone."""
    case = honest_case(port, 1, 37, 5)
    for raw in dec(case["l"]) + dec(case["r"]):
        pt, hits = ristretto_decode(raw)
        assert hits == [] and ristretto_encode(pt) == raw
        assert ristretto_decode(P - raw)[1] == ["negative s"]
        assert ristretto_decode(raw + 2**255)[1] == ["non-canonical"]
    assert ristretto_encode(point_from_abi(case["a_commit"])) == dec(
        port.commit(0, [(case["a"], 0)], None, 5))[0]
    for branch, raws in branch_encodings().items():
        assert raws, branch
        assert all(ristretto_decode(raw)[1] == [branch] for raw in raws), branch
    # p + 1 would hit y = 0 too; the non-canonical values kept are exactly those that decode alone
    assert ristretto_decode(P + 1)[1] == ["non-canonical", "y = 0"]


# ---- A: prove parity ----------------------------------------------------------------------------------
A_SIZES = (2, 3, 4, 63, 64, 65, 127, 128, 129, 255, 256, 257, 1023, 1024, 1025)


def offsets_for(n):
    np_ = 1 << (n - 1).bit_length()
    straddle = NUM_BUILTIN - np_ // 2 if np_ < NUM_BUILTIN else 1  # [offset, offset + np] holds 64
    return (0, 1, straddle, FAR_OFFSET)


def a_cases(n):
    """(class, offset) pairs of one n: every class, at offsets taken in turn"""
    offs = offsets_for(n)
    return [(cls, offs[(i + n) % len(offs)]) for i, cls in enumerate(CLASSES)]


def prove_case(seed, n, cls):
    rng = np.random.default_rng(seed)
    av, bv = scalar_class(cls, rng, n)
    t0 = np.zeros(203, np.uint8)
    t0[:200] = rng.integers(0, 256, 200, dtype=np.uint8)
    return t0, enc(av), enc(bv)


def check_prove(engine, port, refcpu, t0, a, b, offset):
    t_port = t0.copy()
    want = port.prove_inner_product(t_port, a, b, offset)
    t_ref = t0.copy()
    ref = refcpu.prove_inner_product(t_ref, a, b, offset)
    assert all(np.array_equal(x, y) for x, y in zip(want, ref)) and np.array_equal(t_port, t_ref)
    t = t0.copy()
    got = engine.prove_inner_product(t, a, b, offset)
    assert all(np.array_equal(x, y) for x, y in zip(got, want)) and np.array_equal(t, t_port)
    return got


@pytest.mark.parametrize("engine,n", [pytest.param(e.values[0], n, id=f"{e.id}-n{n}", marks=e.marks)
                                      for n in A_SIZES for e in engines(n=n)], indirect=["engine"])
def test_prove_parity(engine, n, port, refcpu):
    """L, R, ap and the advanced transcript equal the port's and the reference's for every scalar
    class; the classes with unreduced scalars give the proof of their residues."""
    for cls, offset in a_cases(n):
        t0, a, b = prove_case(n * 100 + CLASSES.index(cls), n, cls)
        got = check_prove(engine, port, refcpu, t0, a, b, offset)
        if cls == "unreduced":  # the reference reduces every caller scalar mod l first
            t = t0.copy()
            reduced = port.prove_inner_product(t, enc([v % L for v in dec(a)]),
                                               enc([v % L for v in dec(b)]), offset)
            assert all(np.array_equal(x, y) for x, y in zip(got, reduced)), offset


@pytest.mark.parametrize("engine", engines(), indirect=True)
def test_n1_returns_the_callers_a(engine, port, refcpu):
    """n = 1: no rounds, and ap is a[0] as given, reduced or not (proof_computation.cc)."""
    rng = np.random.default_rng(1)
    for a0 in SPECIAL + (L - 1, 0, L + int(rng.integers(1, 2**62))):
        t0 = port.transcript_new(b"n1")
        a, b = enc([a0]), enc([5])
        lv, rv, ap = check_prove(engine, port, refcpu, t0, a, b, 7)
        assert len(lv) == 0 and len(rv) == 0 and np.array_equal(ap, a[0])


# ---- B: large n on the GPU ------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_prove_parity_2_16_plus_1(bb, refcpu):
    n = 2**16 + 1
    t0, a, b = prove_case(16, n, "unreduced")
    t_ref = t0.copy()
    want = refcpu.prove_inner_product(t_ref, a, b, 3)
    t = t0.copy()
    got = bb.prove_inner_product(t, a, b, 3)
    assert all(np.array_equal(x, y) for x, y in zip(got, want)) and np.array_equal(t, t_ref)


@pytest.mark.gpu
def test_gpu_prove_and_verify_2_20(bb):
    n = 2**20
    t0, a, b = prove_case(20, n, "canonical")
    av, bv = dec(a), dec(b)
    t = t0.copy()
    lv, rv, ap = bb.prove_inner_product(t, a, b, 0)
    assert len(lv) == 20
    product = enc([sum(x * y for x, y in zip(av, bv)) % L])[0]
    h = bb.MultiexpHandle(0, bb.get_generators(n, 0))
    a_commit = h.fixed_multiexponentiation(32, 1, n, a)[0]
    h.free()
    tv = t0.copy()
    assert bb.verify_inner_product(tv, b, product, a_commit, lv, rv, ap, 0) == 1
    assert np.array_equal(tv, t)
    bad = product.copy()
    bad[0] ^= 1
    assert bb.verify_inner_product(t0.copy(), b, bad, a_commit, lv, rv, ap, 0) == 0


# ---- C: equivalent inputs are accepted -------------------------------------------------------------------
C_SHAPES = ((1, 9), (5, 0), (16, 60))  # (n, offset); 60: [60, 76] straddles the precomputed table


def equivalents(case):
    """(name, verify_args) of inputs equal to the honest ones as scalars mod l or ristretto points"""
    out = [("honest", verify_args(case))]
    plus_l = lambda v: enc([dec(v)[0] + L])[0]
    out.append(("ap + l", verify_args(case, ap=plus_l(case["ap"]))))
    out.append(("product + l", verify_args(case, product=plus_l(case["product"]))))
    bv = dec(case["b"])
    for i in sorted({0, case["n"] - 1}):
        out.append((f"b_{i} + l", verify_args(case, b=enc(bv[:i] + [bv[i] + L] + bv[i + 1:]))))
    out.append(("every b_i + l", verify_args(case, b=enc([v + L for v in bv]))))
    pt = point_from_abi(case["a_commit"])
    lam = 0xC0FFEE1234567 ** 5 % P
    out.append(("a_commit scaled", verify_args(case, a_commit=point_to_abi(
        tuple(c * lam % P for c in pt)))))
    out.append(("a_commit limbs + 2p", verify_args(case, a_commit=point_to_abi(pt, True))))
    for j, tor in enumerate(TORSION4):
        out.append((f"a_commit + T{j}", verify_args(case, a_commit=point_to_abi(point_add(pt, tor)))))
    return out


@pytest.mark.parametrize("engine", engines(), indirect=True)
@pytest.mark.parametrize("n,offset", C_SHAPES)
def test_equivalent_inputs_are_accepted(engine, n, offset, port, refcpu):
    case = honest_case(port, 30 + n, n, offset)
    named = equivalents(case)
    for name, args in named:
        assert call(refcpu.verify_inner_product, args) == 1, name
        assert call(port.verify_inner_product, args) == 1, name
    assert verify_all(engine, [args for _, args in named]) == [1] * len(named)


# ---- D: single tamperings are rejected --------------------------------------------------------------------
def tamperings(case, generator0):
    n, k = case["n"], len(case["l"])
    bump = lambda v, d: enc([(dec(v)[0] + d) % 2**256])[0]
    out = []
    for d in (1, -1):
        out.append((f"product {d:+}", verify_args(case, product=bump(case["product"], d))))
        out.append((f"ap {d:+}", verify_args(case, ap=bump(case["ap"], d))))
        if case["offset"] + d >= 0:
            out.append((f"offset {d:+}", verify_args(case, offset=case["offset"] + d)))
    for i in range(n):
        b = case["b"].copy()
        b[i] = bump(b[i], 1)
        out.append((f"b_{i} + 1", verify_args(case, b=b)))
    pt = point_from_abi(case["a_commit"])
    out.append(("a_commit + G", verify_args(case, a_commit=point_to_abi(point_add(pt, generator0)))))
    for side in ("l", "r"):
        for j in range(k):  # L_j + G_0: a valid encoding of another point
            v = case[side].copy()
            v[j] = enc([ristretto_encode(point_add(ristretto_decode(dec(v[j])[0])[0],
                                                   generator0))])[0]
            out.append((f"{side}_{j} + G", verify_args(case, **{side: v})))
    out.append(("L and R swapped", verify_args(case, l=case["r"], r=case["l"])))
    for j in range(k - 1):
        v = case["l"].copy()
        v[[j, j + 1]] = v[[j + 1, j]]
        out.append((f"L_{j} <-> L_{j + 1}", verify_args(case, l=v)))
    t = case["t0"].copy()
    t[17] ^= 0x40
    out.append(("transcript byte", verify_args(case, t0=t)))
    return out


@pytest.mark.parametrize("engine", engines(), indirect=True)
@pytest.mark.parametrize("n,offset", ((2, 0), (6, 61), (9, 3)))
def test_single_tamperings_are_rejected(engine, n, offset, port, refcpu):
    case = honest_case(port, 40 + n, n, offset)
    generator0 = point_from_abi(port.ristretto_generators(1, 0)[0])
    named = tamperings(case, generator0)
    for name, args in named:
        assert call(refcpu.verify_inner_product, args) == 0, name
        assert call(port.verify_inner_product, args) == 0, name
    # the honest proof between the tampered ones: flags stay exact
    cases = [verify_args(case)] + [args for _, args in named] + [verify_args(case)]
    assert verify_all(engine, cases) == [1] + [0] * len(named) + [1]


# ---- E and F: encodings -------------------------------------------------------------------------------------
def positions(k):
    """(side, round) of L_0, L_last, R_0, R_last"""
    return [("l", 0), ("l", k - 1), ("r", 0), ("r", k - 1)]


def encoded_case(port, case, side, j, mode, replacement=None):
    """`case`'s proof with L_j or R_j emitted in encoding `mode`, challenges over the emitted bytes,
    and a_commit moved so that the proof verifies if the decoder reads those bytes as the point the
    RFC formulas give: A' = A + e (P' - P), with P the honest point, P' the decoded one and e the
    verifier's exponent of that L_j (-x_j^2) or R_j (-x_j^-2)"""
    k = len(case["l"])
    modes = np.zeros(2 * k, np.uint8)
    modes[j if side == "l" else k + j] = mode
    rep = np.zeros((2 * k, 32), np.uint8)
    if replacement is not None:
        rep[j if side == "l" else k + j] = enc([replacement])[0]
    t = case["t0"].copy()
    lv, rv, ap, x = port.prove_inner_product_encoded(t, case["a"], case["b"], case["offset"],
                                                     modes[:k], modes[k:], rep)
    forged = dict(case, l=lv, r=rv, ap=ap)
    xj = dec(x[j])[0]
    e = -pow(xj, 2 if side == "l" else -2, L) % L
    honest = ristretto_decode(dec(case[side][j])[0])[0]  # round j's point precedes its challenge
    decoded = ristretto_decode(dec(forged[side][j])[0])[0]
    shift = point_mul(e, point_add(decoded, point_neg(honest)))
    forged["a_commit"] = point_to_abi(point_add(point_from_abi(case["a_commit"]), shift))
    return forged


# branch -> (encoding mode, the check a lax decoder skips to accept the proof). Every encoding reads
# as a point on the curve except the non-square ones, whose formulas give no curve point: those
# proofs fail the verification equation whatever the decoder does, and have no lax control.
E_BRANCHES = {"non-canonical": ("ENC_REPLACE", "LAX_CANONICAL"),
              "bit 255": ("ENC_TOP_BIT", "LAX_CANONICAL"),
              "negative s": ("ENC_NEGATED", "LAX_SIGN"),
              "negative t": ("ENC_REPLACE", "LAX_T"),
              "y = 0": ("ENC_REPLACE", "LAX_Y"),
              "non-square": ("ENC_REPLACE", None)}


def e_cases(port, case):
    """(branch, side, j, verify_args, lax) of every branch at every position"""
    raws = branch_encodings()
    out = []
    for side, j in positions(len(case["l"])):
        for branch, (mode, lax) in E_BRANCHES.items():
            for raw in (raws[branch] if mode == "ENC_REPLACE" else [None]):
                forged = encoded_case(port, case, side, j, getattr(port, mode), raw)
                hits = ristretto_decode(dec(forged[side][j])[0])[1]
                assert hits == ["non-canonical" if branch == "bit 255" else branch], hits
                out.append((branch, side, j, verify_args(forged), lax and getattr(port, lax)))
    return out


@pytest.mark.parametrize("engine", engines(), indirect=True)
@pytest.mark.parametrize("n,offset", ((2, 0), (16, 60)))
def test_decoder_rejects_each_branch(engine, n, offset, port):
    """Each placement verifies under a decoder without exactly the check its encoding fails, so
    that check alone rejects it."""
    case = honest_case(port, 50 + n, n, offset)
    named = e_cases(port, case)
    for branch, side, j, args, lax in named:
        assert call(port.verify_inner_product, args) == 0, (branch, side, j)
        if lax is not None:
            assert call(port.verify_inner_product, args, lax=lax) == 1, (branch, side, j)
    # a batch of every placement with honest proofs around them: exactly those are flagged
    cases = [verify_args(case)] + [x[3] for x in named] + [verify_args(case)]
    assert verify_all(engine, cases) == [1] + [0] * len(named) + [1]


# name -> (encoding mode, the lax decoder that reads the forged bytes as the honest point; s + p is
# odd, so its decoder skips the sign check of the raw bytes too). "s + p"
# is not coverage of the canonical check: the device reads s from the low 255 bits, where s + p is
# s - 19, another point, so only a decoder that reduces all 256 bits mod p is fooled by it. The
# forgery that a decoder like the device's without the canonical check accepts is "s + 2^255".
F_FORGERIES = {"negated": ("ENC_NEGATED", "LAX_SIGN"),
               "s + p": ("ENC_PLUS_P", ("LAX_CANONICAL", "LAX_SIGN", "LAX_MOD_P")),
               "s + 2^255": ("ENC_TOP_BIT", "LAX_CANONICAL")}


def forgery(port, case, side, j, name):
    """(forged verify_args, the lax decoder that reads the forged bytes as the honest point)"""
    mode, lax = F_FORGERIES[name]
    lax_bits = 0
    for flag in (lax if isinstance(lax, tuple) else (lax,)):
        lax_bits |= getattr(port, flag)
    forged = encoded_case(port, case, side, j, getattr(port, mode))
    honest = dec(case[side][j])[0]
    assert dec(forged[side][j])[0] == {"negated": P - honest, "s + p": honest + P,
                                       "s + 2^255": honest + 2**255}[name]
    return verify_args(forged, a_commit=case["a_commit"]), lax_bits


@pytest.mark.parametrize("engine", engines(), indirect=True)
@pytest.mark.parametrize("n,offset", ((3, 0), (16, 60)))
def test_malleable_encodings_are_rejected(engine, n, offset, port):
    case = honest_case(port, 60 + n, n, offset)
    control = verify_args(case)
    assert call(port.verify_inner_product, control) == 1
    forged = []
    for side, j in positions(len(case["l"])):
        for name in F_FORGERIES:
            args, lax = forgery(port, case, side, j, name)
            # one encoding check away from acceptance: the lax decoder accepts, the RFC's rejects
            assert call(port.verify_inner_product, args, lax=lax) == 1, (name, side, j)
            assert call(port.verify_inner_product, args) == 0, (name, side, j)
            forged.append(args)
    assert verify_all(engine, [control] + forged + [control]) == [1] + [0] * len(forged) + [1]


# ---- G: mixed batches ---------------------------------------------------------------------------------------
def g_batch(max_n):
    """n = 1 beside the largest n, repeated proofs, every scalar class, offsets across the table"""
    big = 1025 if max_n > EMUL_MAX_N else 129
    spec = [(1, "unreduced", 0), (big, "unreduced", 1), (2, "l - 1", 63), (big, "last a only", 0),
            (1, "canonical", 2), (65, "a zero", 30), (3, "b zero", 62), (64, "canonical", 1),
            (33, "near 2^256", 40), (big, "unreduced", 1)]  # the last one repeats the second
    t0, a_list, b_list, offs = [], [], [], []
    for i, (n, cls, off) in enumerate(spec):
        seed = 1 if (n, cls, off) == spec[1] else 70 + i
        t, a, b = prove_case(seed, n, cls)
        t0.append(t)
        a_list.append(a)
        b_list.append(b)
        offs.append(off)
    return np.stack(t0), a_list, b_list, offs


@pytest.mark.parametrize("engine", engines(), indirect=True)
def test_mixed_batch_of_edge_classes(engine, port):
    max_n = EMUL_MAX_N if isinstance(engine, ipa_batch.Engine) else 2**30
    t0, a_list, b_list, offs = g_batch(max_n)
    want, t_want = _prove_singly(port, t0, a_list, b_list, offs)
    got = check_mixed_batch(engine, t0, a_list, b_list, offs)
    assert _same_proofs(got, want)
    assert _same_proofs([got[1]], [got[-1]])


@pytest.mark.parametrize("engine", engines(), indirect=True)
def test_mixed_verify_batch(engine, port):
    """One verify batch of proofs of different n and offsets, honest, equivalent, tampered and
    mis-encoded: the flags are those of the single calls and of the port."""
    big = 1025 if not isinstance(engine, ipa_batch.Engine) else EMUL_MAX_N
    one, large = honest_case(port, 81, 1, 2), honest_case(port, 82, big, 1)
    two, sixteen = honest_case(port, 83, 2, 63), honest_case(port, 84, 16, 60)
    raws = branch_encodings()
    bump = lambda v: enc([dec(v)[0] + 1])[0]
    torsion = point_to_abi(point_add(point_from_abi(sixteen["a_commit"]), TORSION4[1]))
    y0 = encoded_case(port, two, "r", 0, port.ENC_REPLACE, raws["y = 0"][0])
    neg_t = encoded_case(port, large, "l", 3, port.ENC_REPLACE, raws["negative t"][0])
    entries = [
        (verify_args(large), 1),
        (verify_args(one, ap=enc([dec(one["ap"])[0] + L])[0]), 1),
        (verify_args(sixteen, a_commit=torsion), 1),
        (verify_args(large, product=bump(large["product"])), 0),
        (verify_args(one, product=bump(one["product"])), 0),
        (verify_args(sixteen, l=sixteen["r"], r=sixteen["l"]), 0),
        (verify_args(y0), 0),
        (verify_args(neg_t), 0),
        (forgery(port, sixteen, "l", 0, "s + 2^255")[0], 0),
        (verify_args(one), 1),
        (verify_args(two), 1),
        (verify_args(large), 1),  # repeats the first
    ]
    want = [w for _, w in entries]
    assert [call(port.verify_inner_product, args) for args, _ in entries] == want
    assert verify_all(engine, [args for args, _ in entries]) == want
