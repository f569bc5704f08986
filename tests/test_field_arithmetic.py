"""The field arithmetic under every kernel (field.cuh, lanefield.cuh) and the host scalars mod l
(scalar25.h) against Python integers, one operation at a time (b200_field_op on the GPU, the same
bodies with emulated carries in the CPU emulation).

The model predicts exact limbs, including which loosely reduced representative an F25519 operation
returns, and records which correction each case takes: the wraps of add, the borrows of sub, the
second wrap of the 2^256 = 38 fold, the branches of canonical, Montgomery final subtractions. Every
test asserts that each correction of each operation was taken at least once; the tables print with
`pytest -rP`. Operands are the edge values of each field (0, 1, 2, p - 1, p - 2, (p +- 1)/2, R and
R^-1 mod p, 2^(32k) - 1, and for F25519 p, p + 18, 2^255, 2^256 - 38, 2^256 - 1), each also with
one limb forced to all ones and with equal or zero halves, in full cross product for binary
operations, operands solved for the rarest branches, and 2^16 seeded random pairs."""
import collections
import random

import numpy as np
import pytest

ENGINES = [pytest.param("emul", id="emul"), pytest.param("gpu", id="gpu", marks=pytest.mark.gpu)]
RANDOM = 1 << 16  # random pairs per operation
LADDER_RANDOM = 1 << 10  # random operands of the exponentiation ladders

P25519 = 2**255 - 19
SQRT_M1 = pow(2, (P25519 - 1) // 4, P25519)
L25519 = 2**252 + 27742317777372353535851937790883648493
M256 = 2**256 - 1
MODULI = {  # Montgomery fields: field id -> (p, limbs)
    1: (0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab, 12),
    2: (21888242871839275222246405745257275088696311157297823662689037894645226208583, 8),
    3: (21888242871839275222246405745257275088548364400416034343698204186575808495617, 8),
    4: (L25519, 8),
}
BN254_TO_MONT_REGRESSION = 0xffffffffffffffffbb341875091327163df8432a107a27527357ae2c0975fbde
FIELD_NAMES = {0: "curve25519", 1: "bls12-381", 2: "bn254", 3: "grumpkin", 4: "scalars mod l"}


@pytest.fixture
def engine(request):
    return request.getfixturevalue("emul" if request.param == "emul" else "bb")


# ---- limbs <-> integers ----------------------------------------------------------------------------
def to_limbs(values, width):
    raw = b"".join(v.to_bytes(4 * width, "little") for v in values)
    return np.frombuffer(raw, dtype=np.uint32).reshape(-1, width)


def from_limbs(arr):
    arr = np.ascontiguousarray(arr, dtype=np.uint32)
    w, raw = 4 * arr.shape[1], arr.tobytes()
    return [int.from_bytes(raw[i * w:(i + 1) * w], "little") for i in range(arr.shape[0])]


# ---- operands --------------------------------------------------------------------------------------
def variants(values, limbs):
    """Each value, with one limb forced to all ones, and with equal or zero halves."""
    bits, half = 32 * limbs, 16 * limbs
    lo_mask = (1 << half) - 1
    out = set()
    for v in values:
        out.add(v)
        out.update(v | (0xFFFFFFFF << (32 * k)) for k in range(limbs))
        lo, hi = v & lo_mask, v >> half
        out.update([lo | (lo << half), hi | (hi << half), hi << half, lo])
    return sorted(x for x in out if x < 1 << bits)


def edge_values(p, limbs):
    r = 1 << (32 * limbs)
    vals = {0, 1, 2, p - 1, p - 2, (p - 1) // 2, (p + 1) // 2}
    vals.update((1 << (32 * k)) - 1 for k in range(1, limbs + 1) if (1 << (32 * k)) - 1 < p)
    if p != P25519:
        vals.update([r % p, pow(r, -1, p)])
    return vals


def f25519_fold_wrap_operands():
    """Operands whose product takes the second wrap of the fold (c2 = 1): a = 2^255 with b = 2x + 1,
    38x = -2^255 - 2 (mod 2^256); and a = b = 2^256 - 38 - c for c in 7..37 (a^2 = c^2 mod
    2^256 - 38)."""
    t = (-(2**255) - 2) % 2**256
    x = (t // 2) * pow(19, -1, 2**255) % 2**255
    return [2**255, 2 * x + 1, 2**256 - 45, 2**256 - 75]


def f25519_edges():
    return edge_values(P25519, 8) | {P25519, P25519 + 18, 2**255, 2**256 - 38, 2**256 - 1} | \
        set(f25519_fold_wrap_operands())


def cross(values):
    return [(a, b) for a in values for b in values]


def random_pairs(rng, bound, count):
    return [(rng.randrange(bound), rng.randrange(bound)) for _ in range(count)]


# ---- the model -------------------------------------------------------------------------------------
def f25519_add(a, b):
    s = a + b
    if s >> 256 == 0:
        return s, "no wrap"
    s = (s & M256) + 38
    if s >> 256 == 0:
        return s, "one wrap"
    return (s & M256) + 38, "two wraps"


def f25519_sub(a, b):
    d = a - b
    if d >= 0:
        return d, "no borrow"
    d += 2**256 - 38
    if d >= 0:
        return d, "one borrow"
    return d + 2**256 - 38, "two borrows"


def f25519_fold(t):
    """512-bit product -> loosely reduced residue: lo + 38 hi, then the carry limb times 38, then a
    second wrap of 38 (c2)."""
    t = (t & M256) + 38 * (t >> 256)
    r = (t & M256) + 38 * (t >> 256)
    if r >> 256 == 0:
        return r, "c2 = 0"
    return (r & M256) + 38, "c2 = 1"


def f25519_mul(a, b):
    return f25519_fold(a * b)


def f25519_canonical(v):
    top = v >> 255
    w = (v & (2**255 - 1)) + 19 * top
    ge = (w + 19) >> 255
    r = (w + 19) & (2**255 - 1) if ge else w
    assert r == v % P25519
    return r, f"top bit {top}, >= p {ge}"


def radix51(v):
    return [(v >> (51 * i)) & (2**51 - 1) for i in range(4)] + [v >> 204]


def f25519_from_radix51(h):
    v = sum(x << (51 * i) for i, x in enumerate(h))
    t = (v & M256) + 38 * (v >> 256)
    label = "fold wraps" if t >> 256 else "no wrap"
    r = (t & M256) + 38 * (t >> 256)
    assert r >> 256 == 0  # v < 2^268: the second fold cannot wrap
    return r, label


def sqrt_ratio_m1(u, v):
    """RFC 9496 section 4.2, SQRT_RATIO_M1: (was_square, the non-negative r) and the case taken."""
    p = P25519
    u, v = u % p, v % p
    r = u * pow(v, 3, p) * pow(u * pow(v, 7, p), (p - 5) // 8, p) % p
    check = v * r * r % p
    correct, flipped, flipped_i = check == u, check == (-u) % p, check == (-u * SQRT_M1) % p
    if flipped or flipped_i:
        r = SQRT_M1 * r % p
    if r & 1:
        r = p - r
    if u == 0:
        case = "u = 0"
    elif v == 0:
        case = "v = 0"
    else:
        case = ("check = u" if correct else "check = -u" if flipped else
                "check = -u i" if flipped_i else "check = u i")
    return r, int(correct or flipped), case


class Mont:
    def __init__(self, field):
        self.p, self.limbs = MODULI[field]
        self.r = 1 << (32 * self.limbs)
        self.pinv = pow(self.p, -1, self.r)
        self.r2 = self.r * self.r % self.p

    def mul(self, a, b):
        """CIOS product for a b < R p: (a b + m p) / R < 2p, one final subtraction."""
        t = a * b
        u = (t + (-t * self.pinv % self.r) * self.p) // self.r
        assert u < 2 * self.p
        return (u - self.p, "final subtraction") if u >= self.p else (u, "no final subtraction")

    def add(self, a, b):
        s = a + b
        return (s - self.p, "subtract p") if s >= self.p else (s, "keep")

    def sub(self, a, b):
        d = a - b
        return (d + self.p, "add p back") if d < 0 else (d, "keep")

    def invert(self, x):
        return (0, "zero") if x == 0 else (self.r2 * pow(x, -1, self.p) % self.p, "nonzero")


# ---- running and checking --------------------------------------------------------------------------
class Coverage:
    """Which branch every case of every operation took, against the branches each must reach."""

    def __init__(self, title):
        self.title, self.seen, self.expected = title, collections.defaultdict(collections.Counter), {}

    def add(self, op, labels, expected):
        self.seen[op].update(labels)
        self.expected[op] = set(expected)

    def check(self):
        print(f"\n{self.title}: cases per branch")
        for op in self.seen:
            print(f"  {op:26s} " + ", ".join(f"{k}: {v}" for k, v in sorted(self.seen[op].items())))
        missing = {op: sorted(e - set(self.seen[op])) for op, e in self.expected.items()
                   if e - set(self.seen[op])}
        assert not missing, f"{self.title}: branches never taken: {missing}"


def run(engine, field, op, a_values, width, b_values=None):
    a = to_limbs(a_values, width)
    b = None if b_values is None else to_limbs(b_values, width)
    return engine.field_op(field, op, a, b)


def check_exact(engine, field, op, cases, model, width, cov=None, expected=()):
    """cases: [(a,)] or [(a, b)]; model(*case) -> (want, label)."""
    binary = len(cases[0]) == 2
    got = from_limbs(run(engine, field, op, [c[0] for c in cases], width,
                         [c[1] for c in cases] if binary else None))
    labels = []
    for case, g in zip(cases, got):
        want, label = model(*case)
        assert g == want, f"{FIELD_NAMES[field]} {op}{tuple(hex(x) for x in case)}: " \
                          f"got {g:#x}, want {want:#x} ({label})"
        labels.append(label)
    if cov is not None:
        cov.add(op, labels, expected)


# ---- curve25519 base field -------------------------------------------------------------------------
@pytest.mark.parametrize("engine", ENGINES, indirect=True)
def test_f25519_exact_representatives(engine):
    """add, sub, neg, dbl, mul, mul_ref, mul_lat, sqr return exactly the model's loosely reduced
    representative; canonical, is_negative and to_radix51 are exact on v mod p."""
    rng = random.Random(25519)
    edges = variants(f25519_edges(), 8)
    pairs = cross(edges) + random_pairs(rng, 2**256, RANDOM)
    wrap = f25519_fold_wrap_operands()
    pairs += [(wrap[0], wrap[1]), (wrap[1], wrap[0])]
    singles = [(a,) for a in edges] + [(rng.randrange(2**256),) for _ in range(RANDOM)]
    cov = Coverage("F25519")
    wraps, borrows, c2 = ("no wrap", "one wrap", "two wraps"), \
        ("no borrow", "one borrow", "two borrows"), ("c2 = 0", "c2 = 1")
    check_exact(engine, 0, "add", pairs, f25519_add, 8, cov, wraps)
    check_exact(engine, 0, "sub", pairs, f25519_sub, 8, cov, borrows)
    check_exact(engine, 0, "neg", singles, lambda a: f25519_sub(0, a), 8, cov, borrows)
    check_exact(engine, 0, "dbl", singles, lambda a: f25519_add(a, a), 8, cov, wraps)
    for op in ("mul", "mul_ref", "mul_lat"):
        check_exact(engine, 0, op, pairs, f25519_mul, 8, cov, c2)
    check_exact(engine, 0, "sqr", singles, lambda a: f25519_mul(a, a), 8, cov, c2)
    canon = [f"top bit {t}, >= p {g}" for t in (0, 1) for g in (0, 1)]
    check_exact(engine, 0, "canonical", singles, f25519_canonical, 8, cov, canon)

    a = [s[0] for s in singles]
    neg = engine.field_op(0, "is_negative", to_limbs(a, 8))
    assert neg[:, 0].tolist() == [(v % P25519) & 1 for v in a]
    h = engine.field_op(0, "to_radix51", to_limbs(a, 8)).view(np.uint64)
    assert h.tolist() == [radix51(v % P25519) for v in a]
    cov.check()


@pytest.mark.parametrize("engine", ENGINES, indirect=True)
def test_f25519_from_radix51(engine):
    """Unreduced radix-2^51 limbs (any u64) fold to the model's representative."""
    rng = random.Random(51)
    limbs = [[2**64 - 1] * 5, [2**51 - 1] * 5, [0] * 5, [2**51] * 5, radix51(2**257 - 1),
             radix51(2**268 - 1), radix51(P25519), radix51(2**256 - 1)]
    limbs += [[rng.randrange(2**64) for _ in range(5)] for _ in range(RANDOM)]
    limbs += [radix51(rng.randrange(2**268)) for _ in range(1024)]
    cov = Coverage("F25519 from_radix51")
    arr = np.array(limbs, dtype=np.uint64).view(np.uint32)
    got = from_limbs(engine.field_op(0, "from_radix51", arr))
    labels = []
    for h, g in zip(limbs, got):
        want, label = f25519_from_radix51(h)
        assert g == want, (h, hex(g), hex(want))
        labels.append(label)
    cov.add("from_radix51", labels, ["no wrap", "fold wraps"])
    cov.check()


@pytest.mark.parametrize("engine", ENGINES, indirect=True)
def test_f25519_ladders_and_sqrt_ratio(engine):
    """invert and pow22523 are congruent to a^(p-2) and a^((p-5)/8); sqrt_ratio_m1 equals RFC 9496
    section 4.2, including u = 0, v = 0 and the non-square cases."""
    rng = random.Random(22523)
    base = sorted(f25519_edges())
    a = variants(base, 8) + [rng.randrange(2**256) for _ in range(LADDER_RANDOM)]
    p = P25519
    inv = from_limbs(engine.field_op(0, "invert", to_limbs(a, 8)))
    assert [x % p for x in inv] == [pow(v, p - 2, p) for v in a]
    pw = from_limbs(engine.field_op(0, "pow22523", to_limbs(a, 8)))
    assert [x % p for x in pw] == [pow(v, (p - 5) // 8, p) for v in a]

    pairs = cross(base) + random_pairs(rng, 2**256, LADDER_RANDOM)
    got = engine.field_op(0, "sqrt_ratio_m1", to_limbs([u for u, _ in pairs], 8),
                          to_limbs([v for _, v in pairs], 8))
    xs, flags = from_limbs(got[:, :8]), got[:, 8].tolist()
    cov = Coverage("F25519 sqrt_ratio_m1")
    labels = []
    for (u, v), x, flag in zip(pairs, xs, flags):
        r, was_square, case = sqrt_ratio_m1(u, v)
        assert (x % p, flag) == (r, was_square), (hex(u), hex(v), case)
        labels.append(case)
    cov.add("sqrt_ratio_m1", labels,
            ["u = 0", "v = 0", "check = u", "check = -u", "check = -u i", "check = u i"])
    cov.check()


# ---- Montgomery fields -----------------------------------------------------------------------------
@pytest.mark.parametrize("field", [1, 2, 3, 4], ids=lambda f: FIELD_NAMES[f])
@pytest.mark.parametrize("engine", ENGINES, indirect=True)
def test_montgomery_field(engine, field):
    """mul = a b R^-1 mod p exactly for canonical operands, and for a < p with any b < R;
    to_mont(a) = a R mod p for any a < R (how IpaReduceBody reduces raw caller scalars); add and
    sub on canonical operands; invert and invert_eea map x to R^2 x^-1 and 0 to 0; from_mont and
    lexicographically_largest."""
    F = Mont(field)
    p, n = F.p, F.limbs
    rng = random.Random(1000 + field)
    raw = variants(edge_values(p, n) | {p, p + 1, F.r - 1, F.r - p}, n)  # every value < R
    canon = sorted({v % p for v in raw})
    pairs = cross(canon) + random_pairs(rng, p, RANDOM)
    singles = [(a,) for a in canon] + [(rng.randrange(p),) for _ in range(RANDOM)]
    # the product's first operand must be below p: with a = 2^256 - 2^224 + 1 >= l as the FIRST
    # operand and b = 2^64 - 2^32, the scalars mod l came out 2^64 short (a carry out of the top
    # frame limb); the schedule takes unreduced values as its second operand
    wide = [(a, b) for a in canon[::3] for b in raw + [F.r - F.r // 2**32 + 1]] + \
        [(2**64 - 2**32, F.r - F.r // 2**32 + 1)] + \
        [(rng.randrange(p), rng.randrange(F.r)) for _ in range(RANDOM)]
    cov = Coverage(f"{FIELD_NAMES[field]} Montgomery")
    fin = ("final subtraction", "no final subtraction")
    check_exact(engine, field, "add", pairs, F.add, n, cov, ("subtract p", "keep"))
    check_exact(engine, field, "sub", pairs, F.sub, n, cov, ("add p back", "keep"))
    check_exact(engine, field, "neg", singles, lambda a: F.sub(0, a), n, cov, ("add p back", "keep"))
    check_exact(engine, field, "dbl", singles, lambda a: F.add(a, a), n, cov, ("subtract p", "keep"))
    for op in ("mul", "mul_ref"):
        check_exact(engine, field, op, pairs, F.mul, n, cov, fin)
    check_exact(engine, field, "mul", wide, F.mul, n)
    check_exact(engine, field, "sqr", singles, lambda a: F.mul(a, a), n, cov, fin)
    # to_mont once passed the raw value as the product's first operand: wrong for about half of
    # the values >= p in bn254, e.g. 0xffffffffffffffffbb34...fbde
    wide1 = [(a,) for a in raw + [F.r - F.r // 2**32 + 1, BN254_TO_MONT_REGRESSION]
             if a < F.r] + [(rng.randrange(F.r),) for _ in range(RANDOM)]
    check_exact(engine, field, "to_mont", wide1, lambda a: F.mul(a, F.r2), n, cov, fin)
    check_exact(engine, field, "from_mont", wide1, lambda a: F.mul(a, 1), n, cov, fin)

    a = [s[0] for s in singles[:len(canon) + LADDER_RANDOM]]
    for op in ("invert", "invert_eea"):
        check_exact(engine, field, op, [(x,) for x in a], F.invert, n, cov, ("zero", "nonzero"))
    largest = engine.field_op(field, "lexicographically_largest", to_limbs(a, n))[:, 0].tolist()
    want = [int(x * pow(F.r, -1, p) % p > (p - 1) // 2) for x in a]
    assert largest == want
    cov.add("lexicographically_largest", ["largest" if w else "not largest" for w in want],
            ["largest", "not largest"])
    cov.check()


# ---- lane-sliced curve25519 field (device only) ----------------------------------------------------
LANE_POS = [(51 * m + 1) // 2 for m in range(10)]  # limb m sits at bit ceil(25.5 m)
LANE_BITS = [26 - (m & 1) for m in range(10)]
TWO_P = [0x7FFFFDA] + [0x3FFFFFE if m & 1 else 0x7FFFFFE for m in range(1, 10)]  # limbs of 2p


def lane_value(limbs):
    return sum(x << LANE_POS[m] for m, x in enumerate(limbs))


def per_parity(even, odd):
    return [odd if m & 1 else even for m in range(10)]


def lane_check(engine, op, a_rows, b_rows=None, bound=None, want=None):
    """Runs op on rows of 10 limbs; every result congruent to want(a, b) mod p and every limb below
    bound[m]."""
    b = None if b_rows is None else np.array(b_rows, dtype=np.uint32)
    got = engine.field_op(5, op, np.array(a_rows, dtype=np.uint32), b).astype(np.int64).tolist()
    for i, g in enumerate(got):
        args = (a_rows[i],) if b_rows is None else (a_rows[i], b_rows[i])
        assert lane_value(g) % P25519 == want(*args) % P25519, (op, args, g)
        if bound is not None:
            assert all(x < bound[m] for m, x in enumerate(g)), (op, args, g, bound)
    return got


@pytest.mark.gpu
def test_lane_field_at_its_documented_bounds(bb):
    """Each lane10 operation on operands at the bound its comment documents, at the exact integer
    limit the code allows, and on random operands below them: results congruent mod p, every limb
    within the stated output bound."""
    rng = random.Random(10)
    V = lane_value
    mul_out = per_parity(2**26 + 2**22, 2**25 + 2**22)
    carry_out = per_parity(2**26 + 2**12, 2**25 + 2**12)

    def rows(bound, k=RANDOM // 16):
        return [[rng.randrange(bound[m]) for m in range(10)] for _ in range(k)]

    # slice: any value < 2^256, exactly; limb 9 keeps 26 bits
    vals = sorted(f25519_edges()) + [rng.randrange(2**256) for _ in range(4096)]
    sl = bb.field_op(5, "slice", to_limbs(vals, 8)).astype(np.int64).tolist()
    assert [lane_value(s) for s in sl] == vals
    assert all(s[m] < 2**(26 if m == 9 else LANE_BITS[m]) for s in sl for m in range(10))
    # gather: limbs up to 2^32 - 1
    top = [[2**32 - 1] * 10] + rows([2**32] * 10)
    got = from_limbs(bb.field_op(5, "gather", np.array(top, dtype=np.uint32)))
    assert [g % P25519 for g in got] == [V(t) % P25519 for t in top]
    # carry1: inputs up to 2^32 - 1
    lane_check(bb, "carry1", top, bound=carry_out, want=V)
    # mul: a, b < 2^27.7 on even limbs, one bit less on odd ones; and every limb at the largest b
    # with 19 b < 2^32
    doc = per_parity(int(2**27.7), int(2**26.7))
    exact = [(2**32 - 1) // 19] * 10
    for a_max, b_max in ((doc, doc), (exact, exact), (doc, exact)):
        a_rows, b_rows = [a_max, a_max] + rows(a_max), [b_max, [0] * 10] + rows(b_max)
        lane_check(bb, "mul", a_rows, b_rows, mul_out, lambda a, b: V(a) * V(b))
    # add (lazy) of two products; sub2p of a carried value and a product (b <= 2p limb-wise);
    # sub4p of 0 and up to twice a product (b <= 4p limb-wise: 2^27.9 even, one bit less odd)
    prod = [[x - 1 for x in mul_out]] + rows(mul_out)
    lane_check(bb, "add", prod, prod[::-1], per_parity(2**32, 2**32), lambda a, b: V(a) + V(b))
    carried = [[x - 1 for x in carry_out]] + rows(carry_out, len(prod) - 1)
    lane_check(bb, "sub2p", carried, prod, None, lambda a, b: V(a) - V(b))
    lane_check(bb, "sub2p", [[0] * 10], [TWO_P], None, lambda a, b: V(a) - V(b))
    sub4_doc = per_parity(int(2**27.9), int(2**26.9))
    four_p = [2 * x for x in TWO_P]
    for b_max in (sub4_doc, four_p):
        b_rows = [b_max] + rows([x + 1 for x in b_max])
        lane_check(bb, "sub4p", [[0] * 10] * len(b_rows), b_rows, None, lambda a, b: V(a) - V(b))
    # pow22523 of operands at the multiplier's documented bound
    a_rows = [doc] + rows(doc, 512)
    lane_check(bb, "pow22523", a_rows, None, mul_out,
               lambda a: pow(V(a), (P25519 - 5) // 8, P25519))


def test_lane_field_is_device_only(emul):
    with pytest.raises(ValueError):
        emul.field_op(5, "mul", np.zeros((1, 10), np.uint32), np.zeros((1, 10), np.uint32))


# ---- host scalars mod l (scalar25.h) ---------------------------------------------------------------
def test_host_scalars(emul):
    """sc_reduce of any 256-bit value, sc_mul, sc_mul_mont(sc_to_mont(a), b), sc_add, sc_sub,
    sc_neg, sc_inv and sc_inner_product: exact canonical residues mod l."""
    l = L25519
    rng = random.Random(252)
    F = Mont(4)
    raw = variants(edge_values(l, 8) | {l, l + 1, 2 * l, 15 * l, 2**256 - 1, 2**255}, 8)
    canon = sorted({v % l for v in raw})
    pairs = cross(canon) + random_pairs(rng, l, RANDOM)
    a, b = [x for x, _ in pairs], [y for _, y in pairs]

    def sc(op, xs, ys=None):
        return from_limbs(emul.scalar_op(op, to_limbs(xs, 8), None if ys is None else to_limbs(ys, 8)))

    wide = raw + [rng.randrange(2**256) for _ in range(RANDOM)]
    assert sc("reduce", wide) == [v % l for v in wide]
    assert sc("mul", a, b) == [x * y % l for x, y in pairs]
    assert sc("mul_mont", a, b) == [x * y % l for x, y in pairs]
    assert sc("add", a, b) == [(x + y) % l for x, y in pairs]
    assert sc("sub", a, b) == [(x - y) % l for x, y in pairs]
    assert sc("neg", canon) == [-x % l for x in canon]
    inv_in = canon + [rng.randrange(l) for _ in range(256)]
    assert sc("inv", inv_in) == [pow(x, l - 2, l) for x in inv_in]
    for n in (1, 2, 7, 64, 1000):
        xs, ys = [rng.randrange(l) for _ in range(n)], [rng.randrange(l) for _ in range(n)]
        assert sc("inner_product", xs, ys) == [sum(x * y for x, y in zip(xs, ys)) % l]
    assert sc("inner_product", [l - 1] * 1000, [l - 1] * 1000) == [1000 % l]

    cov = Coverage("host scalars")
    cov.add("add", [F.add(x, y)[1] for x, y in pairs], ("subtract p", "keep"))
    cov.add("sub", [F.sub(x, y)[1] for x, y in pairs], ("add p back", "keep"))
    cov.add("mul (first product)", [F.mul(x, y)[1] for x, y in pairs],
            ("final subtraction", "no final subtraction"))
    cov.check()
