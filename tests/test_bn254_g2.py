"""bn254 G2 (curve id 5) without a GPU: the pure-Python oracle (tests/bn254_g2_reference.BN) against
the EIP-197 generator and twist, then the product's kernel bodies under the CPU emulation (commitments,
pair levels, degenerate buckets, partials, fixed-base handles, synthetic generators) against the
closed form (sum_i s_i k_i mod r) G over synthetic generators G_i = k_i G, and the Fp2 arithmetic
(b200_field_op field 7) against Python integers. The reference has no G2, so nothing here compares
against it. Commitments are uncompressed affine structs, identity {0, 1, infinity = 1}."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from blitzar_b200 import api
from tests import common
from tests import bn254_g2_reference as g2_reference
from tests import test_bls12_381_g2 as bls
from tests import test_field_arithmetic as fa

CURVE, FIELD = 5, 7
g2 = g2_reference.BN
COMMIT = 136
g2_columns, fixed_cases = bls.g2_columns, bls.fixed_cases


def assert_closed_form(got, cols, k):
    want = g2.closed_form(cols, k)
    assert got.shape == want.shape
    bad = [j for j in range(len(cols)) if not np.array_equal(got[j], want[j])]
    assert not bad, f"columns {bad} differ from the closed form"


def proj_points(res):
    return [g2.from_proj_struct(r) for r in res]


# ---- the oracle ------------------------------------------------------------------------------------
def test_oracle_generator():
    """The EIP-197 generator is on y^2 = x^3 + 3 / (9 + u) and has order r; the identity commitment is
    {0, 1 in Montgomery form, infinity = 1}."""
    assert g2.P % 4 == 3
    assert g2.mul(g2.B2, (9, 1)) == (3, 0)
    assert g2.on_curve(g2.G)
    assert g2.scalar_mul(g2.R_ORDER) is None
    assert g2.scalar_mul(g2.R_ORDER - 1) == g2.point_neg(g2.G)
    p5 = g2.scalar_mul(5)
    assert g2.on_curve(p5) and g2.point_add(g2.scalar_mul(2), g2.scalar_mul(3)) == p5
    assert g2.point_add(p5, p5) == g2.scalar_mul(10) and g2.point_add(p5, g2.point_neg(p5)) is None
    ident = g2.commitment(None)
    assert len(ident) == COMMIT and ident[128:] == bytes([1] + [0] * 7)
    assert ident[:32] == bytes(32) and int.from_bytes(ident[64:96], "little") == (1 << 256) % g2.P
    assert g2.from_affine_struct(np.frombuffer(g2.commitment(g2.G), np.uint8)) == g2.G


# ---- the C ABI -------------------------------------------------------------------------------------
class G2Affine(ctypes.Structure):
    _fields_ = [("X", ctypes.c_uint64 * 8), ("Y", ctypes.c_uint64 * 8), ("infinity", ctypes.c_uint8)]


class G2Projective(ctypes.Structure):
    _fields_ = [("X", ctypes.c_uint64 * 8), ("Y", ctypes.c_uint64 * 8), ("Z", ctypes.c_uint64 * 8)]


def test_header_structs_and_curve_id(tmp_path):
    """The two bn254 G2 structs and the curve id of include/blitzar_b200.h, as a C compiler lays them
    out, match their ctypes mirrors and the sizes blitzar_b200.api uses."""
    src = tmp_path / "sizes.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "blitzar_b200.h"\n'
                   "int main(void) { printf(\"%d %zu %zu %zu %zu\\n\", B200_CURVE_BN254_G2,\n"
                   "  sizeof(struct b200_bn254_g2), offsetof(struct b200_bn254_g2, infinity),\n"
                   "  sizeof(struct b200_bn254_g2_p2), offsetof(struct b200_bn254_g2_p2, Z));\n"
                   "  return 0; }\n")
    exe = tmp_path / "sizes"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(common.ROOT, "include"), str(src),
                           "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got == [CURVE, ctypes.sizeof(G2Affine), G2Affine.infinity.offset,
                   ctypes.sizeof(G2Projective), G2Projective.Z.offset]
    assert got == [5, 136, 128, 192, 128]
    assert api.B200_CURVE_BN254_G2 == CURVE
    assert api.CURVE_SIZES[CURVE] == (192, 136, 136) and api.COMPACT_BYTES[CURVE] == 128
    assert api.FIELD_LIMBS[FIELD] == 16
    assert (g2.AFFINE_BYTES, g2.PROJ_BYTES, g2.COMMIT_BYTES, g2.FLAG) == (136, 192, 136, 128)


# ---- synthetic generators --------------------------------------------------------------------------
def check_synthetic_generators(synth):
    """synth(curve, n, first, projective) at sample indices equals (k_i mod 2^255) G in both layouts."""
    for i in bls.SAMPLES:
        want = g2.scalar_mul(g2_reference.synth_log(i))
        aff = synth(CURVE, 2, i, False)
        assert g2.from_affine_struct(aff[0]) == want, i
        assert aff[0, 128:].tolist() == [0] * 8
        assert g2.from_affine_struct(aff[1]) == g2.scalar_mul(g2_reference.synth_log(i + 1)), i
        assert g2.from_proj_struct(synth(CURVE, 1, i, True)[0]) == want, i


def test_synthetic_generators(emul):
    check_synthetic_generators(emul.synth_generators)


# ---- commitments -----------------------------------------------------------------------------------
def test_commitments_closed_form(emul):
    """Every column shape over 2000 synthetic generators, through the commitment call with and
    without generator offsets, equals the closed form."""
    n = 2000
    gens = emul.synth_generators(CURVE, n)
    cols = g2_columns(np.random.default_rng(5), n)
    k = common.synth_scalars_k(n)
    assert_closed_form(emul.commit(CURVE, cols, gens), cols, k)
    offs = np.arange(len(cols), dtype=np.uint64) * 7
    got = emul.commit_offsets(CURVE, cols, offs, emul.synth_generators(CURVE, n + 7 * len(cols)))
    for j, col in enumerate(cols):
        assert_closed_form(got[j:j + 1], [col], common.synth_scalars_k(n, 7 * j))


def test_forced_pair_levels_and_window_widths(emul):
    """Window widths x batch-affine pair levels x pairs per thread, upload pieces with scratch
    buckets, and column groups, on synthetic generators with duplicated rows and +1 / -1 scalars
    (doublings and cancellations inside the pair levels)."""
    n = 600
    gens = emul.synth_generators(CURVE, n)
    ed = g2.edits(gens)
    ed.duplicate(slice(1, n, 7), 0)
    rng = np.random.default_rng(61)
    cols = common.random_columns(rng, n, [(0, 32, 0), (-13, 16, 1), (0, 2, 0)])
    sg = np.zeros((n, 1), dtype=np.uint8)
    sg[::2], sg[1::2] = 1, 0xFF
    cols += [(np.full((n, 1), 3, dtype=np.uint8), 0), (sg, 1)]
    want = g2.closed_form(cols, ed.k)
    for c, levels, batch in ((4, 1, 4), (4, 3, 5), (6, 2, 32), (3, 5, 0), (2, 6, 64), (0, 6, 1),
                             (7, -1, 0), (13, -1, 0)):
        with emul.options(window_bits=c, pair_levels=levels, pair_batch=batch):
            assert np.array_equal(emul.commit(CURVE, cols, gens), want), (c, levels, batch)
    with emul.options(ranges=3, window_bits=4, pair_levels=2, pair_batch=8):
        assert np.array_equal(emul.commit(CURVE, cols, gens), want)
    with emul.options(ranges=3, group_entries=4000, pair_levels=1):
        assert np.array_equal(emul.commit(CURVE, cols, gens), want)


def degenerate_inputs(synth):
    """Synthetic generators edited so that one-bucket columns (scalar 1) hold only copies of +-P,
    identities, or mixes: rows 0..63 P, 64..127 P / -P alternating, 128..159 P / O alternating,
    160..175 another point Q. Returns (gens, edits, cols); column 9 (32 P - 32 P) and column 13
    (identities only) sum to the identity."""
    n = 176
    base = synth(CURVE, 2, 11, False)  # generators 11 and 12
    gens = np.repeat(base[:1], n, axis=0)
    ed = g2.edits(gens)
    ed.k[:] = common.synth_scalars_k(1, 11)[0]
    gens[160:] = base[1]
    ed.k[160:] = common.synth_scalars_k(1, 12)[0]
    ed.negate(slice(65, 128, 2))
    ed.identity(slice(129, 160, 2))

    def ones(rows):
        col = np.zeros((n, 1), dtype=np.uint8)
        col[rows] = 1
        return (col, 0)

    cols = [ones(slice(0, m)) for m in (2, 4, 8, 16, 32, 64, 3, 5, 7)]
    cols += [ones(slice(64, 128)), ones(slice(64, 69)), ones(slice(128, 160)), ones(slice(127, 162)),
             ones(slice(129, 160, 2)), ones(slice(160, 176))]
    mix = np.random.default_rng(5).choice(np.array([1, 1, 1, 2, 0xFF], dtype=np.uint8), (n, 1))
    cols.append((mix, 1))
    return gens, ed, cols


def test_degenerate_buckets(emul):
    """Buckets holding only copies of +-P, identities and mixes at every level count: P + P,
    P + (-P) and O operands in the pair levels and the gathering level."""
    gens, ed, cols = degenerate_inputs(emul.synth_generators)
    want = g2.closed_form(cols, ed.k)
    assert bytes(want[0]) == g2.commitment(g2.scalar_mul(2 * g2_reference.synth_log(11)))
    assert bytes(want[9]) == bytes(want[13]) == g2.commitment(None)
    for levels in (-1, 1, 2, 3, 4, 5, 6):
        with emul.options(pair_levels=levels):
            assert np.array_equal(emul.commit(CURVE, cols, gens), want), levels


def test_partials_combined(emul):
    """Accumulator points of two generator halves, summed by the combine call, give the commitments
    over the whole range."""
    n = 900
    gens = emul.synth_generators(CURVE, n)
    cols = common.random_columns(np.random.default_rng(10), n, [(0, 32, 0), (0, 8, 1), (-100, 3, 0)])
    half = 450
    parts = [emul.commit_partial(CURVE, [(c[lo:hi], s) for c, s in cols], gens[lo:hi])
             for lo, hi in ((0, half), (half, n))]
    assert parts[0].shape[1] == emul.point_bytes(CURVE) == 3 * 64
    got = emul.combine_partials(CURVE, np.concatenate(parts), 2, len(cols))
    assert_closed_form(got, cols, common.synth_scalars_k(n))


# ---- fixed-base handles ----------------------------------------------------------------------------
def check_fixed(res, cols, k):
    for j, col in enumerate(cols):
        assert g2.from_proj_struct(res[j]) == g2.scalar_mul(g2.dot_logs(col, k)), j


@pytest.mark.parametrize("table_window", [0, 10])
def test_fixed_packed_vlen(emul, table_window):
    """The three fixed-base modes over a handle of synthetic projective generators, with and without
    a fixed-base table, and with partition tables of widths 4 and 8 attached."""
    n = 120
    gens_p = emul.synth_generators(CURVE, n, projective=True)
    k = common.synth_scalars_k(n)
    for kwargs, cols in fixed_cases(np.random.default_rng(13), n):
        m = kwargs["num_outputs"]
        with emul.options(table_window=table_window, table_policy=1 if table_window else 0):
            plain = emul.fixed_msm(CURVE, gens_p, n=n, **kwargs)
            check_fixed(plain, cols, k)
            for w in (4, 8):
                for policy in (emul.POLICY_TABLE, emul.POLICY_MODEL):
                    with emul.options(table_window=table_window, table_policy=1 if table_window else 0,
                                      partition_policy=policy):
                        got = emul.fixed_msm(CURVE, gens_p, n=n, partition_window=w,
                                             chunk_groups=5, **kwargs)
                    assert proj_points(got) == proj_points(plain), (w, policy, m)


def test_partition_table_file_round_trip(emul, tmp_path):
    """The partition table of bn254 G2 generators (128-byte compact entries) gives the generators
    back."""
    n = 37
    gens_p = emul.synth_generators(CURVE, n, projective=True)
    for w in (1, 3, 8):
        table = emul.partition_table(CURVE, gens_p, w)
        assert table.size == -(-n // w) * (128 << w)
        raw = np.concatenate([np.frombuffer(np.uint32(w).tobytes(), np.uint8), table])
        path = str(tmp_path / f"bn254_g2_table_{w}.bin")
        raw.tofile(path)
        back = emul.generators_from_reference_table(CURVE, path)
        assert proj_points(back[:n]) == proj_points(gens_p)
        assert all(p is None for p in proj_points(back[n:]))


# ---- Fp2 arithmetic (field 7) ----------------------------------------------------------------------
FP = fa.Mont(2)
P, RM = FP.p, FP.r
RINV = pow(RM, -1, P)


def _m(a, b):  # Montgomery product of residues
    return a * b * RINV % P


def fp2_model(op, a, b=None):
    """Exact result of field 7 op on Montgomery residues a = (a0, a1) (and b)."""
    if op in ("add", "sub"):
        f = (lambda x, y: (x + y) % P) if op == "add" else (lambda x, y: (x - y) % P)
        return (f(a[0], b[0]), f(a[1], b[1]))
    if op == "neg":
        return (-a[0] % P, -a[1] % P)
    if op == "dbl":
        return (2 * a[0] % P, 2 * a[1] % P)
    if op in ("mul", "mul_ref", "sqr"):
        b = a if op == "sqr" else b
        return ((_m(a[0], b[0]) - _m(a[1], b[1])) % P, (_m(a[0], b[1]) + _m(a[1], b[0])) % P)
    if op in ("invert", "invert_eea"):
        if a == (0, 0):
            return (0, 0)
        i = g2.inv(a)
        return (i[0] * RM * RM % P, i[1] * RM * RM % P)
    if op == "from_mont":
        return (_m(a[0], 1), _m(a[1], 1))
    if op == "to_mont":
        return (a[0] * RM % P, a[1] * RM % P)
    raise ValueError(op)


def fp2_limbs(elems):
    return fa.to_limbs([e[0] | e[1] << 256 for e in elems], 16)


def fp2_values(arr):
    return [(v & (RM - 1), v >> 256) for v in fa.from_limbs(arr)]


def fp2_operands(seed):
    """Elements whose components run over the bn254 edge values of tests/test_field_arithmetic.py
    (0, 1, 2, p - 1, p - 2, (p +- 1)/2, R and R^-1 mod p, 2^(32k) - 1, limbs forced to all ones,
    equal or zero halves): each edge e as (e, 0), (0, e), (e, e), (e, p - 1 - e) and next to a random
    component, plus random elements. Returns (elements, binary pairs, the unreduced edge values)."""
    rng = random.Random(seed)
    raw = fa.variants(fa.edge_values(P, 8) | {P, P + 1, RM - 1, RM - P}, 8)
    edges = sorted({v % P for v in raw})
    elems = []
    for e in edges:
        elems += [(e, 0), (0, e), (e, e), (e, P - 1 - e), (e, rng.randrange(P)), (rng.randrange(P), e)]
    elems += [(rng.randrange(P), rng.randrange(P)) for _ in range(2048)]
    few = edges[::9]
    corner = [(x, y) for x in few for y in few]
    pairs = [(a, b) for a in corner for b in corner[::7]]
    pairs += list(zip(elems, elems[1:] + elems[:1])) + list(zip(elems, reversed(elems)))
    return elems, pairs, raw


def check_fp2(engine):
    elems, pairs, raw = fp2_operands(7)
    for op in ("add", "sub", "mul", "mul_ref"):
        got = fp2_values(engine.field_op(FIELD, op, fp2_limbs([a for a, _ in pairs]),
                                         fp2_limbs([b for _, b in pairs])))
        for (a, b), g in zip(pairs, got):
            assert g == fp2_model(op, a, b), (op, a, b)
    for op in ("neg", "dbl", "sqr", "from_mont", "invert", "invert_eea"):
        got = fp2_values(engine.field_op(FIELD, op, fp2_limbs(elems)))
        for a, g in zip(elems, got):
            assert g == fp2_model(op, a), (op, a)
    # to_mont reduces any component below R
    wide = [(x, y) for x, y in zip(raw, reversed(raw))] + [(RM - 1, 0), (0, RM - 1)]
    got = fp2_values(engine.field_op(FIELD, "to_mont", fp2_limbs(wide)))
    assert got == [fp2_model("to_mont", a) for a in wide]
    # the zcash rule: c1 decides unless it is 0
    largest = engine.field_op(FIELD, "lexicographically_largest", fp2_limbs(elems))[:, 0].tolist()
    plain = [fp2_model("from_mont", a) for a in elems]
    assert largest == [int(g2.lex_largest(v)) for v in plain]
    assert {(v[1] == 0, bool(w)) for v, w in zip(plain, largest)} == {(True, True), (True, False),
                                                                      (False, True), (False, False)}
    # operations the field does not offer
    for op in ("mul_lat", "canonical", "pow22523"):
        with pytest.raises(ValueError):
            engine.field_op(FIELD, op, fp2_limbs(elems[:1]), fp2_limbs(elems[:1]))


def test_fp2_field_op(emul):
    check_fp2(emul)
