"""Many inner-product arguments per call (b200_curve25519_prove_inner_products / _verify_): every
proof and transcript of a batch is byte-identical to the single call on that proof alone, on the
reference fixtures (tests/golden/inner_product.npz), on mixed batches and on tampered proofs. The
CPU cases run the batched kernel bodies through the emulation; the GPU cases the product library."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import common
from tests.emul import ipa_batch

L = 2**252 + 27742317777372353535851937790883648493
MIXED_N = (1, 2, 3, 5, 64, 100, 1000)
MIXED_OFFSETS = (0, 3, 70)  # 70 straddles the 64 precomputed generators of the GPU cases
IN_TABLE_N, IN_TABLE_OFFSETS = (2, 3, 5, 16, 20), (0, 3, 30)  # [offset, offset + np] within 64


def _scalars(rng, n):
    s = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    s[:, 31] &= 0x0F
    return s


def _transcripts(rng, count):
    t = np.zeros((count, 203), np.uint8)
    t[:, :200] = rng.integers(0, 256, (count, 200), dtype=np.uint8)
    return t


def _same_proofs(got, want):
    return len(got) == len(want) and all(
        np.array_equal(x, y) for g, w in zip(got, want) for x, y in zip(g, w))


def _prove_singly(engine, t0, a_list, b_list, offsets):
    """(proofs, advanced transcripts) of the single call on each proof alone."""
    ts = t0.copy()
    return [engine.prove_inner_product(ts[p], a, b, int(o))
            for p, (a, b, o) in enumerate(zip(a_list, b_list, offsets))], ts


def _fixture():
    z = np.load(os.path.join(common.GOLDEN, "inner_product.npz"))
    cases = list(range(int(z["num_cases"])))
    return z, int(z["generators_offset"]), cases


def check_fixture_as_one_batch(engine):
    z, off, cases = _fixture()
    t = np.stack([z[f"t0_{c}"] for c in cases])
    b_list = [z[f"b{c}"] for c in cases]
    proofs = engine.prove_inner_products(t, [z[f"a{c}"] for c in cases], b_list, [off] * len(t))
    for c, (lv, rv, ap) in zip(cases, proofs):
        assert np.array_equal(lv, z[f"l{c}"]) and np.array_equal(rv, z[f"r{c}"]), c
        assert np.array_equal(ap, z[f"ap{c}"]), c
        assert np.array_equal(t[c], z[f"t1_{c}"]), c
    tv = np.stack([z[f"t0_{c}"] for c in cases])
    res = engine.verify_inner_products(tv, b_list, np.stack([z[f"product{c}"] for c in cases]),
                                       np.stack([z[f"acommit{c}"] for c in cases]),
                                       [p[0] for p in proofs], [p[1] for p in proofs],
                                       np.stack([p[2] for p in proofs]), [off] * len(tv))
    assert res.tolist() == [1] * len(tv)
    assert all(np.array_equal(tv[c], z[f"t1_{c}"]) for c in cases)


def mixed_batch(seed, ns=MIXED_N, offsets=MIXED_OFFSETS):
    rng = np.random.default_rng(seed)
    a_list = [_scalars(rng, n) for n in ns]
    b_list = [_scalars(rng, n) for n in ns]
    offs = [offsets[i % len(offsets)] for i in range(len(ns))]
    return _transcripts(rng, len(ns)), a_list, b_list, offs


def check_mixed_batch(engine, t0, a_list, b_list, offs, other=None):
    """Batch == the engine's single calls (and == `other`'s single calls when given)."""
    want, t_want = _prove_singly(engine, t0, a_list, b_list, offs)
    t = t0.copy()
    got = engine.prove_inner_products(t, a_list, b_list, offs)
    assert _same_proofs(got, want) and np.array_equal(t, t_want)
    if other is not None:
        want2, t_want2 = _prove_singly(other, t0, a_list, b_list, offs)
        assert _same_proofs(got, want2) and np.array_equal(t, t_want2)
    return got


def check_tampered_verify(engine):
    """The fixture's proofs as one batch with a tampered product (n = 1), an L replaced by an R
    (n = 5) and an L that does not decode (n = 37): the results flag exactly those three, and every
    transcript advances as the single verify advances it."""
    z, off, cases = _fixture()
    b_list = [z[f"b{c}"] for c in cases]
    l_list = [z[f"l{c}"].copy() for c in cases]
    r_list = [z[f"r{c}"] for c in cases]
    products = np.stack([z[f"product{c}"] for c in cases])
    acommits = np.stack([z[f"acommit{c}"] for c in cases])
    ap = np.stack([z[f"ap{c}"] for c in cases])
    ns = [b.shape[0] for b in b_list]
    bad_product, swapped, undecodable = ns.index(1), ns.index(5), ns.index(37)
    products[bad_product][0] ^= 1
    l_list[swapped][0] = r_list[swapped][0]
    l_list[undecodable][2] = 0xFF  # not a canonical field element
    t0 = np.stack([z[f"t0_{c}"] for c in cases])
    t = t0.copy()
    res = engine.verify_inner_products(t, b_list, products, acommits, l_list, r_list, ap,
                                       [off] * len(cases))
    assert sorted(np.flatnonzero(res == 0).tolist()) == sorted([bad_product, swapped, undecodable])
    for p in cases:
        ts = t0[p].copy()
        single = engine.verify_inner_product(ts, b_list[p], products[p], acommits[p], l_list[p],
                                             r_list[p], ap[p], off)
        assert single == res[p] and np.array_equal(ts, t[p]), p


def check_empty_and_repeated(engine, prove_entry, verify_entry):
    # num_proofs == 0 leaves every output buffer untouched
    ptr = lambda x: C.c_void_p(x.ctypes.data)
    lv, rv, ap = (np.full((4, 32), 0xA5, np.uint8) for _ in range(3))
    t = np.full((4, 203), 0xA5, np.uint8)
    n, offs = np.full(4, 3, np.uint64), np.zeros(4, np.uint64)
    ab = np.full((12, 32), 0x01, np.uint8)
    prove_entry(C.c_uint32(0), ptr(lv), ptr(rv), ptr(ap), ptr(t), ptr(n), ptr(offs), ptr(ab),
                ptr(ab))
    assert all((x == 0xA5).all() for x in (lv, rv, ap, t))
    results = np.full(4, 7, np.int32)
    commits = np.zeros((4, 160), np.uint8)
    verify_entry.restype = C.c_uint32
    assert verify_entry(C.c_uint32(0), ptr(results), ptr(t), ptr(n), ptr(offs), ptr(ab), ptr(ab),
                        ptr(commits), ptr(lv), ptr(rv), ptr(ap)) == 0
    assert (results == 7).all() and (t == 0xA5).all()
    # the same proof repeated P times gives P identical proofs
    rng = np.random.default_rng(44)
    a, b = _scalars(rng, 13), _scalars(rng, 13)
    t0 = _transcripts(rng, 1)[0]
    tb = np.stack([t0] * 5)
    got = engine.prove_inner_products(tb, [a] * 5, [b] * 5, [2] * 5)
    t1 = t0.copy()
    want = engine.prove_inner_product(t1, a, b, 2)
    assert _same_proofs(got, [want] * 5)
    assert all(np.array_equal(row, t1) for row in tb)


# ---- CPU, through the emulation ---------------------------------------------------------------------
# (the `emul` fixture builds the harness library; tests/emul/ipa_batch.py adds the batched entries)

def test_emulated_batch_matches_reference_fixture(emul):
    check_fixture_as_one_batch(ipa_batch.Engine())


def test_emulated_mixed_batch_matches_single_calls(emul, port):
    check_mixed_batch(ipa_batch.Engine(), *mixed_batch(3), other=port)


def test_emulated_batch_reads_precomputed_generators_in_place(emul, port):
    """Every proof inside the precomputed range: round 0 addresses the table directly."""
    with emul.options(num_builtin=64):
        check_mixed_batch(ipa_batch.Engine(64),
                          *mixed_batch(4, ns=IN_TABLE_N, offsets=IN_TABLE_OFFSETS), other=port)


def test_emulated_batch_verify_flags_exactly_the_tampered_proofs(emul):
    check_tampered_verify(ipa_batch.Engine())


def test_emulated_empty_batch_and_repeated_proof(emul):
    engine = ipa_batch.Engine()
    check_empty_and_repeated(engine, engine.prove_entry, engine.verify_entry)


# ---- GPU ---------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_gpu_batch_matches_reference_fixture(bb, refcpu):
    check_fixture_as_one_batch(bb)
    z, off, cases = _fixture()
    t0 = np.stack([z[f"t0_{c}"] for c in cases])
    a_list, b_list = [z[f"a{c}"] for c in cases], [z[f"b{c}"] for c in cases]
    check_mixed_batch(bb, t0, a_list, b_list, [off] * len(cases))
    if refcpu.live:  # the reference's own prover, when oracle/_ref is built
        check_mixed_batch(bb, *mixed_batch(8, ns=(3, 8, 21), offsets=(2,)), other=refcpu)


@pytest.mark.gpu
def test_gpu_mixed_batch_matches_single_calls(bb, port):
    check_mixed_batch(bb, *mixed_batch(3), other=port)


@pytest.mark.gpu
def test_gpu_batch_reads_precomputed_generators_in_place(bb, port):
    check_mixed_batch(bb, *mixed_batch(4, ns=IN_TABLE_N, offsets=IN_TABLE_OFFSETS), other=port)


@pytest.mark.gpu
def test_gpu_batch_verify_flags_exactly_the_tampered_proofs(bb):
    check_tampered_verify(bb)


@pytest.mark.gpu
def test_gpu_empty_batch_and_repeated_proof(bb):
    check_empty_and_repeated(bb, bb.lib().b200_curve25519_prove_inner_products,
                             bb.lib().b200_curve25519_verify_inner_products)


@pytest.mark.gpu
def test_gpu_larger_mixed_batch_proves_and_verifies(bb):
    """16 proofs with n between 2^8 and 2^12: byte-identical to the single calls, and the batched
    verifier accepts them all and rejects one with a wrong product."""
    rng = np.random.default_rng(16)
    ns = [int(v) for v in rng.integers(2**8, 2**12 + 1, 16)]
    ns[0], ns[1] = 2**8, 2**12
    av = [[int.from_bytes(rng.bytes(32), "little") % L for _ in range(n)] for n in ns]
    bv = [[int.from_bytes(rng.bytes(32), "little") % L for _ in range(n)] for n in ns]
    enc = lambda vs: np.array([list(x.to_bytes(32, "little")) for x in vs], np.uint8).reshape(-1, 32)
    a_list, b_list = [enc(v) for v in av], [enc(v) for v in bv]
    offs = [int(o) for o in rng.integers(0, 100, 16)]
    t0 = _transcripts(rng, 16)
    proofs = check_mixed_batch(bb, t0, a_list, b_list, offs)
    products = np.stack([enc([sum(x * y for x, y in zip(a, b)) % L])[0] for a, b in zip(av, bv)])
    commits = []
    for a, o in zip(a_list, offs):
        h = bb.MultiexpHandle(0, bb.get_generators(a.shape[0], o))
        commits.append(h.fixed_multiexponentiation(32, 1, a.shape[0], a)[0])
        h.free()
    products[7][3] ^= 4
    t = t0.copy()
    res = bb.verify_inner_products(t, b_list, products, np.stack(commits), [p[0] for p in proofs],
                                   [p[1] for p in proofs], np.stack([p[2] for p in proofs]), offs)
    assert res.tolist() == [1] * 7 + [0] + [1] * 8
    for p in (0, 7):
        ts = t0[p].copy()
        assert bb.verify_inner_product(ts, b_list[p], products[p], commits[p], proofs[p][0],
                                       proofs[p][1], proofs[p][2], offs[p]) == res[p]
        assert np.array_equal(ts, t[p])


@pytest.mark.gpu
def test_gpu_batch_runs_rounds_together_not_one_proof_after_another(bb):
    """16 proofs of equal n issue fewer than twice the launches of one: the rounds are batched."""
    rng = np.random.default_rng(17)
    n = 2**10
    a_list = [_scalars(rng, n) for _ in range(16)]
    b_list = [_scalars(rng, n) for _ in range(16)]
    t = _transcripts(rng, 16)

    def launches(count):
        before = bb.launch_count()
        bb.prove_inner_products(t[:count].copy(), a_list[:count], b_list[:count], [0] * count)
        return bb.launch_count() - before

    launches(16)  # first use of every kernel and pool allocation
    one, sixteen = launches(1), launches(16)
    assert 0 < sixteen < 2 * one, (one, sixteen)
