"""Batch-affine bucket accumulation of the short Weierstrass curves (blitzar_b200/csrc/batch_affine.cuh)
on the device, against the C oracle port and, at full size, the closed form of tests/common.py.

The CPU emulation (tests/test_emul.py) checks the same inputs' logic; what only the device shows is
kept here: the two halves of every pair level running concurrently on two streams, the atomic
scatter deciding which entries of a bucket meet at level 0, the PTX field arithmetic, and the
automatic level count at the sizes where it turns on. Calls whose level count is asserted run in a
fresh process, because the library reads BLITZAR_LOG_LEVEL once per process."""
import os
import re
import sys

import numpy as np
import pytest

from tests import common

pytestmark = pytest.mark.gpu
CURVES = [1, 2, 3]


def case(label):
    """Marks the start of a labelled case in the child's stderr (_run_logged)."""
    sys.stderr.write("@case %s\n" % label)
    sys.stderr.flush()


def _run_logged(body, curve):
    """Runs body(bb, port, curve) in a fresh process with BLITZAR_LOG_LEVEL=debug and returns, per
    case label, the pair level counts of every generator range the calls accumulated."""
    r = common.run_fresh((body, curve), env={"BLITZAR_LOG_LEVEL": "debug"})
    levels, label = {}, None
    for line in r.stderr.splitlines():
        if line.startswith("@case "):
            label = line[len("@case "):]
            levels[label] = []
        m = re.search(r"pair levels (\d+)", line)
        if m and label is not None:
            levels[label].append(int(m.group(1)))
    return levels


# ---- (a) forced level counts and pairs per thread --------------------------------------------------
def _fresh_forced_levels(bb, port, curve):
    rng = np.random.default_rng(60 + curve)
    n = 3000
    gens, _ = common.generators_for(port, curve, n)
    gens[1::7] = gens[0]
    cols = common.random_columns(rng, n, [(0, 32, 0), (-13, 16, 1), (0, 8, 1), (-1, 5, 0), (-2999, 32, 0),
                                          (-1000, 2, 0), (0, 1, 0)])
    sg = np.zeros((n, 1), dtype=np.uint8)
    sg[::2], sg[1::2] = 1, 0xFF  # +1 / -1 alternating: P + (-P) on the duplicated generators
    cols.append((sg, 1))
    want = port.commit(curve, cols, gens)
    tiny = common.random_columns(rng, 3, [(0, 32, 0), (0, 1, 1), (-1, 2, 0)])
    tiny_gens = gens[:3].copy()
    tiny_gens[1] = tiny_gens[0]
    want_tiny = port.commit(curve, tiny, tiny_gens)
    # (window bits (0 = automatic), levels, pairs per thread (0 = default), extra environment)
    cases = [(4, 1, 4, {}), (4, 3, 5, {}), (6, 2, 32, {}), (3, 5, 0, {}), (2, 6, 64, {}), (0, 6, 1, {}),
             (4, 2, 8, {"BLITZAR_B200_RANGES": "3"}),  # later pieces: scratch buckets + merge
             (5, 3, 16, {"BLITZAR_B200_GROUP_ENTRIES": "20000"})]  # several column groups
    for c, levels, batch, extra in cases:
        os.environ.update(BLITZAR_B200_PAIR_LEVELS=str(levels), BLITZAR_B200_PAIR_BATCH=str(batch), **extra)
        bb.set_tuning(window_bits=c)
        case("%d c=%d batch=%d %s" % (levels, c, batch, sorted(extra)))
        got = bb.compute_pedersen_commitments(curve, cols, gens)
        assert common.same(curve, got, want), (c, levels, batch, extra)
        for k in extra:
            del os.environ[k]
    bb.set_tuning()
    os.environ.update(BLITZAR_B200_PAIR_LEVELS="6", BLITZAR_B200_PAIR_BATCH="0")
    case("6 tiny")  # one thread: the first half of the level is empty
    assert common.same(curve, bb.compute_pedersen_commitments(curve, tiny, tiny_gens), want_tiny)


@pytest.mark.parametrize("curve", CURVES)
def test_forced_pair_levels(curve):
    """The emulator's sweep of window widths x levels x pairs per thread on the device, plus upload
    pieces, column groups and a single-thread call; every range ran with the forced level count."""
    levels = _run_logged(_fresh_forced_levels, curve)
    assert len(levels) == 9, levels
    for label, used in levels.items():
        want = int(label.split()[0])
        assert used and all(v == want for v in used), (label, used)


# ---- (b) degenerate buckets ------------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES)
def test_degenerate_buckets(bb, port, curve, monkeypatch):
    """Buckets holding only copies of +-P, identities or (bls12-381) the x = 0 points (0, +-2), at
    every level count: doublings, cancellations and identity operands, with the atomic scatter
    choosing which entries meet."""
    gens, cols, equal = common.degenerate_buckets(port, curve)
    want = port.commit(curve, cols, gens)
    for j, m in equal:
        assert common.same(curve, want[j:j + 1],
                           port.commit(curve, [(np.array([[m]], dtype=np.uint8), 0)], gens[:1])), m
    monkeypatch.delenv("BLITZAR_B200_PAIR_LEVELS", raising=False)
    assert common.same(curve, bb.compute_pedersen_commitments(curve, cols, gens), want)
    for levels in range(1, 7):
        monkeypatch.setenv("BLITZAR_B200_PAIR_LEVELS", str(levels))
        assert common.same(curve, bb.compute_pedersen_commitments(curve, cols, gens), want), levels


# ---- (c) identity generators -----------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES)
@pytest.mark.parametrize("levels", [None, 1, 3, 6])
def test_identity_generators(bb, port, curve, levels, monkeypatch):
    """Affine generators flagged `infinity` next to real points in the pair levels, and handles whose
    projective generators have Z = 0 with the table forced on, forced off and under the cost model."""
    if levels is None:
        monkeypatch.delenv("BLITZAR_B200_PAIR_LEVELS", raising=False)
    else:
        monkeypatch.setenv("BLITZAR_B200_PAIR_LEVELS", str(levels))
    rng = np.random.default_rng(80 + curve)
    n = 2000
    gens, gens_p = common.generators_for(port, curve, n)
    gens, gens_p = gens.copy(), gens_p.copy()
    ident = [0, 7, 19, n - 1] + list(range(100, n, 13))
    common.set_identity(curve, gens, ident)
    cols = common.random_columns(rng, n, [(0, 32, 0), (0, 2, 0), (-7, 16, 1)])
    cols.append((np.ones((n, 1), dtype=np.uint8), 0))
    assert common.same(curve, bb.compute_pedersen_commitments(curve, cols, gens),
                       port.commit(curve, cols, gens))
    common.set_identity(curve, gens_p, ident)
    sc = rng.integers(0, 256, (n, 2, 32), dtype=np.uint8)
    sc[:, 1] = 0
    sc[:, 1, 0] = 1
    sc = sc.reshape(n, 64)
    want = port.normalize(curve, port.fixed_msm(curve, gens_p, 2, n, sc, element_num_bytes=32))
    h = bb.MultiexpHandle(curve, gens_p)
    try:
        for policy in ("1", "2", "0"):
            monkeypatch.setenv("BLITZAR_B200_TABLE_POLICY", policy)
            got = h.fixed_multiexponentiation(32, 2, n, sc)
            assert common.same(curve, port.normalize(curve, got), want), policy
    finally:
        h.free()


# ---- (d) cross-window collisions in table mode -----------------------------------------------------
@pytest.mark.parametrize("curve", [0, 1, 2, 3])
@pytest.mark.parametrize("window_bits", [10, 16])
def test_table_cross_window_collisions(bb, port, curve, window_bits, monkeypatch):
    """G_j = +-2^c G_i: window 1 of i and window 0 of j share a bucket of the table's one bucket set
    (ristretto255, with complete formulas and no pair levels, is the control)."""
    gens_p, sc = common.cross_window_handle(port, curve, window_bits)
    m = gens_p.shape[0]
    want = port.normalize(curve, port.fixed_msm(curve, gens_p, 2, m, sc, element_num_bytes=32))
    monkeypatch.setenv("BLITZAR_B200_TABLE_WINDOW", str(window_bits))
    monkeypatch.setenv("BLITZAR_B200_TABLE_POLICY", "1")
    h = bb.MultiexpHandle(curve, gens_p)
    try:
        for levels in (None, 1, 2, 3):
            if levels is None:
                monkeypatch.delenv("BLITZAR_B200_PAIR_LEVELS", raising=False)
            else:
                monkeypatch.setenv("BLITZAR_B200_PAIR_LEVELS", str(levels))
            got = h.fixed_multiexponentiation(32, 2, m, sc)
            assert common.same(curve, port.normalize(curve, got), want), levels
    finally:
        h.free()


# ---- (e) full size, automatic level count ----------------------------------------------------------
def _fresh_full_size(bb, port, curve):
    n = 1 << 20
    gens = bb.synthetic_generators(curve, n, 0, projective=False)
    ed = common.GeneratorEdits(curve, gens)
    rng = np.random.default_rng(70 + curve)
    s = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    rows = np.arange(16, n, 16)
    ed.duplicate(rows, rows - 1)  # equal points with equal scalars: doublings
    s[rows] = s[rows - 1]
    ed.duplicate(rows[:-1] + 1, rows[:-1])  # and their negations: cancellations
    ed.negate(rows[:-1] + 1)
    s[rows[:-1] + 1] = s[rows[:-1]]
    block = slice(1 << 19, (1 << 19) + 4096)  # 4096 copies of one point, scalar 1: one loaded bucket
    ed.duplicate(block, 1 << 19)
    s[block] = 0
    s[block, 0] = 1
    ed.identity(slice(5, n, 3001))
    want = common.closed_form_commitment(port, curve, s, k=ed.k)
    dg = bb.DeviceBuffer(host=gens)
    ds = bb.DeviceBuffer(host=s)
    out = bb.DeviceBuffer(bb.CURVE_SIZES[curve][2])
    case("full")
    bb.commit_device(curve, [(n, 32, 0)], [ds.ptr], dg.ptr, out.ptr)  # one generator range
    got = out.to_host()[None]
    assert common.same(curve, got, want)
    for b in (dg, ds, out):
        b.free()


@pytest.mark.parametrize("curve", CURVES)
def test_full_size_automatic_pair_levels(curve):
    """n = 2^20 synthetic generators with duplicated, negated, identity rows and one bucket of 4096
    equal points, device-resident in one generator range: the automatic level count turns on, and
    the commitment equals the closed form over the edited discrete logs."""
    levels = _run_logged(_fresh_full_size, curve)
    print(f"curve {curve}: pair levels {levels['full']}")
    assert levels["full"] and min(levels["full"]) >= 1, levels
