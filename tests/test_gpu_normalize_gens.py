"""Normalising ingestion of ed25519 caller generators on the GPU: generators in scaled projective
representations (with duplicated, negated and identity generators) through the device call and the
host call with its upload pieces, at 2^16 and 2^20 terms, with BLITZAR_B200_NORMALIZE_GENS on and
off. Both must equal the commitments over the same points in their plain representation, also
when one generator has Z = 0 (and zero scalars)."""
import numpy as np
import pytest

from tests import common
from tests import normalize_emul as ne

pytestmark = pytest.mark.gpu
BLOCK = 4096  # distinct generators, tiled to n (Python big-integer scaling is slow)
SPECIAL = dict(identity=(5, 4000), negated=(9, 2048), duplicated=(10, 11, 2049))


def _device_call(bb, cols, gens):
    dg = bb.DeviceBuffer(host=gens)
    ds = [bb.DeviceBuffer(host=np.ascontiguousarray(c)) for c, _ in cols]
    out = bb.DeviceBuffer(32 * len(cols))
    bb.commit_device(0, [(c.shape[0], c.shape[1], s) for c, s in cols], [d.ptr for d in ds], dg.ptr,
                     out.ptr)
    got = out.to_host((len(cols), 32))
    for b in [dg, out] + ds:
        b.free()
    return got


@pytest.mark.parametrize("logn", [16, 20])
def test_scaled_generators(bb, port, logn, monkeypatch):
    n = 1 << logn
    base = port.ristretto_generators(BLOCK)
    reps = n // BLOCK
    gens = np.tile(ne.scaled_generators(base, logn, **SPECIAL), (reps, 1))
    plain = np.tile(ne.scaled_generators(base, 0, scale=False, **SPECIAL), (reps, 1))
    cols = common.random_columns(np.random.default_rng(logn), n,
                                 [(0, 32, 0), (-(n // 3), 16, 1), (0, 8, 0)])
    # A Z = 0 generator whose scalars are all 0: it never reaches a bucket, so the commitments stay
    # those of the valid generators, but its range must fall back to the unnormalised generators and
    # the 8-multiplication path (7 multiplications over generators with Z != 1 give other points).
    # With non-zero scalars the bytes of such an input depend on the order of the additions within
    # a bucket, which the sort does not fix: the emulation tests compare those on and off.
    bad_row = n - 100
    for c, _ in cols:
        if c.shape[0] > bad_row:
            c[bad_row] = 0
    bad = gens.copy()
    bad[bad_row] = ne.scaled_generators(gens[bad_row:bad_row + 1], 1, zero_z=(0,))[0]
    monkeypatch.setenv("BLITZAR_B200_NORMALIZE_GENS", "0")
    want = bb.compute_pedersen_commitments(0, cols, plain)
    if logn == 16:
        assert np.array_equal(want, port.commit(0, cols, plain))
    for norm in ("1", "0"):
        monkeypatch.setenv("BLITZAR_B200_NORMALIZE_GENS", norm)
        for ranges in ("1", "4"):  # upload pieces of the host call
            monkeypatch.setenv("BLITZAR_B200_RANGES", ranges)
            for g, label in ((gens, "scaled"), (bad, "Z = 0")):
                got = bb.compute_pedersen_commitments(0, cols, g)
                assert np.array_equal(got, want), (norm, ranges, label)
        monkeypatch.delenv("BLITZAR_B200_RANGES")
        for g, label in ((gens, "scaled"), (bad, "Z = 0")):
            assert np.array_equal(_device_call(bb, cols, g), want), (norm, label)
