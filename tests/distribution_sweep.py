"""Value-distribution sensitivity of the variable-base MSM (SURVEY §8d): the bucket load depends on the
scalars. Device-resident ristretto MSM, n = 2^20, for uniform 252-bit scalars, all-ones scalars (every
digit lands in ONE bucket per window), tiny scalars (one non-zero window), a boolean column and a column
that is 99 % zeros. Run on a GPU: python tests/distribution_sweep.py [log2 n]"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import blitzar_b200 as bb  # noqa: E402

logn = int(sys.argv[1]) if len(sys.argv) > 1 else 20
n = 1 << logn
bb.sxt_init()
rng = np.random.default_rng(0)
gens = bb.get_generators(n, 0)
dg = bb.DeviceBuffer(host=gens)
do = bb.DeviceBuffer(64)


def column(kind):
    if kind == "uniform 252-bit":
        s = rng.integers(0, 256, (n, 32), dtype=np.uint8)
        s[:, 31] &= 0x0f
        return s
    if kind == "all-ones (2^252 - 1)":
        s = np.full((n, 32), 0xFF, dtype=np.uint8)
        s[:, 31] = 0x0f
        return s
    if kind == "tiny (< 2^8, 1-byte column)":
        return rng.integers(0, 256, (n, 1), dtype=np.uint8)
    if kind == "boolean (1-byte column of 0/1)":
        return rng.integers(0, 2, (n, 1), dtype=np.uint8)
    if kind == "99% zeros, 32-byte":
        s = np.zeros((n, 32), dtype=np.uint8)
        idx = rng.choice(n, n // 100, replace=False)
        s[idx] = rng.integers(0, 256, (len(idx), 32), dtype=np.uint8)
        s[:, 31] &= 0x0f
        return s
    raise ValueError(kind)


for kind in ("uniform 252-bit", "all-ones (2^252 - 1)", "tiny (< 2^8, 1-byte column)",
             "boolean (1-byte column of 0/1)", "99% zeros, 32-byte"):
    s = column(kind)
    ds = bb.DeviceBuffer(host=s)
    best = 1e9
    for _ in range(4):
        e0, e1 = bb.Event(), bb.Event()
        e0.record()
        bb.commit_device(0, [(n, s.shape[1], 0)], [ds.ptr], dg.ptr, do.ptr)
        e1.record()
        best = min(best, e0.elapsed_ms(e1))
    print(f"n=2^{logn} {kind:34s}: {best:7.3f} ms  {n / best * 1e3:.3e} terms/s", flush=True)
    ds.free()
