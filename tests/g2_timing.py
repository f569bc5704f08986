"""Device time of bls12-381 G2 MSMs next to G1 ones, in one process on one card:
  - variable-base, device-resident (b200_commit_device): one 32-byte column over n distinct synthetic
    generators, n in {2^16, 2^18, 2^20}, G2 (curve 4) and G1 (curve 1);
  - fixed-base (b200_fixed_msm_device): one 32-byte output over a G2 handle of 2^20 synthetic
    generators, and the same over a G1 handle for comparison.
CUDA events around each call: two warm-up calls per shape, then the median and range of 5. An Fp2
multiplication is three Fp ones, so G2 should cost roughly 3x G1 per term; the ratio is printed. The
G2 results are checked against the closed form. Prints the card's name and power limit first.
    python tests/g2_timing.py"""
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import blitzar_b200 as bb  # noqa: E402
from tests import common  # noqa: E402
from tests import g2_reference as g2  # noqa: E402

NAMES = {1: "G1", 4: "G2"}
REPS = 5


def card():
    try:
        return subprocess.check_output(
            ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
            text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown card"


def timed(fn):
    fn()
    fn()
    bb.synchronize()
    times = []
    for _ in range(REPS):
        e0, e1 = bb.Event(), bb.Event()
        e0.record()
        fn()
        e1.record()
        times.append(e0.elapsed_ms(e1))
    return statistics.median(times), min(times), max(times)


def main():
    assert bb.sxt_init() == 0
    print(f"card (name, power limit, max SM clock): {card()}", flush=True)
    rng = np.random.default_rng(16)
    print("| call | n | G1 ms (range) | G2 ms (range) | G2 / G1 |")
    print("|---|---|---|---|---|")
    for n in (1 << 16, 1 << 18, 1 << 20):
        s = rng.integers(0, 256, (n, 32), dtype=np.uint8)
        ds = bb.DeviceBuffer(host=s)
        row = {}
        for curve in (1, 4):
            dg = bb.DeviceBuffer(n * bb.CURVE_SIZES[curve][1])
            bb.synthetic_generators_device(curve, dg.ptr, n)
            out = bb.DeviceBuffer(bb.CURVE_SIZES[curve][2])
            row[curve] = timed(lambda: bb.commit_device(curve, [(n, 32, 0)], [ds.ptr], dg.ptr, out.ptr))
            if curve == 4:
                want = g2.compress(g2.scalar_mul(common.dot_mod(s, common.synth_scalars_k(n), g2.R_ORDER)))
                assert bytes(out.to_host()) == want, n
            dg.free()
            out.free()
        ds.free()
        print(f"| variable-base, device-resident | 2^{n.bit_length() - 1} | "
              f"{row[1][0]:.2f} ({row[1][1]:.2f}-{row[1][2]:.2f}) | "
              f"{row[4][0]:.2f} ({row[4][1]:.2f}-{row[4][2]:.2f}) | {row[4][0] / row[1][0]:.2f} |",
              flush=True)

    n = 1 << 20
    s = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    ds = bb.DeviceBuffer(host=s)
    row = {}
    for curve in (1, 4):
        gp = bb.DeviceBuffer(n * bb.CURVE_SIZES[curve][0])
        bb.synthetic_generators_device(curve, gp.ptr, n, projective=True)
        h = bb.MultiexpHandle(curve, device_ptr=gp.ptr, n=n)
        out = bb.DeviceBuffer(bb.CURVE_SIZES[curve][0])
        row[curve] = timed(lambda: bb.fixed_msm_device(h, out.ptr, None, 32, 1, n, ds.ptr))
        if curve == 4:
            want = g2.scalar_mul(common.dot_mod(s, common.synth_scalars_k(n), g2.R_ORDER))
            assert g2.from_proj_struct(out.to_host()) == want
        h.free()
        gp.free()
        out.free()
    ds.free()
    print(f"| fixed-base over a handle | 2^20 | {row[1][0]:.2f} ({row[1][1]:.2f}-{row[1][2]:.2f}) | "
          f"{row[4][0]:.2f} ({row[4][1]:.2f}-{row[4][2]:.2f}) | {row[4][0] / row[1][0]:.2f} |", flush=True)


if __name__ == "__main__":
    main()
