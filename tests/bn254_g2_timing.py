"""Device time of bn254 G2 MSMs (curve 5) next to bn254 G1 ones (curve 2), in one process on one card:
  - variable-base, device-resident (b200_commit_device): one 32-byte column over n distinct synthetic
    generators, n in {2^16, 2^18, 2^20};
  - fixed-base (b200_fixed_msm_device): one 32-byte output over a handle of 2^20 synthetic
    generators, G2 and G1.
CUDA events around each call: two warm-up calls per shape, then the median and range of 5. An Fp2
multiplication is three Fp ones, so G2 should cost roughly 3x G1 per term, plus the Fp2 product by 3b'
in the projective formulas; the ratio is printed. The G2 results are checked against the closed form.
Prints the card's name and power limit first.
    python tests/bn254_g2_timing.py"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import blitzar_b200 as bb  # noqa: E402
from tests import common  # noqa: E402
from tests.bn254_g2_reference import BN  # noqa: E402
from tests.g2_timing import card, timed  # noqa: E402

G1, G2 = 2, 5


def cell(t):
    return f"{t[0]:.2f} ({t[1]:.2f}-{t[2]:.2f})"


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
        for curve in (G1, G2):
            dg = bb.DeviceBuffer(n * bb.CURVE_SIZES[curve][1])
            bb.synthetic_generators_device(curve, dg.ptr, n)
            out = bb.DeviceBuffer(bb.CURVE_SIZES[curve][2])
            row[curve] = timed(lambda: bb.commit_device(curve, [(n, 32, 0)], [ds.ptr], dg.ptr, out.ptr))
            if curve == G2:
                want = BN.commitment(BN.scalar_mul(
                    common.dot_mod(s, common.synth_scalars_k(n), BN.R_ORDER)))
                assert bytes(out.to_host()) == want, n
            dg.free()
            out.free()
        ds.free()
        print(f"| variable-base, device-resident | 2^{n.bit_length() - 1} | {cell(row[G1])} | "
              f"{cell(row[G2])} | {row[G2][0] / row[G1][0]:.2f} |", flush=True)

    n = 1 << 20
    s = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    ds = bb.DeviceBuffer(host=s)
    row = {}
    for curve in (G1, G2):
        gp = bb.DeviceBuffer(n * bb.CURVE_SIZES[curve][0])
        bb.synthetic_generators_device(curve, gp.ptr, n, projective=True)
        h = bb.MultiexpHandle(curve, device_ptr=gp.ptr, n=n)
        out = bb.DeviceBuffer(bb.CURVE_SIZES[curve][0])
        row[curve] = timed(lambda: bb.fixed_msm_device(h, out.ptr, None, 32, 1, n, ds.ptr))
        if curve == G2:
            want = BN.scalar_mul(common.dot_mod(s, common.synth_scalars_k(n), BN.R_ORDER))
            assert BN.from_proj_struct(out.to_host()) == want
        h.free()
        gp.free()
        out.free()
    ds.free()
    print(f"| fixed-base over a handle | 2^20 | {cell(row[G1])} | {cell(row[G2])} | "
          f"{row[G2][0] / row[G1][0]:.2f} |", flush=True)


if __name__ == "__main__":
    main()
