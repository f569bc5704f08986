"""Many columns at their own generator offsets: k calls of the existing entry point, one per offset
(a), against one call of b200_compute_pedersen_commitments_with_offsets (b).
  - k in {16, 64, 256} columns of n in {2^12, 2^14, 2^16} rows of 32-byte scalars (top nibble
    cleared), at k distinct offsets drawn from [0, 4n);
  - ristretto255 with the built-in generators (sxt_curve25519_compute_pedersen_commitments with
    offset_generators) and bn254 with explicit generators (the *_with_generators call on the slice
    that starts at the offset);
  - scalars and generators in pinned host memory; a host clock around each call, which synchronises;
  - one warm-up of both per shape, then `reps` rounds alternating (a) and (b); medians in ms;
  - (a) and (b) must give the same bytes.
Prints the card's name and power limit first, then one line per shape.
    python tests/offsets_timing.py [reps]"""
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import blitzar_b200 as bb  # noqa: E402

CURVES = {0: "ristretto255 built-in", 2: "bn254 explicit"}


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit",
                                        "--format=csv,noheader"], text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown card"


def pinned(shape):
    return torch.empty(shape, dtype=torch.uint8, pin_memory=True).numpy()


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    assert bb.sxt_init() == 0
    print(f"card: {card()}", flush=True)
    rng = np.random.default_rng(1)
    for curve, name in CURVES.items():
        for n in (1 << 12, 1 << 14, 1 << 16):
            gens = None
            if curve:
                gens = pinned((5 * n, bb.CURVE_SIZES[curve][1]))
                gens[:] = bb.synthetic_generators(curve, 5 * n)
            for k in (16, 64, 256):
                s = pinned((k, n, 32))
                s[:] = rng.integers(0, 256, (k, n, 32), dtype=np.uint8)
                s[:, :, 31] &= 0x0F
                cols = [(s[j], 0) for j in range(k)]
                offsets = [int(v) for v in rng.choice(4 * n, k, replace=False)]

                def separate():
                    if curve == 0:
                        return np.concatenate([bb.compute_pedersen_commitments(0, [c], None, o)
                                               for c, o in zip(cols, offsets)])
                    return np.concatenate([bb.compute_pedersen_commitments(curve, [c], gens[o:])
                                           for c, o in zip(cols, offsets)])

                def one_pass():
                    return bb.compute_pedersen_commitments_with_offsets(curve, cols, offsets, gens)

                a, b = separate(), one_pass()  # warm-up
                assert np.array_equal(a, b), (name, n, k)
                ta, tb = [], []
                for _ in range(reps):
                    for fn, times in ((separate, ta), (one_pass, tb)):
                        t = time.perf_counter()
                        out = fn()
                        times.append((time.perf_counter() - t) * 1e3)
                        assert np.array_equal(out, a), (name, n, k)
                ma, mb = float(np.median(ta)), float(np.median(tb))
                print(f"{name} k={k} n=2^{n.bit_length() - 1}: (a) {k} calls {ma:.2f} ms "
                      f"[{min(ta):.2f}-{max(ta):.2f}], (b) one call {mb:.2f} ms "
                      f"[{min(tb):.2f}-{max(tb):.2f}], (a)/(b) {ma / mb:.2f}x", flush=True)
                del s, cols


if __name__ == "__main__":
    main()
