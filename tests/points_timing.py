"""Times b200_check_points_device and b200_decode_points_device per curve at n = 2^16, 2^20 and 2^22
(CUDA events on the library stream after a warm-up call, device-resident inputs), beside the time of a
device commitment over the same n (one column of 32-byte scalars, b200_commit_device). Prints one JSON
line per measurement, after the card's name and power limit. Inputs are synthetic generators: their
*_p2 structs for the check, and for decoding their affine structs (curves 2, 3, 5) or 4096 distinct
compressed commitments tiled to n (curves 1, 4).

    python tests/points_timing.py [--out DIR] [--reps N]   # --out: also write points_timing.json there"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = (1 << 16, 1 << 20, 1 << 22)


def timed(bb, fn, reps):
    fn()  # warm-up
    bb.synchronize()
    start, stop = bb.Event(), bb.Event()
    start.record()
    for _ in range(reps):
        fn()
    stop.record()
    return start.elapsed_ms(stop) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import blitzar_b200 as bb
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu}), flush=True)
    assert bb.sxt_init() == 0
    results = []
    for curve in (1, 2, 3, 4, 5):
        proj, stride, commit = bb.CURVE_SIZES[curve]
        compressed = curve in (1, 4)
        if compressed:
            m = 4096
            gens = bb.synthetic_generators(curve, m)
            ones = [(np.ones((1, 1), np.uint8), 0)] * m
            unique = bb.compute_pedersen_commitments_with_offsets(curve, ones, np.arange(m), gens)
        for n in SIZES:
            pts, affine = bb.DeviceBuffer(n * proj), bb.DeviceBuffer(n * stride)
            bb.synthetic_generators_device(curve, pts.ptr, n, 0, projective=True)
            bb.synthetic_generators_device(curve, affine.ptr, n, 0, projective=False)
            enc = bb.DeviceBuffer(host=np.tile(unique, (n // m, 1))) if compressed else affine
            valid, out = bb.DeviceBuffer(n), bb.DeviceBuffer(n * proj)
            scalars = bb.DeviceBuffer(host=np.random.default_rng(n).integers(0, 256, (n, 32), np.uint8))
            com = bb.DeviceBuffer(commit)
            t_check = timed(bb, lambda: bb.check_points_device(curve, valid.ptr, pts.ptr, n), args.reps)
            bb.check_points_device(curve, valid.ptr, pts.ptr, n)
            ok_check = int(valid.to_host().sum())
            t_decode = timed(bb, lambda: bb.decode_points_device(curve, out.ptr, valid.ptr, enc.ptr, n),
                             args.reps)
            ok_decode = int(valid.to_host().sum())
            t_commit = timed(bb, lambda: bb.commit_device(curve, [(n, 32, 0)], [scalars.ptr], affine.ptr,
                                                          com.ptr), args.reps)
            r = {"curve": curve, "n": n, "check_ms": round(t_check, 3),
                 "check_points_per_s": round(n / t_check * 1e3),
                 "decode_ms": round(t_decode, 3), "decode_points_per_s": round(n / t_decode * 1e3),
                 "commit_ms": round(t_commit, 3), "valid_check": ok_check, "valid_decode": ok_decode}
            assert ok_check == n and ok_decode == n, r
            print(json.dumps(r), flush=True)
            results.append(r)
            for b in {id(x): x for x in (pts, affine, enc, valid, out, scalars, com)}.values():
                b.free()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "points_timing.json"), "w") as f:
            json.dump({"gpu": gpu, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
