"""Times b200_multi_pairing_device on the GPU: single products of 1, 4, 2^10, 2^14 and 2^16 pairs and
4096 products of 4 pairs (CUDA events on the library stream, device-resident synthetic inputs), then,
in a torch.profiler run of its own, the per-launch device time of each pairing kernel, from which the
per-pair Miller-loop throughput and the final-exponentiation latency per product follow. With
--ptxas (no GPU needed) it compiles the two pairing units with -Xptxas -v and prints the registers,
stack frames and spills of every pairing kernel.

    python tests/pairing_timing.py [--out DIR] [--reps N]   # --out: also write pairing_timing.json there
    python tests/pairing_timing.py --ptxas"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = [("1 x 1", [1]), ("1 x 4", [4]), ("1 x 2^10", [1 << 10]), ("1 x 2^14", [1 << 14]),
          ("1 x 2^16", [1 << 16]), ("4096 x 4", [4] * 4096)]


def ptxas():
    from blitzar_b200 import build as b
    tmp = tempfile.mkdtemp()
    for unit in ("pairing_bls12381.cu", "pairing_bn254.cu"):
        out = subprocess.run([b.NVCC] + b.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(b.CSRC, unit),
                              "-o", os.path.join(tmp, "u.o")], capture_output=True, text=True, check=True)
        text = out.stdout + out.stderr
        for m in re.finditer(r"Compiling entry function '(\S+)'[^\n]*\n[^\n]*\n\s*(\d+) bytes stack frame, "
                             r"(\d+) bytes spill stores, (\d+) bytes spill loads\n[^\n]*Used (\d+) registers",
                             text):
            name = re.search(r"(Pairing\w+?Body|Fp12OpBody)\w*?(BlsTower|BnTower)", m.group(1))
            print(json.dumps({"kernel": name.group(1) + "<" + name.group(2) + ">", "registers": int(m.group(5)),
                              "stack_bytes": int(m.group(2)), "spill_stores": int(m.group(3)),
                              "spill_loads": int(m.group(4))}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ptxas", action="store_true")
    args = ap.parse_args()
    if args.ptxas:
        return ptxas()
    import numpy as np
    import torch
    import blitzar_b200 as bb
    from tests.pairing_reference import G2_CURVE, TOWERS
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu}))
    assert bb.sxt_init() == 0
    results = []
    for curve in (1, 2):
        t = TOWERS[curve]
        n_max = 1 << 16
        s1, s2 = bb.CURVE_SIZES[curve][0], bb.CURVE_SIZES[G2_CURVE[curve]][0]
        g1, g2 = bb.DeviceBuffer(n_max * s1), bb.DeviceBuffer(n_max * s2)
        bb.synthetic_generators_device(curve, g1.ptr, n_max, 0, True)
        bb.synthetic_generators_device(G2_CURVE[curve], g2.ptr, n_max, 1 << 20, True)
        out = bb.DeviceBuffer(4096 * t.GT_BYTES)
        start, stop = bb.Event(), bb.Event()
        for label, lengths in SHAPES:
            bb.multi_pairing_device(curve, out.ptr, lengths, g1.ptr, g2.ptr)  # warm-up
            ms = []
            for _ in range(args.reps):
                start.record()
                bb.multi_pairing_device(curve, out.ptr, lengths, g1.ptr, g2.ptr)
                stop.record()
                ms.append(start.elapsed_ms(stop))
            r = {"curve": curve, "shape": label, "pairs": sum(lengths), "ms_median": float(np.median(ms)),
                 "ms_min": min(ms)}
            print(json.dumps(r), flush=True)
            results.append(r)
        # per-kernel device times in a profiled run of its own: 2^16 pairs in one product, and 4096
        # products of 4
        from torch.profiler import ProfilerActivity, profile
        for label, lengths in (SHAPES[4], SHAPES[5]):
            bb.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                bb.multi_pairing_device(curve, out.ptr, lengths, g1.ptr, g2.ptr)
                bb.synchronize()
            kern = {}
            for e in prof.events():
                m = re.search(r"Pairing(\w+?)Body", e.name)
                if m and e.device_type.name == "CUDA":
                    kern[m.group(1)] = kern.get(m.group(1), 0.0) + e.device_time_total / 1000.0
            r = {"curve": curve, "profiled": label, "kernel_ms": kern,
                 "miller_pairs_per_s": sum(lengths) / (kern.get("Miller", float("nan")) / 1000.0),
                 "final_exp_ms": kern.get("FinalExp")}
            print(json.dumps(r), flush=True)
            results.append(r)
        for b in (g1, g2, out):
            b.free()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "pairing_timing.json"), "w") as f:
            json.dump({"gpu": gpu, "results": results}, f, indent=1)
    torch.cuda.synchronize()


if __name__ == "__main__":
    main()
