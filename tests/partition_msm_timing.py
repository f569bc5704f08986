"""Fixed-base MSMs over a handle with and without a partition table (partition_msm.cuh), ristretto255
and bn254, synthetic generators, the partition table at the reference's default width (w = 16):
  n in {2^10, 2^12, 2^14, 2^16}; 64, 256 and 1024 outputs; four width mixes (all 1-bit, the 1..64-bit
  mix of tests/many_columns.py, all 64-bit, all 256-bit); packed rows and vlen (output j spans
  n (j + 1) / m rows).
For every shape the same handle runs under BLITZAR_B200_PARTITION_POLICY=2 (the engine alone, as
without a table), 1 (every output from the table) and 0 (the cost model):
  - device time: CUDA events around b200_fixed_msm_device, one warm-up, then median and range of 3;
  - host time: the sxt_fixed_packed / _vlen call end to end (perf_counter, one call after the warm-up);
  - the table's attach time and size, once per (curve, n).
Shapes with n x (total bits) > 2^31 are skipped (seconds per call), and so is everything once the run
has taken 25 minutes; both are printed as "not measured". The results of the three policies are
compared on the host for every shape. Prints the card's name, power limit and SM clock first, then
one markdown row per shape; also writes the rows as JSON to out_dir.
    python tests/partition_msm_timing.py [out_dir]"""
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import blitzar_b200 as bb  # noqa: E402
from oracle import port  # noqa: E402

CURVES = {0: "ristretto255", 2: "bn254"}
MIXES = {"1-bit": [1], "1..64 mix": [1, 8, 16, 32, 64, 5, 12, 64], "64-bit": [64], "256-bit": [256]}
PROJ = {0: 160, 2: 96}
GEN_BYTES = {0: 128, 2: 64}  # a partition-table entry (device generator layout)
BUDGET_S = 25 * 60


def card():
    try:
        return subprocess.check_output(
            ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
             "--format=csv,noheader"], text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown card"


def measure(h, bt, lens, m, n, out, sc, psc, policy):
    os.environ["BLITZAR_B200_PARTITION_POLICY"] = str(policy)
    bb.fixed_msm_device(h, out.ptr, None, 0, m, n, sc.ptr, bit_table=bt, lengths=lens)
    bb.synchronize()
    times = []
    for _ in range(3):
        e0, e1 = bb.Event(), bb.Event()
        e0.record()
        bb.fixed_msm_device(h, out.ptr, None, 0, m, n, sc.ptr, bit_table=bt, lengths=lens)
        e1.record()
        times.append(e0.elapsed_ms(e1))
    res = out.to_host()
    t = time.perf_counter()
    if lens:
        h.fixed_vlen_multiexponentiation(bt, lens, psc)
    else:
        h.fixed_packed_multiexponentiation(bt, n, psc)
    host = (time.perf_counter() - t) * 1e3
    return statistics.median(times), min(times), max(times), host, res


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else "."
    os.makedirs(out_dir, exist_ok=True)
    assert bb.sxt_init() == 0
    port.build()
    start = time.perf_counter()
    print(f"card (name, power limit, max SM clock, SM clock): {card()}", flush=True)
    print("| curve | n | outputs | widths | layout | engine ms (range) | table ms (range) | "
          "model ms (range) | host engine / table / model ms |")
    print("|---|---|---|---|---|---|---|---|---|")
    rows = []
    rng = np.random.default_rng(1)
    for curve, name in CURVES.items():
        for n in (1 << 10, 1 << 12, 1 << 14, 1 << 16):
            gens = bb.synthetic_generators(curve, n, projective=True)
            h = bb.MultiexpHandle(curve, gens)
            t = time.perf_counter()
            w = h.add_partition_table(16)
            attach = (time.perf_counter() - t) * 1e3
            size = (-(-n // 16) << 16) * GEN_BYTES[curve]
            print(f"{name} n={n}: partition table w=16, {size / 2**30:.2f} GiB: "
                  + (f"attached in {attach:.1f} ms" if w else "does not fit (not attached)"),
                  flush=True)
            rows.append(dict(curve=name, n=n, attach_ms=attach if w else None, table_bytes=size))
            for m in (64, 256, 1024):
                for mix, pattern in MIXES.items():
                    bt = [pattern[j % len(pattern)] for j in range(m)]
                    for layout in ("packed", "vlen"):
                        label = f"| {name} | {n} | {m} | {mix} | {layout} |"
                        if not w or n * sum(bt) > 1 << 31 or time.perf_counter() - start > BUDGET_S:
                            print(f"{label} not measured | | | |", flush=True)
                            continue
                        lens = [max(1, n * (j + 1) // m) for j in range(m)] if layout == "vlen" else None
                        row_bytes = (sum(bt) + 7) // 8
                        psc = rng.integers(0, 256, (n, row_bytes), dtype=np.uint8)
                        sc = bb.DeviceBuffer(host=np.concatenate([psc.reshape(-1),
                                                                  np.zeros(64, np.uint8)]))
                        out = bb.DeviceBuffer(m * PROJ[curve])
                        r = {p: measure(h, bt, lens, m, n, out, sc, psc, p)
                             for p in (2, 1, 0)}
                        ref = port.normalize(curve, r[2][4].reshape(m, PROJ[curve]))
                        same = all(np.array_equal(port.normalize(curve, r[p][4].reshape(m, PROJ[curve])),
                                                  ref) for p in (0, 1))
                        sc.free()
                        out.free()
                        cells = " | ".join(f"{r[p][0]:.3f} ({r[p][1]:.3f}-{r[p][2]:.3f})"
                                           for p in (2, 1, 0))
                        print(f"{label} {cells} | {r[2][3]:.2f} / {r[1][3]:.2f} / {r[0][3]:.2f} |"
                              + ("" if same else " RESULTS DIFFER"), flush=True)
                        rows.append(dict(curve=name, n=n, outputs=m, widths=mix, layout=layout,
                                         engine=r[2][:4], table=r[1][:4], model=r[0][:4],
                                         same=bool(same)))
            h.free()
    os.environ.pop("BLITZAR_B200_PARTITION_POLICY", None)
    with open(os.path.join(out_dir, "partition_msm_timing.json"), "w") as f:
        json.dump(dict(card=card(), rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
