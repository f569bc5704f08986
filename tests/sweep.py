"""Throughput sweep n = 2^16 .. 2^24 (BASELINE.md §4): device-resident time and end-to-end C-ABI time
per curve / API on one GPU, on the reference benchmarks' own generators (distinct points produced in
HBM by b200_synthetic_generators_device — no tiling). Prints a markdown table and, given a path,
writes the rows there as JSON.   python tests/sweep.py [out.json]   (SWEEP_MAX=22 to stop earlier)"""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import blitzar_b200 as bb  # noqa: E402

bb.sxt_init()
rng = np.random.default_rng(0)
rows = []
STRIDE = {0: 160, 1: 104, 2: 72, 3: 72}
PSTRIDE = {0: 160, 1: 144, 2: 96, 3: 96}


def timed(fn, iters=3):
    best = 1e9
    for _ in range(iters):
        e0, e1 = bb.Event(), bb.Event()
        e0.record()
        fn()
        e1.record()
        best = min(best, e0.elapsed_ms(e1))
    return best


def wall(fn, iters=3):
    best = 1e9
    for _ in range(iters):
        t = time.perf_counter()
        fn()
        best = min(best, time.perf_counter() - t)
    return best * 1e3


max_log = int(os.environ.get("SWEEP_MAX", "24"))
for logn in range(16, max_log + 1, 2):
    n = 1 << logn
    s = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    for curve, name, mask, bpt, cap in ((0, "ristretto255 var-base", 0x0F, 192, 24),
                                        (1, "bls12-381 var-base", 0x7F, 136, 22),
                                        (2, "bn254 var-base", 0x3F, 104, 24)):
        if logn > cap:
            continue
        sc = s.copy()
        sc[:, 31] &= mask
        dg = bb.DeviceBuffer(n * STRIDE[curve])
        bb.synthetic_generators_device(curve, dg.ptr, n, 0, False)
        gens = dg.to_host((n, STRIDE[curve]))
        ds, do = bb.DeviceBuffer(host=sc), bb.DeviceBuffer(128)
        ms = timed(lambda: bb.commit_device(curve, [(n, 32, 0)], [ds.ptr], dg.ptr, do.ptr))
        e2e = wall(lambda: bb.compute_pedersen_commitments(curve, [(sc, 0)], gens), iters=2)
        rows.append(dict(path=name, logn=logn, kernel_ms=ms, e2e_ms=e2e, bytes_per_term=bpt))
        for b in (dg, ds, do):
            b.free()
        del gens
    # bn254 fixed-base (handle resident, table built on the device; e2e = H2D scalars + MSM + D2H)
    sc = s.copy()
    sc[:, 31] &= 0x3F
    dg = bb.DeviceBuffer(n * PSTRIDE[2])
    bb.synthetic_generators_device(2, dg.ptr, n, 0, True)
    bb.synchronize()
    t = time.perf_counter()
    h = bb.MultiexpHandle(2, device_ptr=dg.ptr, n=n)
    bb.synchronize()
    t_handle = time.perf_counter() - t
    dg.free()
    ds, do = bb.DeviceBuffer(host=sc), bb.DeviceBuffer(128)
    ms = timed(lambda: bb.fixed_msm_device(h, do.ptr, None, 32, 1, n, ds.ptr))
    e2e = wall(lambda: h.fixed_multiexponentiation(32, 1, n, sc), iters=2)
    rows.append(dict(path="bn254 fixed-base (handle)", logn=logn, kernel_ms=ms, e2e_ms=e2e,
                     bytes_per_term=96, handle_s=t_handle))
    h.free()
    ds.free()
    do.free()
    print("done 2^%d" % logn, flush=True)

if len(sys.argv) > 1:
    json.dump(rows, open(sys.argv[1], "w"), indent=1)
print("| path | n | device ms | terms/s (device) | GB/s algorithmic | e2e ms (pageable host) | terms/s (e2e) |")
print("|---|---|---|---|---|---|---|")
for r in rows:
    n = 1 << r["logn"]
    k = r["kernel_ms"]
    extra = f" (handle_new {r['handle_s'] * 1e3:.0f} ms)" if "handle_s" in r else ""
    print(f"| {r['path']}{extra} | 2^{r['logn']} | {k:.3f} | {n / k * 1e3:.3e} | "
          f"{r['bytes_per_term'] * n / k / 1e6:.1f} | {r['e2e_ms']:.2f} | {n / r['e2e_ms'] * 1e3:.3e} |")
