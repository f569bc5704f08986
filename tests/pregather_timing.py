#!/usr/bin/env python3
"""Time from the first kernel of a C2 call to the start of its gathering level.

    python tests/pregather_timing.py [--calls 5] [--warmup 5] [--out DIR]

C2 as bench.py builds it (ristretto255, n = 2^20, synthetic generators in HBM, make_scalars with seed
12345 and top-byte mask 0x0F, b200_commit_device). Each of `--calls` calls is traced on its own under
torch.profiler (CUDA activity only), the calls 20 ms apart. For every call the script takes the start of its first kernel and
the start of the gathering level (the first `AccumulateBody<Ed25519, true, ...>` launch), and the time
of every sort and normalisation kernel; it prints the median over the calls. The bytes this phase must
move are computed from n, the window width c and the layouts (not measured), and divided by the
median phase time. The card name and power limit are read in the same run and written with the
table to DIR/pregather.json.
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import make_scalars  # noqa: E402
from tests.kernel_breakdown import body_name, card  # noqa: E402

PHASE_BODIES = ("MicroCountBody", "PlanBinsBody", "CoarseScatterBody", "BinSortBody",
                "NormalizeUpBlockBody", "NormalizeMidBody", "NormalizeDownBody", "FillIdentityBody")


def phase_bytes(n, c, windows, scalar_bytes=32):
    """Bytes the path ahead of the gathering level moves at least once, from the layouts: M = n x
    (windows - 1) 8-byte sort entries (the top window of a 252-bit scalar holds only carries),
    2^(c-1) buckets per window, 160-byte ABI generators of which the up
    pass reads the two 32-byte sectors holding Z, 32-byte prefix products, 128-byte device generators."""
    m = n * (windows - 1)
    nkeys = windows << (c - 1)
    rows = [
        ("scalars, read", n * scalar_bytes),
        ("tmp, written and read", 2 * 8 * m),
        ("sorted entries, written", 8 * m),
        ("bucket offsets, written", 4 * nkeys),
        ("ABI generators: read, and the Z sectors of the up pass", 160 * n + 64 * n),
        ("prefix products, written and read", 2 * 32 * n),
        ("device generators, written", 128 * n),
    ]
    return rows, sum(b for _, b in rows)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--c", type=int, default=16, help="window width the engine picks at n = 2^20")
    ap.add_argument("--windows", type=int, default=17, help="digit windows of a 32-byte scalar at c")
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "pregather_timing"))
    args = ap.parse_args()

    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    import blitzar_b200 as bb

    n = 1 << 20
    torch.cuda.set_device(0)
    assert bb.sxt_init(device=0) == 0
    gens = torch.empty((n, bb.CURVE_SIZES[0][1]), dtype=torch.uint8, device="cuda")
    bb.synthetic_generators_device(0, gens.data_ptr(), n, 0, projective=False)
    scal = torch.from_numpy(make_scalars(n, 12345, 0x0F)).cuda()
    out = torch.zeros((72 + 64,), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def call():
        bb.commit_device(0, [(n, 32, 0)], [scal.data_ptr()], gens.data_ptr(), out.data_ptr())

    for _ in range(args.warmup):
        call()
    bb.synchronize()

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.calls):
            call()
            bb.synchronize()
            time.sleep(0.02)
        torch.cuda.synchronize()
    kernels = sorted((ev for ev in prof.events() if ev.device_type == DeviceType.CUDA
                      and ("k_run<" in ev.name or "k_block<" in ev.name)),
                     key=lambda ev: ev.time_range.start)
    calls, end = [], None  # a new call starts after a gap of more than 10 ms
    for ev in kernels:
        if end is None or ev.time_range.start - end > 1e4:
            calls.append([])
        calls[-1].append(ev)
        end = ev.time_range.end if end is None else max(end, ev.time_range.end)
    starts, kernel_us = [], {}
    for evs in calls:
        first = evs[0].time_range.start
        gather = min(ev.time_range.start for ev in evs
                     if body_name(ev.name).startswith("AccumulateBody<Ed25519, true"))
        starts.append(gather - first)
        per_call = {}
        for ev in evs:
            b = body_name(ev.name).split("<")[0]
            if b in PHASE_BODIES:
                per_call[b] = per_call.get(b, 0.0) + (ev.time_range.end - ev.time_range.start)
        for b, us in per_call.items():
            kernel_us.setdefault(b, []).append(us)

    start_us = statistics.median(starts)
    rows, total = phase_bytes(n, args.c, args.windows)
    result = {"card": card(), "n": n, "c": args.c, "windows": args.windows, "calls": args.calls,
              "gather_start_us": {"median": start_us, "min": min(starts), "max": max(starts)},
              "kernels_us": {b: statistics.median(v) for b, v in kernel_us.items()},
              "bytes": dict(rows), "bytes_total": total, "gb_per_s": total / start_us / 1e3}

    c = result["card"]
    print(f"C2 on {c.get('name')} at a {c.get('power_limit')} power limit, {len(calls)} calls traced")
    print(f"gathering level starts {start_us:.1f} us after the call's first kernel "
          f"(median; {min(starts):.1f}-{max(starts):.1f})")
    print(f"{'kernel':24s} {'us (median)':>12s}")
    for b in PHASE_BODIES:
        if b in result["kernels_us"]:
            print(f"{b:24s} {result['kernels_us'][b]:12.1f}")
    print("bytes of the phase (computed from the layouts):")
    for name, b in rows:
        print(f"  {name:58s} {b / 1e6:8.1f} MB")
    print(f"  {'total':58s} {total / 1e6:8.1f} MB -> {result['gb_per_s']:.0f} GB/s over the phase")
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "pregather.json"), "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
