#!/usr/bin/env python3
"""Device step time of C2 and of the C4 share with the normalising ingestion of caller generators on
and off (BLITZAR_B200_NORMALIZE_GENS, read on every call), alternating in one process.

    python tests/normalize_timing.py [--runs 5] [--steps 50] [--warmup 5] [--out DIR]

Inputs are built as bench.py builds them (synthetic generators in HBM, make_scalars with seed
12345 + 1000 j and mask 0x0F, b200_commit_device on the library stream). Every run times `steps`
steps with CUDA events after `warmup` untimed ones; the two paths alternate run by run, and the
median and range of each are printed. The commitments of both paths are compared byte for byte.
A last, separate run traces 5 C2 steps of each path with torch.profiler and reports where the
ingestion (IngestBody, or the normalisation's NormalizeUp/Down bodies and its inversion tree) ends
relative to the end of the bucket sort and to the start of the gathering level: the ingestion is
hidden under the sort when it ends before the sort does. Card name, power limit and SM clock go
with the numbers to DIR/normalize_timing.json.
"""
import argparse
import json
import os
import statistics
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import make_scalars  # noqa: E402
from tests.kernel_breakdown import SORT_BODIES, body_name, card  # noqa: E402

WORKLOADS = {"c2": 1, "c4_share": 8}  # columns of 2^20 ristretto255 terms
INGEST = ("IngestBody", "NormalizeUpBody", "NormalizeDownBody", "BatchUpBody", "BatchTopBody",
          "BatchDownBody")


def trace(bb, step, steps):
    """Per step (ms): end of the ingestion and start of the gathering level, both relative to the end
    of the sort."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step()
        bb.synchronize()
        torch.cuda.synchronize()
    kernels = []
    for ev in prof.events():
        if str(getattr(ev, "device_type", "")).endswith("CUDA"):
            kernels.append((ev.time_range.start, ev.time_range.end, body_name(ev.name)))
    kernels.sort()
    rows, sort_end, ingest_end = [], None, None
    for start, end, name in kernels:
        base = name.split("<")[0]
        if base in SORT_BODIES:
            sort_end = max(sort_end or end, end)
        elif base in INGEST:
            ingest_end = max(ingest_end or end, end)
        elif base == "AccumulateBody" and name.split(",")[1].strip() == "true" and sort_end:
            rows.append({"ingest_end_after_sort_end_us": (ingest_end - sort_end) if ingest_end else None,
                         "gather_start_after_sort_end_us": start - sort_end})
            sort_end = ingest_end = None
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "normalize_timing"))
    args = ap.parse_args()

    import numpy as np
    import torch
    import blitzar_b200 as bb

    n = 1 << 20
    torch.cuda.set_device(0)
    assert bb.sxt_init(device=0) == 0
    gens = torch.empty((n, 160), dtype=torch.uint8, device="cuda")
    bb.synthetic_generators_device(0, gens.data_ptr(), n, 0, projective=False)
    result = {"card": card(), "runs": args.runs, "steps": args.steps, "warmup": args.warmup,
              "workloads": {}}
    c = result["card"]
    print(f"{c.get('name')}, power limit {c.get('power_limit')}, max SM clock {c.get('sm_max_clock')}")
    for name, ncol in WORKLOADS.items():
        scal = [torch.from_numpy(make_scalars(n, 12345 + 1000 * j, 0x0F)).cuda() for j in range(ncol)]
        out = torch.zeros((ncol * 32,), dtype=torch.uint8, device="cuda")
        shapes, ptrs = [(n, 32, 0)] * ncol, [s.data_ptr() for s in scal]

        def step():
            bb.commit_device(0, shapes, ptrs, gens.data_ptr(), out.data_ptr())

        times = {"1": [], "0": []}
        outputs = {}
        for _ in range(args.runs):
            for path in ("1", "0"):
                os.environ["BLITZAR_B200_NORMALIZE_GENS"] = path
                for _ in range(args.warmup):
                    step()
                bb.synchronize()
                e0, e1 = bb.Event(), bb.Event()
                e0.record()
                for _ in range(args.steps):
                    step()
                e1.record()
                bb.synchronize()
                times[path].append(e0.elapsed_ms(e1) / args.steps)
                outputs[path] = out.cpu().numpy().copy()
        same = bool(np.array_equal(outputs["1"], outputs["0"]))
        w = {"same_commitments": same}
        for path, label in (("1", "normalised"), ("0", "caller Z")):
            t = times[path]
            w[label] = {"median_ms": statistics.median(t), "min_ms": min(t), "max_ms": max(t), "runs_ms": t}
            print(f"{name:9s} {label:10s}: median {statistics.median(t):.4f} ms/step "
                  f"(range {min(t):.4f}-{max(t):.4f}, {args.runs} runs x {args.steps} steps)")
        gain = 1 - w["normalised"]["median_ms"] / w["caller Z"]["median_ms"]
        w["gain"] = gain
        print(f"{name:9s} gain {100 * gain:.1f} %, commitments identical: {same}")
        if name == "c2":
            for path, label in (("1", "normalised"), ("0", "caller Z")):
                os.environ["BLITZAR_B200_NORMALIZE_GENS"] = path
                rows = trace(bb, step, 5)
                w[label]["trace"] = rows
                ie = [r["ingest_end_after_sort_end_us"] for r in rows
                      if r["ingest_end_after_sort_end_us"] is not None]
                gs = [r["gather_start_after_sort_end_us"] for r in rows]
                if gs:
                    print(f"c2 {label:10s}: ingestion ends {statistics.median(ie) if ie else float('nan'):+.1f} us "
                          f"after the sort, gathering level starts {statistics.median(gs):+.1f} us after it "
                          f"(median of {len(gs)} steps)")
        result["workloads"][name] = w
        assert same, f"{name}: commitments differ between the two paths"
    os.environ.pop("BLITZAR_B200_NORMALIZE_GENS", None)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "normalize_timing.json"), "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
