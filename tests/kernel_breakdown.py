#!/usr/bin/env python3
"""Per-kernel time of one device-resident bench step, grouped by kernel body.

    python tests/kernel_breakdown.py [--workload {c2,c3,c4_share}] [--steps 20] [--warmup 5] [--out DIR]

The inputs are built exactly as bench.py builds them (synthetic generators in HBM, make_scalars with
seed 12345 and the workload's top-byte mask, b200_commit_device on the library stream). The step time
is taken first with CUDA events and no profiler attached; the kernels are then traced with
torch.profiler (CUDA activity only) in a run of their own. Kernel time is summed per body name
(`k_run<b200::CountBody>` -> CountBody, `k_block<b200::BinSortBody>` -> BinSortBody) and reported in
microseconds per step and as a share of the event-timed step. Kernels on the tail stream overlap the main stream, so the shares can add up to more
than 100 %. The card name and power limit are printed and written with the table to DIR/<workload>.json.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import make_scalars  # noqa: E402

# name -> (curve, log2 n, columns, top-byte mask), as in bench.py
WORKLOADS = {
    "c2": (0, 20, 1, 0x0F),
    "c3": (1, 22, 1, 0x7F),
    "c4_share": (0, 20, 8, 0x0F),
}
# the bucket sort: atomic path, then binned path
SORT_BODIES = ("CountBody", "ScanUpBody", "ScanTopBody", "ScanDownBody", "ScatterBody",
               "MicroCountBody", "PlanBinsBody", "CoarseScatterBody", "BinSortBody")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                           timeout=30).stdout.strip()
        name, power, clock = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clock}
    except Exception as e:  # the table is still useful without it, but say so
        return {"name": None, "error": str(e)}


def body_name(kernel):
    """`void b200::k_run<b200::AccumulateBody<b200::Ed25519, true, ...> >(...)` -> AccumulateBody<Ed25519,
    true, ...>; kernels that are not engine bodies (memset, memcpy, ...) keep their own name."""
    m = re.search(r"k_(?:run|block)<(.*)>\s*\(", kernel)
    if not m:
        return kernel[:80]
    return m.group(1).replace("b200::", "").strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c2", choices=sorted(WORKLOADS))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "kernel_breakdown"))
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    import blitzar_b200 as bb

    curve, logn, ncol, mask = WORKLOADS[args.workload]
    n = 1 << logn
    torch.cuda.set_device(0)
    assert bb.sxt_init(device=0) == 0
    gens = torch.empty((n, bb.CURVE_SIZES[curve][1]), dtype=torch.uint8, device="cuda")
    bb.synthetic_generators_device(curve, gens.data_ptr(), n, 0, projective=False)
    scal = [torch.from_numpy(make_scalars(n, 12345 + 1000 * j, mask)).cuda() for j in range(ncol)]
    out = torch.zeros((ncol * 72 + 64,), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    shapes, ptrs = [(n, 32, 0)] * ncol, [s.data_ptr() for s in scal]

    def step():
        bb.commit_device(curve, shapes, ptrs, gens.data_ptr(), out.data_ptr())

    for _ in range(args.warmup):
        step()
    bb.synchronize()
    e0, e1 = bb.Event(), bb.Event()
    e0.record()
    for _ in range(args.steps):
        step()
    e1.record()
    bb.synchronize()
    step_us = 1e3 * e0.elapsed_ms(e1) / args.steps

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        bb.synchronize()
        torch.cuda.synchronize()

    groups = {}
    for ev in prof.key_averages():
        us = getattr(ev, "self_device_time_total", None)
        if us is None:
            us = ev.self_cuda_time_total
        if us <= 0:
            continue
        g = groups.setdefault(body_name(ev.key), [0.0, 0])
        g[0] += us
        g[1] += ev.count
    rows = sorted(({"kernel": k, "us_per_step": v[0] / args.steps, "launches_per_step": v[1] / args.steps,
                    "share_of_step": v[0] / args.steps / step_us} for k, v in groups.items()),
                  key=lambda r: -r["us_per_step"])
    sort_us = sum(r["us_per_step"] for r in rows if r["kernel"] in SORT_BODIES)
    result = {"workload": args.workload, "card": card(), "steps": args.steps, "step_us": step_us,
              "kernel_us_sum": sum(r["us_per_step"] for r in rows), "sort_us": sort_us,
              "sort_bodies": list(SORT_BODIES), "kernels": rows}

    c = result["card"]
    print(f"{args.workload}: {step_us:.1f} us per step (CUDA events, {args.steps} steps) on "
          f"{c.get('name')} at a {c.get('power_limit')} power limit")
    print(f"{'kernel':70s} {'us/step':>9s} {'launches':>9s} {'share':>7s}")
    for r in rows:
        print(f"{r['kernel'][:70]:70s} {r['us_per_step']:9.1f} {r['launches_per_step']:9.1f} "
              f"{100 * r['share_of_step']:6.1f}%")
    print(f"bucket sort: {sort_us:.1f} us per step ({100 * sort_us / step_us:.1f}%)")
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, f"{args.workload}.json"), "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
