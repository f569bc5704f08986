"""Batched inner-product arguments on the GPU: P proofs per b200_curve25519_prove_inner_products /
_verify_ call against the same P proofs through the single calls one after another, in the same
process and alternating. Prints per-proof times, proofs per second, whether batched and looped
results are byte-identical, and the share of a batched round that the device waits for the host
(transcript, challenge inversions, table staging and the launch of the first fold: the gap between
the end of the round's device-to-host copy and the start of its first fold kernel, from a
torch.profiler trace).

    python tests/ipa_batch_timing.py [TRACE_DIR]   # traces kept in TRACE_DIR (default: a temp dir)"""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import blitzar_b200 as bb  # noqa: E402

L = 2**252 + 27742317777372353535851937790883648493
REPS = 3
OUT = sys.argv[1] if len(sys.argv) > 1 else tempfile.mkdtemp(prefix="ipa_batch_")


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit",
                                        "--format=csv,noheader"]).decode().strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def scalars(rng, n):
    v = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    v[:, 31] &= 0x0F
    return v


def problem(rng, ns):
    a = [scalars(rng, n) for n in ns]
    b = [scalars(rng, n) for n in ns]
    t = np.zeros((len(ns), 203), np.uint8)
    t[:, :200] = rng.integers(0, 256, (len(ns), 200), dtype=np.uint8)
    return a, b, t


def verifier_inputs(a, b):
    """products <a_p, b_p> and a_commits <a_p, g(0 ..)> (one fixed-base call for the batch)."""
    P, nmax = len(a), max(x.shape[0] for x in a)
    to_int = lambda m: [int.from_bytes(bytes(r), "little") for r in m]
    products = np.stack([np.frombuffer((sum(x * y for x, y in zip(to_int(ap), to_int(bp))) % L)
                                       .to_bytes(32, "little"), np.uint8) for ap, bp in zip(a, b)])
    rows = np.zeros((nmax, P, 32), np.uint8)
    for p, x in enumerate(a):
        rows[:x.shape[0], p] = x
    h = bb.MultiexpHandle(0, bb.get_generators(nmax, 0))
    commits = h.fixed_multiexponentiation(32, P, nmax, rows.reshape(nmax, P * 32))
    h.free()
    return products, commits


def prove_loop(a, b, t0):
    t = t0.copy()
    return [bb.prove_inner_product(t[p], a[p], b[p], 0) for p in range(len(a))], t


def prove_batch(a, b, t0):
    t = t0.copy()
    return bb.prove_inner_products(t, a, b, [0] * len(a)), t


def verify_loop(b, prods, commits, proofs, t0):
    t = t0.copy()
    return np.array([bb.verify_inner_product(t[p], b[p], prods[p], commits[p], *proofs[p], 0)
                     for p in range(len(b))]), t


def verify_batch(b, prods, commits, proofs, t0):
    t = t0.copy()
    return bb.verify_inner_products(t, b, prods, commits, [x[0] for x in proofs],
                                    [x[1] for x in proofs], np.stack([x[2] for x in proofs]),
                                    [0] * len(b)), t


def alternate(f_loop, f_batch):
    """best-of-REPS seconds of each, run alternately (after one warm-up call of each)"""
    f_loop(), f_batch()
    tl, tb = [], []
    for _ in range(REPS):
        for f, acc in ((f_loop, tl), (f_batch, tb)):
            s = time.perf_counter()
            f()
            acc.append(time.perf_counter() - s)
    return min(tl), min(tb)


def host_share(a, b, t0, label):
    """share of each batched round the device spends waiting for the host, from a kernel trace"""
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            prove_batch(a, b, t0)
        os.makedirs(OUT, exist_ok=True)
        path = os.path.join(OUT, f"ipa_batch_{label}.pt.trace.json")
        prof.export_chrome_trace(path)
        ev = [e for e in json.load(open(path))["traceEvents"]
              if e.get("cat") in ("kernel", "gpu_memcpy") and "ts" in e]
        ev.sort(key=lambda e: e["ts"])
        dots = [e["ts"] for e in ev if "IpaDotSegBody" in e["name"]]
        shares = []
        for r, start in enumerate(dots):
            end = dots[r + 1] if r + 1 < len(dots) else None
            inside = [e for e in ev if e["ts"] >= start and (end is None or e["ts"] < end)]
            fold = next((e for e in inside if "IpaFoldScalarsSegBody" in e["name"]), None)
            copy = [e for e in inside if e["cat"] == "gpu_memcpy" and "DtoH" in e["name"] and fold
                    and e["ts"] < fold["ts"]]
            if fold is None or not copy or end is None:
                continue
            gap = fold["ts"] - (copy[-1]["ts"] + copy[-1]["dur"])
            shares.append(gap / (end - start))
        if not shares:
            return "not measured (no rounds in the trace)"
        return (f"host share per round: median {100 * np.median(shares):.0f} %, "
                f"min {100 * min(shares):.0f} %, max {100 * max(shares):.0f} % ({len(shares)} rounds)")
    except Exception as e:  # noqa: BLE001
        return f"not measured ({type(e).__name__}: {e})"


def main():
    print(f"card: {card()}", flush=True)
    bb.sxt_init(num_precomputed_generators=(1 << 18) + 1)
    rng = np.random.default_rng(0)
    shapes = [(P, [1 << logn] * P, f"P={P} n=2^{logn}") for logn in (10, 14) for P in (1, 16, 256)]
    mixed = [int(v) for v in rng.integers(1 << 8, (1 << 14) + 1, 64)]
    shapes.append((64, mixed, "P=64 mixed n in [2^8, 2^14]"))
    for P, ns, label in shapes:
        a, b, t0 = problem(rng, ns)
        (pl, tl), (pb, tb) = prove_loop(a, b, t0), prove_batch(a, b, t0)
        same = all(np.array_equal(x, y) for u, v in zip(pl, pb) for x, y in zip(u, v)) and \
            np.array_equal(tl, tb)
        lo, ba = alternate(lambda: prove_loop(a, b, t0), lambda: prove_batch(a, b, t0))
        print(f"{label}: prove  loop {1e3 * lo / P:8.2f} ms/proof ({P / lo:8.1f}/s), batch "
              f"{1e3 * ba / P:8.2f} ms/proof ({P / ba:8.1f}/s), x{lo / ba:.2f}, identical: {same}",
              flush=True)
        prods, commits = verifier_inputs(a, b)
        (rl, vl), (rb, vb) = verify_loop(b, prods, commits, pb, t0), verify_batch(b, prods, commits,
                                                                                  pb, t0)
        same_v = np.array_equal(rl, rb) and np.array_equal(vl, vb) and bool(rb.all())
        lo, ba = alternate(lambda: verify_loop(b, prods, commits, pb, t0),
                           lambda: verify_batch(b, prods, commits, pb, t0))
        print(f"{label}: verify loop {1e3 * lo / P:8.2f} ms/proof ({P / lo:8.1f}/s), batch "
              f"{1e3 * ba / P:8.2f} ms/proof ({P / ba:8.1f}/s), x{lo / ba:.2f}, all accepted and "
              f"identical: {same_v}", flush=True)
        if P >= 16:
            print(f"{label}: {host_share(a, b, t0, f'P{P}_nmax{max(ns)}')}", flush=True)


if __name__ == "__main__":
    main()
