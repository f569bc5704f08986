"""Partition tables in the reference's handle-file format at the reference's default window width
(w = 16), bn254 and ristretto255, n = 256 and 4096 synthetic generators:
  - device build: b200_partition_table_device into HBM, CUDA events, best of 3 after a warm-up;
  - file write: MultiexpHandle.write_partition_table end to end (build, copy, fwrite, fclose; the
    page cache absorbs what the disk has not taken yet), best of 3, and its rate in MB/s;
  - the reference's own writer (oracle/_ref, refcpu.write_partition_table) for n = 256 on one core,
    when that library has been built.
Prints one line per measurement, with the card's name and power limit first.
    python tests/partition_table_timing.py [out_dir]"""
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import blitzar_b200 as bb  # noqa: E402

W = 16
CURVES = {2: "bn254", 0: "ristretto255"}


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit",
                                        "--format=csv,noheader"], text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown card"


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else tempfile.mkdtemp()
    os.makedirs(out_dir, exist_ok=True)
    assert bb.sxt_init() == 0
    print(f"card: {card()}", flush=True)
    for curve, name in CURVES.items():
        for n in (256, 4096):
            gens = bb.synthetic_generators(curve, n, projective=True)
            g = bb.DeviceBuffer(host=gens)
            nbytes = bb.partition_table_bytes(curve, n, W)
            out = bb.DeviceBuffer(nbytes)
            best = 1e9
            for rep in range(4):
                e0, e1 = bb.Event(), bb.Event()
                e0.record()
                bb.partition_table_device(curve, out.ptr, g.ptr, n, W)
                e1.record()
                if rep:
                    best = min(best, e0.elapsed_ms(e1))
                else:
                    bb.synchronize()
            out.free()
            g.free()
            h = bb.MultiexpHandle(curve, gens)
            path = os.path.join(tempfile.mkdtemp(), "table.bin")
            best_file = 1e9
            for _ in range(3):
                t = time.perf_counter()
                h.write_partition_table(path, W)
                best_file = min(best_file, time.perf_counter() - t)
                os.remove(path)
            h.free()
            mb = (nbytes + 4) / 1e6
            print(f"{name} n={n} w={W} table={mb:.1f} MB: device build {best:.2f} ms "
                  f"({mb / best * 1e3:.0f} MB/s of table), file write {best_file * 1e3:.1f} ms "
                  f"({mb / best_file:.0f} MB/s)", flush=True)
    from oracle import refcpu
    if not refcpu.available():
        print("reference writer: not built (oracle/_ref)")
        return
    os.sched_setaffinity(0, {sorted(os.sched_getaffinity(0))[0]})
    with open("/proc/cpuinfo") as f:
        cpu = next((line.split(":", 1)[1].strip() for line in f if line.startswith("model name")), "?")
    print(f"host cpu: {cpu}", flush=True)
    for curve, name in CURVES.items():
        n = 256
        gens = bb.synthetic_generators(curve, n, projective=True)
        path = os.path.join(out_dir, f"ref_{name}.bin")
        t = time.perf_counter()
        refcpu.write_partition_table(curve, path, gens, W)
        dt = time.perf_counter() - t
        os.remove(path)
        print(f"reference writer (one core) {name} n={n} w={W}: {dt:.2f} s", flush=True)


if __name__ == "__main__":
    main()
