"""Generates tests/golden/ptable_curve{c}.npz: the input generators of every case of
tests/partition_tables.py and the digest (partition_tables.table_digest) of the partition table the
REFERENCE's own writer (oracle/_ref, in_memory_partition_table_accessor::write_to_file) produces for
them. The n = 7, w = 3 case is tests/golden/ref_table_curve{c}_w3.bin (make_table_files.py).
Run where the reference oracle is built:  python tests/golden/make_partition_table_files.py"""
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import port, refcpu  # noqa: E402
from tests import partition_tables as pt  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))

if __name__ == "__main__":
    port.build()
    tmp = tempfile.mkdtemp()
    for curve in range(4):
        out = {}
        for name, (n, w, _) in pt.CASES.items():
            g = pt.case_generators(port, curve, name)
            path = os.path.join(tmp, f"{curve}_{name}.bin")
            refcpu.write_partition_table(curve, path, g, w)
            raw = np.fromfile(path, dtype=np.uint8)
            assert int(raw[:4].view("<u4")[0]) == w
            out[f"gens_{name}"] = g
            out[f"sha_{name}"] = np.array(pt.table_digest(curve, raw[4:]))
        np.savez(os.path.join(HERE, f"ptable_curve{curve}.npz"), **out)
