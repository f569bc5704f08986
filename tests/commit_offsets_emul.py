"""Python side of the emulated per-column-offset commitments (tests/emul/offsets_emul.cpp), in the
emulation library that tests/emul/harness.py builds and loads."""
import ctypes as C

import numpy as np

from tests.emul import harness


def configure(ranges=1, range_entries=0, group_entries=0, pair_levels=-1, table_policy=0,
              num_builtin=0, window_bits=0):
    """Engine options of commit_offsets: upload pieces, sort-pass and column-group entry limits
    (0 = default), batch-affine pair levels (-1 = automatic), fixed-base table policy (1 = always,
    2 = never, 0 = cost model), and num_builtin precomputed built-in generators with a fixed-base
    table of window_bits (0 = none). Every call resets what it is not given."""
    harness.lib().emul_offsets_configure(C.c_uint(ranges), C.c_ulonglong(range_entries),
                                         C.c_ulonglong(group_entries), C.c_int(pair_levels),
                                         C.c_uint(table_policy), C.c_uint64(num_builtin),
                                         C.c_uint(window_bits))


def commit_offsets(curve_id, columns, offsets=None, generators=None):
    """emul_commit_offsets: column j at generator offsets[j] (None = all 0); generators None = the
    built-in ristretto255 generators."""
    desc, keep = harness._desc(columns)
    out = np.zeros((len(columns), harness.SIZES[curve_id][2]), dtype=np.uint8)
    gp = C.c_void_p(generators.ctypes.data) if generators is not None else C.c_void_p(None)
    offs = None if offsets is None else np.ascontiguousarray(offsets, dtype=np.uint64)
    harness.lib().emul_commit_offsets(C.c_uint(curve_id), C.c_void_p(out.ctypes.data),
                                      C.c_uint32(len(columns)), desc, gp,
                                      C.c_void_p(offs.ctypes.data) if offs is not None
                                      else C.c_void_p(None))
    return out
