"""TEST INFRASTRUCTURE — Python side of tests/emul/partition_msm_emul.cpp: fixed-base MSMs over a
handle that carries a partition table, through the product's kernel bodies run as serial host loops,
and the routing of the cost model."""
import ctypes as C

import numpy as np

POLICY_MODEL, POLICY_TABLE, POLICY_ENGINE = 0, 1, 2


def fixed_msm(emul, curve_id, generators_p, window_width, policy, num_outputs, n, scalars,
              element_num_bytes=0, output_bit_table=None, output_lengths=None, chunk_groups=0):
    """Projective ABI results of a fixed MSM over a handle with a partition table of the given width
    (0 = none), built chunk_groups groups at a time (0 = one chunk)."""
    res = np.zeros((num_outputs, emul.SIZES[curve_id][0]), dtype=np.uint8)
    mode = 0 if output_bit_table is None else (1 if output_lengths is None else 2)
    bt = (C.c_uint * num_outputs)(*output_bit_table) if output_bit_table is not None else None
    ol = (C.c_uint * num_outputs)(*output_lengths) if output_lengths is not None else None
    scalars = np.ascontiguousarray(scalars, dtype=np.uint8).reshape(-1)
    scalars = np.concatenate([scalars, np.zeros(64, dtype=np.uint8)])
    generators_p = np.ascontiguousarray(generators_p, dtype=np.uint8)
    emul.lib().emul_partition_fixed_msm(
        C.c_uint(curve_id), C.c_void_p(res.ctypes.data), C.c_void_p(generators_p.ctypes.data),
        C.c_uint(generators_p.shape[0]), C.c_uint(window_width), C.c_uint64(chunk_groups),
        C.c_uint(policy), C.c_int(mode), C.c_uint(element_num_bytes), bt, ol,
        C.c_uint(num_outputs), C.c_uint(n), C.c_void_p(scalars.ctypes.data))
    return res


def route(emul, curve_id, num_gens, window_width, policy, widths, lengths):
    """Indices of the outputs the cost model answers from the table."""
    k = len(widths)
    out = (C.c_uint * max(k, 1))()
    emul.lib().emul_partition_route.restype = C.c_uint
    cnt = emul.lib().emul_partition_route(
        C.c_uint(curve_id), C.c_uint(num_gens), C.c_uint(window_width), C.c_uint(policy),
        (C.c_uint * k)(*widths), (C.c_uint * k)(*lengths), C.c_uint(k), out)
    return [int(out[i]) for i in range(cnt)]
