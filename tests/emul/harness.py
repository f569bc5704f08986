"""TEST INFRASTRUCTURE — Python side of the CPU emulation harness (tests/emul/emul.cpp).

Runs the product's kernel BODIES as serial host loops; used only by the `not gpu` tests to check
the pipeline logic without a GPU. The product library never links or calls any of this.

Every entry runs under one set of engine options: configure() sets them, options() sets them for a
block and restores the defaults after it.
"""
import contextlib
import ctypes as C

import numpy as np

from blitzar_b200 import build as _build
from blitzar_b200.api import (COMPACT_BYTES, CURVE_SIZES, call_field_op, make_descriptors,
                               partition_table_bytes)

# partition_policy: outputs of a fixed MSM over a handle with a partition table are answered from
# the table as the cost model decides, all of them, or none
POLICY_MODEL, POLICY_TABLE, POLICY_ENGINE = 0, 1, 2

# the arguments of emul_configure in order: name -> (C type, default)
_OPTIONS = {
    "ranges": (C.c_uint, 1),               # generator ranges (upload pieces) of a commitment
    "window_bits": (C.c_uint, 0),          # digit window (0 = chosen from the shape)
    "chunk1": (C.c_uint, 0),               # chunk lengths of the accumulation levels (0 = default)
    "chunkn": (C.c_uint, 0),
    "range_entries": (C.c_ulonglong, 0),   # entries of one sort pass (0 = 2^31)
    "group_entries": (C.c_ulonglong, 0),   # entries of one column group (0 = 2^30)
    "pair_levels": (C.c_int, -1),          # batch-affine pair levels (-1 = automatic)
    "pair_batch": (C.c_uint, 0),           # pairs per thread of a pair level (0 = 32)
    "scatter_window_major": (C.c_uint, 0),
    "normalize": (C.c_uint, 1),            # ed25519 caller generators normalised at ingestion
    "table_policy": (C.c_uint, 0),         # fixed-base tables: 0 cost model, 1 always, 2 never
    "table_window": (C.c_uint, 0),         # fixed-base table window of fixed_msm handles (0 = none)
    "partition_policy": (C.c_uint, POLICY_MODEL),
    "num_builtin": (C.c_uint64, 0),        # sxt_config::num_precomputed_generators
    "builtin_window": (C.c_uint, 0),       # fixed-base table window of the built-in generators
}

_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(_build.build_emul())
        for f in ("emul_point_bytes", "emul_partition_route", "emul_ingest_generators"):
            getattr(_lib, f).restype = C.c_uint
    return _lib


def configure(**options):
    """Sets every engine option: those given, and the others to their defaults (_OPTIONS)."""
    unknown = set(options) - set(_OPTIONS)
    if unknown:
        raise TypeError(f"unknown emulation options: {sorted(unknown)}")
    lib().emul_configure(*[t(options.get(k, d)) for k, (t, d) in _OPTIONS.items()])


@contextlib.contextmanager
def options(**opts):
    """configure(**opts) for the block; the defaults after it."""
    configure(**opts)
    try:
        yield
    finally:
        configure()


def _ptr(a):
    return C.c_void_p(None if a is None else a.ctypes.data)


def _commit(entry, curve_id, columns, generators, last, partials=False):
    desc, keep = make_descriptors(columns)
    width = point_bytes(curve_id) if partials else CURVE_SIZES[curve_id][2]
    out = np.zeros((len(columns), width), dtype=np.uint8)
    outs = (None, out) if partials else (out, None)
    entry(C.c_uint(curve_id), _ptr(outs[0]), _ptr(outs[1]), C.c_uint32(len(columns)), desc,
          _ptr(generators), last)
    return out


def commit(curve_id, columns, generators=None, offset=0):
    """emul_commit: commitments over generators (None = the built-in ristretto255 generators from
    `offset`)."""
    return _commit(lib().emul_commit, curve_id, columns, generators, C.c_uint64(offset))


def commit_partial(curve_id, columns, generators=None, offset=0):
    """emul_commit: the accumulator points of the commitments (point_bytes each)."""
    return _commit(lib().emul_commit, curve_id, columns, generators, C.c_uint64(offset), True)


def commit_offsets(curve_id, columns, offsets=None, generators=None):
    """emul_commit_offsets: column j at generator offsets[j] (None = all 0); generators None = the
    built-in ristretto255 generators."""
    offs = None if offsets is None else np.ascontiguousarray(offsets, dtype=np.uint64)
    return _commit(lib().emul_commit_offsets, curve_id, columns, generators, _ptr(offs))


def combine_partials(curve_id, partials, num_parts, count):
    out = np.zeros((count, CURVE_SIZES[curve_id][2]), dtype=np.uint8)
    partials = np.ascontiguousarray(partials)
    lib().emul_combine_partials(C.c_uint(curve_id), _ptr(out), _ptr(partials),
                                C.c_uint32(num_parts), C.c_uint32(count))
    return out


def point_bytes(curve_id):
    return int(lib().emul_point_bytes(C.c_uint(curve_id)))


def fixed_msm(curve_id, generators_p, num_outputs, n, scalars, element_num_bytes=0,
              output_bit_table=None, output_lengths=None, partition_window=0, chunk_groups=0):
    """emul_fixed: projective ABI results of a fixed MSM over a handle of generators_p with the
    configured fixed-base table window and, for partition_window != 0, a partition table of that
    width built chunk_groups groups at a time (0 = one chunk)."""
    res = np.zeros((num_outputs, CURVE_SIZES[curve_id][0]), dtype=np.uint8)
    mode = 0 if output_bit_table is None else (1 if output_lengths is None else 2)
    bt = (C.c_uint * num_outputs)(*output_bit_table) if output_bit_table is not None else None
    ol = (C.c_uint * num_outputs)(*output_lengths) if output_lengths is not None else None
    scalars = np.ascontiguousarray(scalars, dtype=np.uint8)
    scalars = np.concatenate([scalars.reshape(-1), np.zeros(64, dtype=np.uint8)])
    generators_p = np.ascontiguousarray(generators_p, dtype=np.uint8)
    lib().emul_fixed(C.c_uint(curve_id), _ptr(res), _ptr(generators_p),
                     C.c_uint(generators_p.shape[0]), C.c_uint(partition_window),
                     C.c_uint64(chunk_groups), C.c_int(mode), C.c_uint(element_num_bytes), bt, ol,
                     C.c_uint(num_outputs), C.c_uint(n), _ptr(scalars))
    return res


def partition_route(curve_id, num_gens, window_width, widths, lengths):
    """Indices of the outputs the configured partition policy answers from a table of width
    window_width."""
    k = len(widths)
    out = (C.c_uint * max(k, 1))()
    cnt = lib().emul_partition_route(C.c_uint(curve_id), C.c_uint(num_gens), C.c_uint(window_width),
                                     (C.c_uint * k)(*widths), (C.c_uint * k)(*lengths), C.c_uint(k),
                                     out)
    return [int(out[i]) for i in range(cnt)]


def partition_table(curve_id, generators_p, window_width, chunk_groups=0):
    """The partition table (no header) of projective ABI generators, `chunk_groups` groups per
    chunk (0 = one chunk)."""
    generators_p = np.ascontiguousarray(generators_p, dtype=np.uint8)
    n = generators_p.shape[0]
    out = np.zeros(partition_table_bytes(curve_id, n, window_width), dtype=np.uint8)
    lib().emul_partition_table(C.c_uint(curve_id), _ptr(out), _ptr(generators_p), C.c_uint64(n),
                               C.c_uint(window_width), C.c_uint64(chunk_groups))
    return out


def ingest_generators(generators):
    """(device generators [n, 128] bytes, Z = 0 flag) as the ingestion of ristretto255 ABI
    generators writes them, normalised or not as configured."""
    gens = np.ascontiguousarray(generators)
    out = np.zeros((gens.shape[0], 128), dtype=np.uint8)
    flag = lib().emul_ingest_generators(_ptr(gens), C.c_uint64(gens.shape[0]), _ptr(out))
    return out, int(flag)


def generators_from_reference_table(curve_id, path):
    """Generators (projective ABI structs) recovered from a reference-format handle file."""
    raw = np.fromfile(path, dtype=np.uint8)
    w = int(raw[:4].view("<u4")[0])
    groups = (raw.size - 4) // (COMPACT_BYTES[curve_id] << w)
    n = groups * w
    table = np.ascontiguousarray(raw[4:])
    out = np.zeros((n, CURVE_SIZES[curve_id][0]), dtype=np.uint8)
    lib().emul_ingest_compact(C.c_uint(curve_id), _ptr(table), C.c_uint(w), C.c_uint64(n),
                              _ptr(out))
    return out


def get_generators(n, offset=0):
    out = np.zeros((n, 160), dtype=np.uint8)
    lib().emul_get_generators(_ptr(out), C.c_uint64(n), C.c_uint64(offset))
    return out


def synth_generators(curve_id, n, first=0, projective=False):
    stride = CURVE_SIZES[curve_id][0 if (projective or curve_id == 0) else 1]
    out = np.zeros((n, stride), dtype=np.uint8)
    lib().emul_synth_generators(C.c_uint(curve_id), _ptr(out), C.c_uint64(n), C.c_uint64(first),
                                C.c_int(1 if projective else 0))
    return out


def field_op(field, op, a, b=None):
    """emul_field_op: b200_field_op's contract (blitzar_b200.api.call_field_op) on the CPU."""
    return call_field_op(lib().emul_field_op, field, op, a, b)


SCALAR_OPS = {name: code for code, name in enumerate(
    ["reduce", "mul", "mul_mont", "add", "sub", "neg", "inv", "inner_product"])}


def scalar_op(op, a, b=None):
    """emul_scalar_op: the host scalar arithmetic mod l (scalar25.h) on rows of 8 u32 limbs;
    inner_product returns the one sum over all rows."""
    a = np.ascontiguousarray(a, dtype=np.uint32).reshape(-1, 8)
    if b is not None:
        b = np.ascontiguousarray(b, dtype=np.uint32).reshape(a.shape)
    out = np.zeros((1 if op == "inner_product" else a.shape[0], 8), dtype=np.uint32)
    lib().emul_scalar_op.restype = C.c_uint
    rc = lib().emul_scalar_op(C.c_uint(SCALAR_OPS[op]), C.c_uint64(a.shape[0]), _ptr(a), _ptr(b),
                              _ptr(out))
    assert rc == 0, op
    return out


def prove_inner_product(transcript, a, b, generators_offset=0):
    """Emulated sxt_curve25519_prove_inner_product; returns (l_vector, r_vector, ap_value)."""
    n = a.shape[0]
    rounds = max(0, (n - 1).bit_length())
    lv = np.zeros((max(rounds, 1), 32), dtype=np.uint8)
    rv = np.zeros((max(rounds, 1), 32), dtype=np.uint8)
    ap = np.zeros(32, dtype=np.uint8)
    a = np.ascontiguousarray(a, dtype=np.uint8)
    b = np.ascontiguousarray(b, dtype=np.uint8)
    lib().emul_prove_inner_product(_ptr(lv), _ptr(rv), _ptr(ap), _ptr(transcript), C.c_uint64(n),
                                   C.c_uint64(generators_offset), _ptr(a), _ptr(b))
    return lv[:rounds], rv[:rounds], ap


def verify_inner_product(transcript, b, product, a_commit, l_vector, r_vector, ap_value,
                         generators_offset=0):
    n = b.shape[0]
    b = np.ascontiguousarray(b, dtype=np.uint8)
    lv = np.ascontiguousarray(l_vector if len(l_vector) else np.zeros((1, 32), np.uint8))
    rv = np.ascontiguousarray(r_vector if len(r_vector) else np.zeros((1, 32), np.uint8))
    product = np.ascontiguousarray(product)
    a_commit = np.ascontiguousarray(a_commit)
    ap_value = np.ascontiguousarray(ap_value)
    return int(lib().emul_verify_inner_product(
        _ptr(transcript), C.c_uint64(n), C.c_uint64(generators_offset), _ptr(b), _ptr(product),
        _ptr(a_commit), _ptr(lv), _ptr(rv), _ptr(ap_value)))
