"""TEST INFRASTRUCTURE — ctypes binding of the C oracle port (oracle/msm_oracle.c).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this module; the product never does. Same call shapes as oracle/refcpu.py so tests can swap them.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(_HERE, "msm_oracle.c")
LIB_PATH = os.path.join(_HERE, "libmsm_oracle.so")
SIZES = {0: (160, 160, 32), 1: (144, 104, 48), 2: (96, 72, 72), 3: (96, 72, 72)}


class SequenceDescriptor(C.Structure):
    _fields_ = [("element_nbytes", C.c_uint8), ("n", C.c_uint64), ("data", C.c_void_p),
                ("is_signed", C.c_int)]


_lib = None


def build():
    if not os.path.exists(LIB_PATH) or os.path.getmtime(LIB_PATH) < os.path.getmtime(SRC):
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-w", SRC, "-o", LIB_PATH])
    return LIB_PATH


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
    return _lib


def make_descriptors(columns):
    arr = (SequenceDescriptor * max(1, len(columns)))()
    keep = []
    for i, (data, is_signed) in enumerate(columns):
        data = np.ascontiguousarray(data, dtype=np.uint8)
        keep.append(data)
        arr[i].element_nbytes = data.shape[1]
        arr[i].n = data.shape[0]
        arr[i].data = data.ctypes.data if data.shape[0] else None
        arr[i].is_signed = int(is_signed)
    return arr, keep


def ristretto_generators(n, offset=0):
    out = np.zeros((n, 160), dtype=np.uint8)
    if n:
        lib().oracle_ristretto255_get_generators(C.c_void_p(out.ctypes.data), C.c_uint64(n),
                                                 C.c_uint64(offset))
    return out


def test_points(curve_id, n, seed=0):
    """(projective ABI array, commitment-API affine array) of deterministic test points."""
    psz, asz, _ = SIZES[curve_id]
    p2 = np.zeros((n, psz), dtype=np.uint8)
    af = np.zeros((n, asz), dtype=np.uint8)
    lib().oracle_test_points(C.c_uint(curve_id), C.c_void_p(af.ctypes.data),
                             C.c_void_p(p2.ctypes.data), C.c_uint64(n), C.c_uint64(seed))
    return p2, af


def commit(curve_id, columns, generators=None, offset=0):
    desc, keep = make_descriptors(columns)
    out = np.zeros((len(columns), SIZES[curve_id][2]), dtype=np.uint8)
    gp = C.c_void_p(generators.ctypes.data) if generators is not None else C.c_void_p(None)
    lib().oracle_commit(C.c_uint(curve_id), C.c_void_p(out.ctypes.data), C.c_uint32(len(columns)),
                        desc, gp, C.c_uint64(offset))
    return out


def normalize(curve_id, projective):
    n = projective.shape[0]
    out = np.zeros((n, SIZES[curve_id][2]), dtype=np.uint8)
    projective = np.ascontiguousarray(projective)
    lib().oracle_normalize(C.c_uint(curve_id), C.c_void_p(out.ctypes.data),
                           C.c_void_p(projective.ctypes.data), C.c_uint64(n))
    return out


def fixed_msm(curve_id, generators_p, num_outputs, n, scalars, element_num_bytes=0,
              output_bit_table=None, output_lengths=None):
    res = np.zeros((num_outputs, SIZES[curve_id][0]), dtype=np.uint8)
    mode = 0 if output_bit_table is None else (1 if output_lengths is None else 2)
    bt = (C.c_uint * num_outputs)(*output_bit_table) if output_bit_table is not None else None
    ol = (C.c_uint * num_outputs)(*output_lengths) if output_lengths is not None else None
    scalars = np.ascontiguousarray(scalars, dtype=np.uint8)
    generators_p = np.ascontiguousarray(generators_p)
    lib().oracle_fixed_msm(C.c_uint(curve_id), C.c_void_p(res.ctypes.data),
                           C.c_void_p(generators_p.ctypes.data), C.c_uint(generators_p.shape[0]),
                           C.c_int(mode), C.c_uint(element_num_bytes), bt, ol,
                           C.c_uint(num_outputs), C.c_uint(n), C.c_void_p(scalars.ctypes.data))
    return res


# ---- inner-product argument ---------------------------------------------------------------------
def transcript_new(label=b"ip-test"):
    t = np.zeros(203, dtype=np.uint8)
    lib().oracle_transcript_new(C.c_void_p(t.ctypes.data), C.c_char_p(label))
    return t


def prove_inner_product(transcript, a, b, generators_offset=0):
    n = a.shape[0]
    rounds = max(0, (n - 1).bit_length())
    lv = np.zeros((max(rounds, 1), 32), dtype=np.uint8)
    rv = np.zeros((max(rounds, 1), 32), dtype=np.uint8)
    ap = np.zeros(32, dtype=np.uint8)
    a = np.ascontiguousarray(a, dtype=np.uint8)
    b = np.ascontiguousarray(b, dtype=np.uint8)
    lib().oracle_prove_inner_product(C.c_void_p(lv.ctypes.data), C.c_void_p(rv.ctypes.data),
                                     C.c_void_p(ap.ctypes.data), C.c_void_p(transcript.ctypes.data),
                                     C.c_uint64(n), C.c_uint64(generators_offset),
                                     C.c_void_p(a.ctypes.data), C.c_void_p(b.ctypes.data))
    return lv[:rounds], rv[:rounds], ap


# encodings the test-only prover can emit for L_j / R_j (oracle_prove_inner_product_encoded)
ENC_CANONICAL, ENC_NEGATED, ENC_PLUS_P, ENC_TOP_BIT, ENC_REPLACE = range(5)
# checks of RFC 9496 decoding that the test-only lax verifier skips (bits, combined with |): the
# canonical check, the sign of s, the sign of t, y != 0; LAX_MOD_P reads s as the 256-bit integer
# mod p instead of from its low 255 bits
LAX_NONE, LAX_CANONICAL, LAX_SIGN, LAX_MOD_P, LAX_T, LAX_Y = 0, 1, 2, 4, 8, 16


def prove_inner_product_encoded(transcript, a, b, generators_offset=0, l_modes=None, r_modes=None,
                                replacements=None):
    """The prover, emitting L_j in encoding l_modes[j] and R_j in r_modes[j] (ENC_*; ENC_REPLACE
    emits replacements[j] / replacements[k + j]) and taking every challenge over the emitted bytes.
    Returns (l_vector, r_vector, ap_value, the challenges x_j as [k, 32] bytes)."""
    n = a.shape[0]
    rounds = max(0, (n - 1).bit_length())
    lv = np.zeros((max(rounds, 1), 32), dtype=np.uint8)
    rv = np.zeros((max(rounds, 1), 32), dtype=np.uint8)
    ap = np.zeros(32, dtype=np.uint8)
    modes = np.zeros(2 * rounds + 1, dtype=np.uint8)
    if l_modes is not None:
        modes[:rounds] = l_modes
    if r_modes is not None:
        modes[rounds:2 * rounds] = r_modes
    rep = np.zeros((2 * rounds + 1, 32), dtype=np.uint8)
    x = np.zeros((max(rounds, 1), 32), dtype=np.uint8)
    if replacements is not None:
        rep[:2 * rounds] = replacements
    a = np.ascontiguousarray(a, dtype=np.uint8)
    b = np.ascontiguousarray(b, dtype=np.uint8)
    lib().oracle_prove_inner_product_encoded(
        C.c_void_p(lv.ctypes.data), C.c_void_p(rv.ctypes.data), C.c_void_p(ap.ctypes.data),
        C.c_void_p(transcript.ctypes.data), C.c_uint64(n), C.c_uint64(generators_offset),
        C.c_void_p(a.ctypes.data), C.c_void_p(b.ctypes.data), C.c_void_p(modes.ctypes.data),
        C.c_void_p(rep.ctypes.data), C.c_void_p(x.ctypes.data))
    return lv[:rounds], rv[:rounds], ap, x[:rounds]


def verify_inner_product(transcript, b, product, a_commit, l_vector, r_vector, ap_value,
                         generators_offset=0, lax=LAX_NONE):
    n = b.shape[0]
    b = np.ascontiguousarray(b, dtype=np.uint8)
    lv = np.ascontiguousarray(l_vector if len(l_vector) else np.zeros((1, 32), np.uint8))
    rv = np.ascontiguousarray(r_vector if len(r_vector) else np.zeros((1, 32), np.uint8))
    lib().oracle_verify_inner_product_lax.restype = C.c_int
    return int(lib().oracle_verify_inner_product_lax(
        C.c_void_p(transcript.ctypes.data), C.c_uint64(n), C.c_uint64(generators_offset),
        C.c_void_p(b.ctypes.data), C.c_void_p(np.ascontiguousarray(product).ctypes.data),
        C.c_void_p(np.ascontiguousarray(a_commit).ctypes.data), C.c_void_p(lv.ctypes.data),
        C.c_void_p(rv.ctypes.data), C.c_void_p(np.ascontiguousarray(ap_value).ctypes.data),
        C.c_int(lax)))
