"""The C-ABI shared library loads and exports every symbol include/blitzar_b200.h declares
(no compute calls — there is no GPU here), and the product has no CPU fallback."""
import ctypes
import os
import re
import subprocess

import pytest

from tests.common import ROOT

HEADER = os.path.join(ROOT, "include", "blitzar_b200.h")


def declared_symbols():
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b((?:sxt|b200)_[a-z0-9_]+)\s*\(", text)))


@pytest.fixture(scope="module")
def lib():
    from blitzar_b200 import api
    if not os.path.exists(api.LIB_PATH):
        from blitzar_b200 import build
        build.build_product()
    return ctypes.CDLL(api.LIB_PATH), api


def test_header_declares_the_18_reference_entry_points():
    from blitzar_b200 import api
    sxt = [s for s in declared_symbols() if s.startswith("sxt_")]
    assert sorted(sxt) == sorted(api.SXT_SYMBOLS) and len(sxt) == 18


def test_library_exports_every_declared_symbol(lib):
    L, api = lib
    for name in declared_symbols():
        assert hasattr(L, name), name
    assert sorted(declared_symbols()) == sorted(api.SXT_SYMBOLS + api.B200_SYMBOLS)


def test_only_declared_symbols_are_exported(lib):
    _, api = lib
    out = subprocess.check_output(["nm", "-D", "--defined-only", api.LIB_PATH]).decode()
    exported = sorted(l.split()[-1] for l in out.splitlines() if " T " in l)
    assert exported == sorted(declared_symbols())


def test_struct_layouts_match_the_reference_abi():
    from blitzar_b200 import api
    assert ctypes.sizeof(api.sxt_sequence_descriptor) == 32
    assert api.sxt_sequence_descriptor.n.offset == 8
    assert api.sxt_sequence_descriptor.data.offset == 16
    assert api.sxt_sequence_descriptor.is_signed.offset == 24
    assert ctypes.sizeof(api.sxt_config) == 16


def test_product_sources_never_reference_the_oracle():
    """No product source includes, imports, links or opens anything under oracle/ or tests/ (the
    emulation switch B200_EMULATE is only ever defined by tests/emul/emul.cpp)."""
    bad = []
    pat = re.compile(r'#\s*include\s+"[^"]*(oracle|tests)/|^\s*(from|import)\s+(oracle|tests)\b|'
                     r'#\s*define\s+B200_EMULATE|libmsm_oracle|libblitzar_ref_cpu|libb200_emul',
                     re.M)
    for base, _, files in os.walk(os.path.join(ROOT, "blitzar_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")) and f != "build.py":
                if pat.search(open(os.path.join(base, f)).read()):
                    bad.append(f)
    assert not bad, bad


def test_c_example_compiles_and_links_against_the_library(lib, tmp_path):
    """examples/cbindings1.c (the reference's example/cbindings1/main.cc in plain C99) compiles against
    include/blitzar_b200.h and links against the product library: the header is valid C and every
    entry point it uses resolves. (It is not run here: no GPU, no CPU fallback.)"""
    _, api = lib
    exe = str(tmp_path / "cbindings1")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "examples", "cbindings1.c"),
                           "-L", os.path.dirname(api.LIB_PATH), "-lblitzar_b200",
                           "-Wl,-rpath," + os.path.dirname(api.LIB_PATH), "-o", exe])
    out = subprocess.check_output(["nm", "-u", exe]).decode()
    for sym in ("sxt_init", "sxt_curve25519_compute_pedersen_commitments", "sxt_multiexp_handle_new",
                "sxt_fixed_multiexponentiation"):
        assert sym in out
