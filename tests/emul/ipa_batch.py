"""TEST INFRASTRUCTURE — Python side of the emulated batch inner-product entries
(tests/emul/emul_ipa_batch.cpp), in the library of the emulation harness (tests/emul/harness.py).

Engine(num_builtin) offers the batched calls beside the harness's single calls, with the names of the
product's Python API, so that tests can run the same checks on both."""
import ctypes as C
import functools

from blitzar_b200.api import call_prove_inner_products, call_verify_inner_products
from tests.emul import harness


class Engine:
    """Emulated single and batched inner-product calls. The batched calls see `num_builtin`
    precomputed generators; the single calls see what harness.configure set (give both the same
    number when they are compared)."""

    def __init__(self, num_builtin=0):
        self.num_builtin = num_builtin
        self.prove_inner_product = harness.prove_inner_product
        self.verify_inner_product = harness.verify_inner_product

    def _entry(self, name):
        f = getattr(harness.lib(), name)
        if name.startswith("emul_verify"):
            f.restype = C.c_uint32
        return functools.partial(f, C.c_uint64(self.num_builtin))

    @property
    def prove_entry(self):
        """emul_prove_inner_products with b200_curve25519_prove_inner_products's arguments"""
        return self._entry("emul_prove_inner_products")

    @property
    def verify_entry(self):
        """emul_verify_inner_products with b200_curve25519_verify_inner_products's arguments"""
        return self._entry("emul_verify_inner_products")

    def prove_inner_products(self, transcripts, a_list, b_list, offsets=None):
        return call_prove_inner_products(self.prove_entry, transcripts, a_list, b_list, offsets)

    def verify_inner_products(self, transcripts, b_list, products, a_commits, l_list, r_list,
                              ap_values, offsets=None):
        return call_verify_inner_products(self.verify_entry, transcripts, b_list, products,
                                          a_commits, l_list, r_list, ap_values, offsets)
