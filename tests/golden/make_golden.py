"""Generates the committed golden fixtures from the REFERENCE's own CPU implementation
(oracle/_ref, built from a reference checkout by oracle/ref_build/Makefile). Run where it is built:

    python tests/golden/make_golden.py

Inputs are seeded; generators for the Weierstrass curves come from the reference's
fast_random_number_generator{i+1,i+2} -> generate_random_element scheme
(cbindings/pedersen.t.cc:81-123)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import refcpu  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def main():
    rng = np.random.default_rng(20260922)
    n = 96
    for curve in range(4):
        if curve == 0:
            gens = refcpu.ristretto_generators(n, 7)
            gens_p = gens
        else:
            gens_p, gens = refcpu.random_elements(curve, n, first=5)
        cols = [(rng.integers(0, 256, (n, 32), dtype=np.uint8), 0),
                (rng.integers(0, 256, (n - 5, 16), dtype=np.uint8), 1),
                (rng.integers(0, 256, (n, 1), dtype=np.uint8), 0),
                (rng.integers(0, 256, (1, 8), dtype=np.uint8), 1),
                (np.zeros((0, 4), dtype=np.uint8), 0)]
        out = refcpu.commit(curve, cols, gens)
        np.savez_compressed(os.path.join(HERE, f"commit_curve{curve}.npz"), generators=gens,
                            commitments=out, signed=np.array([c[1] for c in cols]),
                            **{f"col{j}": c[0] for j, c in enumerate(cols)})
        m, outs, nb = 24, 3, 4
        sc = rng.integers(0, 256, (m, outs * nb), dtype=np.uint8)
        res = refcpu.fixed_msm(curve, gens_p[:m], outs, m, sc, element_num_bytes=nb)
        bt = [3, 11, 1, 9]
        row = (sum(bt) + 7) // 8
        psc = rng.integers(0, 256, (m, row), dtype=np.uint8)
        pres = refcpu.fixed_msm(curve, gens_p[:m], len(bt), m, psc, output_bit_table=bt)
        np.savez_compressed(os.path.join(HERE, f"fixed_curve{curve}.npz"), generators_p=gens_p[:m],
                            scalars=sc, num_outputs=outs, n=m, element_num_bytes=nb,
                            normalized=refcpu.normalize(curve, res), bit_table=np.array(bt),
                            packed_scalars=psc, packed_normalized=refcpu.normalize(curve, pres))
    g = refcpu.ristretto_generators(16, 1000)
    np.savez_compressed(os.path.join(HERE, "ristretto_generators.npz"), n=16, offset=1000,
                        compressed=refcpu.normalize(0, g))


if __name__ == "__main__":
    main()


def make_inner_product_fixture():
    """tests/golden/inner_product.npz: proofs produced by the reference's cpu backend
    (sxt_curve25519_prove_inner_product semantics) for n = 1, 2, 5, 16, 37 with a transcript
    labelled b"golden-ipa" and generators_offset = 11: inputs, the transcript before / after, the
    proof, <a,b> and the commitment <a, G> that the verifier takes."""
    L = 2**252 + 27742317777372353535851937790883648493
    rng = np.random.default_rng(777)
    out = {}
    cases = [1, 2, 5, 16, 37]
    for ci, n in enumerate(cases):
        av = [int.from_bytes(rng.bytes(32), "little") % L for _ in range(n)]
        bv = [int.from_bytes(rng.bytes(32), "little") % L for _ in range(n)]
        a = np.array([list(v.to_bytes(32, "little")) for v in av], dtype=np.uint8)
        b = np.array([list(v.to_bytes(32, "little")) for v in bv], dtype=np.uint8)
        t0 = refcpu.transcript_new(b"golden-ipa")
        t = t0.copy()
        lv, rv, ap = refcpu.prove_inner_product(t, a, b, generators_offset=11)
        prod = sum(x * y for x, y in zip(av, bv)) % L
        np_ = 1 << max(0, (n - 1).bit_length())
        g = refcpu.ristretto_generators(np_, 11)
        acommit = refcpu.fixed_msm(0, g[:n], 1, n, a, element_num_bytes=32)[0]
        out.update({f"n{ci}": n, f"a{ci}": a, f"b{ci}": b, f"t0_{ci}": t0, f"t1_{ci}": t,
                    f"l{ci}": lv, f"r{ci}": rv, f"ap{ci}": ap,
                    f"product{ci}": np.array(list(prod.to_bytes(32, "little")), dtype=np.uint8),
                    f"acommit{ci}": acommit})
    out["num_cases"] = len(cases)
    out["generators_offset"] = 11
    np.savez_compressed(os.path.join(HERE, "inner_product.npz"), **out)
