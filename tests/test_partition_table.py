"""The reference's partition-table format, built by the product's kernel bodies run as serial host
loops (tests/emul): every fixture case of tests/golden/ptable_curve{c}.npz and ref_table_curve{c}_w3.bin
(written by the reference's own code) is reproduced byte for byte on bls12-381 / bn254 / grumpkin and
value for value on ristretto255, in one chunk and in many; the table's generators read back."""
import os

import numpy as np
import pytest

from tests import partition_tables as pt

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
def test_reference_w3_file_is_reproduced(emul, curve):
    g7 = np.load(os.path.join(GOLDEN, f"fixed_curve{curve}.npz"))["generators_p"][:7]
    ref = np.fromfile(os.path.join(GOLDEN, f"ref_table_curve{curve}_w3.bin"), dtype=np.uint8)
    assert int(ref[:4].view("<u4")[0]) == 3
    got = emul.partition_table(curve, g7, 3)
    want = pt.canonicalise_ristretto_table(ref[4:]) if curve == 0 else ref[4:]
    assert np.array_equal(got, want)
    assert np.array_equal(emul.partition_table(curve, g7, 3, chunk_groups=1), got)


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
@pytest.mark.parametrize("case", list(pt.CASES))
def test_fixture_digests(emul, curve, case):
    z = np.load(os.path.join(GOLDEN, f"ptable_curve{curve}.npz"))
    gens = z[f"gens_{case}"]
    _, w, _ = pt.CASES[case]
    got = emul.partition_table(curve, gens, w)
    # the device writes canonical limbs: its raw bytes already carry the canonicalised digest
    assert pt.table_digest(curve, got) == str(z[f"sha_{case}"])
    assert pt.sha256(got) == str(z[f"sha_{case}"])
    if w < 16:
        assert np.array_equal(emul.partition_table(curve, gens, w, chunk_groups=3), got)


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
def test_generators_read_back(emul, port, curve, tmp_path):
    """Entry 1 << j of group g is generator g w + j: the reader of reference handle files recovers
    the generators (the padding of the last group reads back as the identity)."""
    z = np.load(os.path.join(GOLDEN, f"ptable_curve{curve}.npz"))
    for case in ("n37_w8", "n24_w6_edited"):
        gens = z[f"gens_{case}"]
        _, w, _ = pt.CASES[case]
        path = str(tmp_path / f"{case}.bin")
        with open(path, "wb") as f:
            f.write(np.uint32(w).tobytes())
            f.write(emul.partition_table(curve, gens, w).tobytes())
        back = emul.generators_from_reference_table(curve, path)
        n = gens.shape[0]
        assert back.shape[0] == -(-n // w) * w
        assert np.array_equal(port.normalize(curve, back[:n]), port.normalize(curve, gens)), case
