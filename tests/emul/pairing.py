"""TEST INFRASTRUCTURE — Python side of the emulated pairing entry (tests/emul/emul_pairing.cpp), in the
library of the emulation harness (tests/emul/harness.py), with the name of the product's Python API so
that tests can run the same checks on both."""
from blitzar_b200.api import call_multi_pairing
from tests.emul import harness


def multi_pairing(curve_id, g1_p2, g2_p2, lengths):
    """emul_multi_pairing: b200_multi_pairing's contract (blitzar_b200.api.call_multi_pairing) on the
    CPU."""
    return call_multi_pairing(harness.lib().emul_multi_pairing, curve_id, g1_p2, g2_p2, lengths)
