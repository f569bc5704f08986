"""TEST INFRASTRUCTURE — Python side of the emulated point checks (tests/emul/emul_points.cpp), in the
library of the emulation harness (tests/emul/harness.py), with the names of the product's Python API so
that tests can run the same checks on both. Each call returns what the product's call does, plus the
count the C entry returned."""
from blitzar_b200.api import call_check_points, call_decode_points
from tests.emul import harness


def check_points(curve_id, p2):
    """emul_check_points: (valid uint8 [n], count)."""
    return call_check_points(harness.lib().emul_check_points, curve_id, p2)


def decode_points(curve_id, encoded):
    """emul_decode_points: (p2 uint8 [n, projective bytes], valid uint8 [n], count)."""
    return call_decode_points(harness.lib().emul_decode_points, curve_id, encoded)
