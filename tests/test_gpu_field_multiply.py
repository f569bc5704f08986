"""The curve25519 field multiplier as the device runs it (the carry-chain PTX of F25519::mul, whose
2^256 = 38 fold is a shift-and-add chain) against the plain 64-bit reference schedule mul_ref, limb
for limb, on pseudo-random and edge-case operands. The CPU emulation checks the same schedule with
emulated carries; this checks the real instructions."""
import pytest

pytestmark = pytest.mark.gpu


def test_field_multiply_selftest(bb):
    for seed in (1, 2, 3):
        assert bb.selftest_field_multiply(1 << 18, seed) == 0, seed
