"""blitzar_b200 — H100-native MSM / Pedersen-commitment backend behind Blitzar's C ABI.

The product is blitzar_b200/lib/libblitzar_b200.so (hand-written sm_90a CUDA + C++ host);
this package is only the thin ctypes mirror of the C ABI used by the tests and bench.py.
"""
from .api import *  # noqa: F401,F403
