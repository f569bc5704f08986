"""Binned bucket sort against the atomic sort at the coarse scatter's tile boundaries (msm.cuh,
CoarseScatterBody): a tile stages tile x W entries, W = the column's windows, in the shared memory left
by its two per-bin arrays of nmicro counters, in whole rounds of its 1024 threads. Shapes just below,
at and above a tile,
a column whose every entry falls in one bucket (every tile writes one run into one bin, and that bin
is sorted out of global memory), a boolean column (one window, the longest tile), and buckets of
exactly kBinCap and kBinCap + 1 entries (sorted in shared memory at the limit, and out of global
memory just above it)."""
import numpy as np
import pytest

from tests.test_gpu_sort import _selftest

pytestmark = pytest.mark.gpu
SCATTER_SMEM = 220 * 1024  # binned_sort: shared memory of a coarse-scatter block
MICRO_BINS = 16384         # kMicroBins
BLOCK = 1024               # CoarseScatterBody::kBlock
CAP = 16384                # kBinCap


def scatter_tile(nkeys, windows):
    shift = 0
    while (nkeys + (1 << shift) - 1) >> shift > MICRO_BINS:
        shift += 1
    nmicro = (nkeys + (1 << shift) - 1) >> shift
    tile = (SCATTER_SMEM - (2 * nmicro + 2) * 4) // 8 // windows
    return tile - tile % BLOCK if tile > BLOCK else tile


C = 16
WIDE = scatter_tile(17 << (C - 1), 17)  # 32-byte scalars: 256 / 16 + 1 windows
BOOL = scatter_tile(1 << (C - 1), 1)    # 1-byte scalars: one window


def _shapes():
    rng = np.random.default_rng(9)
    ones = np.zeros((1 << 20, 32), dtype=np.uint8)
    ones[:, 0] = 1  # digit 1 in window 0: every entry in bucket 0
    shapes = {"single_bucket": ([(ones, 0)], C)}
    for k, n in (("below", 3 * WIDE - 1), ("at", 3 * WIDE), ("above", 3 * WIDE + 1)):
        shapes[f"wide_{k}_tile"] = ([(rng.integers(0, 256, (n, 32), dtype=np.uint8), 0)], C)
    for k, n in (("below", BOOL - 1), ("at", BOOL), ("above", BOOL + 1)):
        shapes[f"boolean_{k}_tile"] = ([(rng.integers(0, 2, (n, 1), dtype=np.uint8), 0)], C)
    # as test_gpu_sort's cap shape, at this cap: window 0 of c = 16, bucket 999 holds CAP entries and
    # bucket 1999 CAP + 1, the rest of their micro-bins empty
    vals = rng.integers(1, 1 << 15, 1 << 17)
    vals[((vals >= 993) & (vals <= 1004)) | ((vals >= 1993) & (vals <= 2004))] = 5
    vals[:CAP] = 1000
    vals[CAP:2 * CAP + 1] = 2000
    rng.shuffle(vals)
    u16 = np.ascontiguousarray(vals.astype("<u2").view(np.uint8).reshape(-1, 2))
    shapes["cap_and_cap_plus_1"] = ([(u16, 0)], C)
    return shapes


@pytest.mark.parametrize("name", list(_shapes()))
def test_binned_sort_at_tile_boundaries(bb, name):
    columns, c = _shapes()[name]
    assert _selftest(bb, columns, c) == 0
