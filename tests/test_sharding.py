"""Multi-GPU host logic on CPU: world_size-2 gloo run of the generator-range sharding
(blitzar_b200/sharding.py) with the emulation harness standing in for the kernels."""
import os
import socket
import sys

import numpy as np
import pytest

from tests import common


def test_shard_ranges_cover_and_balance():
    from blitzar_b200.sharding import shard_range
    for n in (0, 1, 7, 8, 1000, 2**20 + 3):
        for ws in (1, 2, 3, 8):
            r = [shard_range(n, k, ws) for k in range(ws)]
            assert r[0][0] == 0 and r[-1][1] == n
            assert all(r[k][1] == r[k + 1][0] for k in range(ws - 1))
            sizes = [e - b for b, e in r]
            assert max(sizes) - min(sizes) <= 1


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world_size, port_no, curve, out_queue):
    sys.path.insert(0, common.ROOT)
    import torch
    import torch.distributed as dist
    from blitzar_b200.sharding import sharded_commit
    from oracle import port
    from tests.emul import harness
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port_no)
    dist.init_process_group("gloo", rank=rank, world_size=world_size)
    rng = np.random.default_rng(77)  # same inputs on every rank
    n = 333
    gens, _ = common.generators_for(port, curve, n)
    cols = common.random_columns(rng, n, [(0, 32, 0), (-100, 16, 1), (-332, 8, 0)])

    def all_gather(x):
        t = torch.from_numpy(x.copy())
        outs = [torch.empty_like(t) for _ in range(world_size)]
        dist.all_gather(outs, t)
        return torch.stack(outs).numpy()

    got = sharded_commit(
        cols, gens, rank, world_size, harness.point_bytes(curve),
        partial_fn=lambda c, g, first: harness.commit_partial(curve, c, g),
        combine_fn=lambda p, parts, count: harness.combine_partials(curve, p, parts, count),
        all_gather_fn=all_gather)
    want = port.commit(curve, cols, gens)
    out_queue.put((rank, bool(common.same(curve, got, want))))
    dist.destroy_process_group()


@pytest.mark.parametrize("curve", [0, 2])
def test_two_rank_gloo_sharded_commit(curve):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port_no = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port_no, curve, q)) for r in range(2)]
    for p in procs:
        p.start()
    results = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(results) == [(0, True), (1, True)]
