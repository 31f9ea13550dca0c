"""CPU tests of the multi-GPU host logic: shard geometry, and a world_size-2 gloo run showing that the sharded reductions
(local partial + all-reduce) reproduce the unsharded scalars that drive the line search."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from lbfgspp_b200.sharding import all_shards, collectives_per_iteration, shard_bounds

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("n", [2, 8, 10, 1000, 10_000_000, 1_000_003])
@pytest.mark.parametrize("nranks", [1, 2, 3, 4, 8])
def test_shards_tile_the_vector(n, nranks):
    sh = all_shards(n, nranks)
    assert sh[0][0] == 0 and sh[-1][1] == n
    for (lo, hi), (lo2, _) in zip(sh, sh[1:]):
        assert hi == lo2 and lo <= hi
    for lo, hi in sh[:-1]:
        assert lo % 4 == 0 and hi % 4 == 0          # 4-element packs and Rosenbrock pairs stay intact
    sizes = [hi - lo for lo, hi in sh[:-1]]
    if sizes:
        assert max(sizes) - min(sizes) <= 4


def test_bad_rank_rejected():
    with pytest.raises(ValueError):
        shard_bounds(10, 2, 2)


def test_collective_counts():
    assert collectives_per_iteration(1, 10, "gram") == 4
    assert collectives_per_iteration(2, 10, "two_loop") == 2 + 1 + 21
    assert collectives_per_iteration(1, 0) == 3


def _worker(rank, world, port, n, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import pyoracle as po
    orc = po.Oracle("orc")
    rng = np.random.default_rng(0)                    # same stream on every rank: replicated inputs
    xp = rng.uniform(-1, 1, n)
    d = rng.standard_normal(n)
    step = 0.25
    lo, hi = shard_bounds(n, rank, world)
    x = xp[lo:hi] + step * d[lo:hi]                   # local part of the trial point
    f_loc, g_loc = orc.objective(po.OBJ_ROSENBROCK_PAIRED, x)   # paired objective: shards are independent
    part = torch.tensor([f_loc, float(np.dot(g_loc, d[lo:hi])), float(np.dot(g_loc, g_loc)), float(np.dot(x, x))],
                        dtype=torch.float64)
    dist.all_reduce(part)                             # the {f, g.d, g.g, x.x} all-reduce of one trial
    if rank == 0:
        f, g = orc.objective(po.OBJ_ROSENBROCK_PAIRED, xp + step * d)
        full = np.array([f, np.dot(g, d), np.dot(g, g), np.dot(xp + step * d, xp + step * d)])
        out.put((part.numpy().copy(), full))
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_trial_scalars_match_unsharded_gloo_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    n = 100_000
    port = 29600 + os.getpid() % 300
    procs = [ctx.Process(target=_worker, args=(r, 2, port, n, q)) for r in range(2)]
    for p in procs:
        p.start()
    got, full = q.get(timeout=120)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert np.allclose(got, full, rtol=1e-12, atol=0)
