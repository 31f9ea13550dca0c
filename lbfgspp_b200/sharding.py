"""Host-side logic of the n-sharded (multi-GPU) mode -- no device code here.

Rank r of N owns the contiguous block [lo, hi) of every n-vector and of every S/Y column; all scalars are replicated.
Blocks are even-length (the paired Rosenbrock couples coordinates (2i, 2i+1)) and 4-aligned where possible so that
every shard keeps the 4-element pack access path.  A reduction is: local deterministic partial -> sum over ranks in rank order
(NCCL all-reduce on the GPU; tests use gloo) -> identical scalar on every rank -> identical host decisions everywhere.
"""


def shard_bounds(n, rank, nranks, granule=4):
    """[lo, hi) of `rank`; sizes differ by at most one granule; the last rank takes the ragged tail."""
    if nranks < 1 or not (0 <= rank < nranks):
        raise ValueError("bad rank/nranks")
    units = n // granule
    base, extra = divmod(units, nranks)
    lo_u = rank * base + min(rank, extra)
    hi_u = lo_u + base + (1 if rank < extra else 0)
    lo, hi = lo_u * granule, hi_u * granule
    if rank == nranks - 1:
        hi = n
    return lo, hi


def all_shards(n, nranks, granule=4):
    return [shard_bounds(n, r, nranks, granule) for r in range(nranks)]


def collectives_per_iteration(trials, c, algo="gram"):
    """Number of scalar all-reduces one L-BFGS iteration issues (DESIGN.md section 6)."""
    hv = 2 if algo == "gram" else (2 * c + 1)   # gram: dots + v.res ; two-loop: one per stage
    return trials + 1 + (hv if c > 0 else 1)
