"""The plan of a top_k None sparse search (csrc/sparse.cu sparse_all_chunk, csrc/shard_group.cu sparse_all_sharded_run),
restated in Python: scoring chunks from the largest shard's tiles and live rows, the key exchange's sub-batches from the
gathered counts (cosdata_b200.sharding.key_batches), and the kernel launches a group search makes.
tests/test_sparse_all_sharded_abi.py pins the budget to the source."""
from cosdata_b200.sharding import key_batches
from tests.text_plan import GROUP_GATHER_BUDGET, MAX_GRID_Y, TILE_ROWS, chunks

SP_ALL_BUDGET = 512 << 20      # device scratch of one scoring chunk of a top_k None search


def all_chunk(nq, n_tiles, n_live):
    """queries per scoring chunk over at most n_tiles tiles and n_live live rows"""
    per_q = n_tiles * TILE_ROWS * 8 + n_tiles * 8 + n_live * 24
    return max(1, min(nq, MAX_GRID_Y, SP_ALL_BUDGET // max(per_q, 1)))


def group_plan(counts, shard_bounds):
    """counts: [world, nq] candidates of every (rank, query); shard_bounds: (tiles, live rows) per rank ->
    (chunk sizes, [sub-batches of each chunk]); no chunk when no rank has a tile and a live row"""
    nq = counts.shape[1]
    t = max(b[0] for b in shard_bounds)
    live = max(b[1] for b in shard_bounds)
    if not nq or not t or not live:
        return [], []
    sizes = chunks(nq, all_chunk(nq, t, live))
    batches, q0 = [], 0
    for c in sizes:
        batches.append(key_batches(counts[:, q0:q0 + c], GROUP_GATHER_BUDGET))
        q0 += c
    return sizes, batches


def group_launches(counts, shard_bounds, rerank):
    """kernel launches of one group search (counted ones: the scoring and gather kernels of every shard with a tile and a
    live row, its re-rank when the chunk gave it a candidate, and one merge per sub-batch)"""
    sizes, batches = group_plan(counts, shard_bounds)
    total, q0 = 0, 0
    for c, kb in zip(sizes, batches):
        for r, (t, live) in enumerate(shard_bounds):
            if t and live:
                total += 2 + (1 if rerank and counts[r, q0:q0 + c].sum() else 0)
        total += len(kb)
        q0 += c
    return total
