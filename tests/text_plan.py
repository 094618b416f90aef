"""The plans the sparse and TF-IDF host drivers (csrc/sparse.cu, csrc/tfidf.cu, csrc/shard_group.cu) choose from the shape
of a request, restated in Python: merge-group widths, merge-tree levels, query chunks and the kernel launches each search
makes.  tests/test_text_plan.py pins the constants to the sources; tests/test_gpu_text_limits.py asserts that every case
launches exactly the plan it names, so no case can quietly take a shallower path."""
import os
import re

_CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "cosdata_b200", "csrc")

SP_MERGE_KEYS = 25600          # keys a merge CTA holds in shared memory
SP_MERGE_MAX_LISTS = 63        # lists a merge CTA takes at once
SP_MAX_CAND = 5120             # k * reranking_factor, at most
SP_QCHUNK = 512                # query pairs per pass of sp_score_tile_kernel
TF_QCHUNK = 512                # query terms per pass of tf_score_tile_kernel
TF_BUCKETS = 512
TILE_SHIFT = 15
TILE_ROWS = 1 << TILE_SHIFT
SCRATCH_BUDGET = 512 << 20     # device scratch of one chunk of a single-index search
GROUP_GATHER_BUDGET = 256 << 20
MAX_GRID_Y = 65535             # a chunk is one grid's y dimension


def source_constants():
    """the constants above as the sources define them: name -> int"""
    want = {"SP_THREADS": "sparse.cu", "SP_MERGE_KEYS": "sparse.cu", "SP_MERGE_MAX_LISTS": "sparse.cu", "SP_MAX_CAND": "sparse.cu",
            "SP_QCHUNK": "sparse.cu", "TF_THREADS": "tfidf.cu", "TF_QCHUNK": "tfidf.cu", "TF_BUCKETS": "tfidf.cu",
            "TILE_SHIFT": "posting_tiles.cuh", "GROUP_GATHER_BUDGET": "shard_group.cu"}
    got = {}
    for name, f in want.items():
        with open(os.path.join(_CSRC, f)) as fh:
            src = fh.read()
        m = re.search(r"constexpr\s+(?:u?int\w*|size_t)\s+" + name + r"\s*=\s*([^;/]+);", src)
        assert m, f"{name} not found in {f}"
        got[name] = m.group(1).strip()
    # resolve the `SP_QCHUNK = SP_THREADS` aliases (defined earlier in `want`) and `256ull << 20` forms
    out = {}
    for name, expr in got.items():
        e = expr
        for other, v in out.items():
            e = re.sub(r"\b" + other + r"\b", str(v), e)
        e = re.sub(r"(\d+)(?:ull|ul|u|ll)\b", r"\1", e)
        assert re.fullmatch(r"[\d\s<>()*+]+", e), f"{name} = {expr}"
        out[name] = int(eval(e))
    return out


def ceil_div(a, b):
    return -(-a // b)


# ----------------------------------------------------------------------------- sparse
def merge_group(m):
    """lists a merge CTA takes: as many m-key lists as fit in its shared memory, 2..63"""
    return min(SP_MERGE_MAX_LISTS, max(2, SP_MERGE_KEYS // m))


def tree_levels(n_tiles, m):
    """search_locked's merge tree over the tile lists: the list count after each level (none for one tile)"""
    g, n, out = merge_group(m), n_tiles, []
    while n > 1:
        n = ceil_div(n, g)
        out.append(n)
    return out


def merge_lists_levels(n_lists, m):
    """merge_lists (a shard's tiles, a group's ranks): like tree_levels, but at least one level, so one list is copied"""
    g, n, out = merge_group(m), n_lists, []
    while True:
        n = ceil_div(n, g)
        out.append(n)
        if n == 1:
            return out


def sparse_chunk(nq, n_tiles, m):
    """queries per chunk of search_locked: the tile lists and the first merge level of a chunk fit the scratch budget"""
    n1 = ceil_div(n_tiles, merge_group(m))
    per_q = (n_tiles + n1) * m * 8 + (n_tiles + n1) * 4
    return max(1, min(nq, MAX_GRID_Y, SCRATCH_BUDGET // per_q))


def chunks(nq, chunk):
    """the chunk sizes of a batch of nq queries"""
    return [min(chunk, nq - q0) for q0 in range(0, nq, chunk)]


def sparse_launches(nq, n_tiles, m):
    """kernel launches of one top-k search: per chunk the scoring kernel, one merge per level, the finalize kernel"""
    if nq == 0 or n_tiles == 0:
        return 0                            # an empty index: memsets only
    return len(chunks(nq, sparse_chunk(nq, n_tiles, m))) * (1 + len(tree_levels(n_tiles, m)) + 1)


def shard_select_chunk(nq, n_tiles, m):
    """queries per chunk of sparse_shard_select (a shard group's phase 1): the tile lists only"""
    return max(1, min(nq, MAX_GRID_Y, SCRATCH_BUDGET // (n_tiles * m * 12)))


def group_chunk(nq, world, per_q):
    """queries per chunk of a shard group's search: every rank's slot of the gather buffer fits its budget"""
    return max(1, min(nq, MAX_GRID_Y, GROUP_GATHER_BUDGET // (world * per_q)))


def sparse_group_launches(nq, shard_tiles, m, rerank):
    """kernel launches of one top-k search over a one-process group of len(shard_tiles) slots (loopback or not, one
    selection on slot 0 in loopback): per group chunk, every non-empty shard's scoring chunks each with its merge_lists
    levels, the group's selection over the ranks, with re-rank one re-rank kernel per shard and the OR of the ranks, and
    the finalize kernel"""
    world = len(shard_tiles)
    total = 0
    for c in chunks(nq, group_chunk(nq, world, m * 8 + 4)):
        for t in shard_tiles:
            if t:
                total += len(chunks(c, shard_select_chunk(c, t, m))) * (1 + len(merge_lists_levels(t, m)))
        total += len(merge_lists_levels(world, m))
        total += (world + 1 if rerank else 0) + 1
    return total


# ----------------------------------------------------------------------------- TF-IDF
def tfidf_chunk(nq, n_tiles):
    """queries per chunk of a TF-IDF search: every tile's 512 bucket winners of a chunk fit the scratch budget"""
    return max(1, min(nq, MAX_GRID_Y, SCRATCH_BUDGET // (n_tiles * TF_BUCKETS * 8)))


def tfidf_launches(nq, n_tiles):
    """per chunk the scoring kernel and the finalize kernel"""
    if nq == 0 or n_tiles == 0:
        return 0
    return len(chunks(nq, tfidf_chunk(nq, n_tiles))) * 2


def tfidf_group_launches(nq, shard_tiles):
    """per group chunk: every non-empty shard's scoring and winner kernels per its own chunk, and the group finalize"""
    total = 0
    for c in chunks(nq, group_chunk(nq, len(shard_tiles), TF_BUCKETS * 8)):
        for t in shard_tiles:
            if t:
                total += len(chunks(c, tfidf_chunk(c, t))) * 2
        total += 1
    return total


def tfidf_group_search_launches(nq, shard_tiles, n_hashes, loopback):
    """one sharded TF-IDF search, host or device form: a statistics kernel per local slot, the idf kernel (when the batch
    has a query term) on every local slot, or on slot 0 alone in a loopback group, then tfidf_group_launches; nothing for
    an empty batch"""
    if nq == 0:
        return 0
    n = len(shard_tiles)
    return n + (0 if not n_hashes else 1 if loopback else n) + tfidf_group_launches(nq, shard_tiles)


def n_tiles(n_rows):
    return ceil_div(n_rows, TILE_ROWS)
