"""Row-sharding of a corpus over the GPUs of one node (SURVEY.md 8e).

The reference is single-process; the natural multi-GPU form is one index shard per GPU (contiguous id ranges), the same
query batch on every shard, a local search, ONE all-gather of the per-shard top-k as packed 64-bit keys
(order_key(score) << 32 | ~global_id; B*k*8 bytes per rank, latency bound on NVLink) and a k-way merge with the common
ordering rule (better score, then smaller id).  On GPUs all of that lives behind the C ABI (`ShardGroup` ->
cdb_shard_group_*, cdb_search_batch_sharded*: csrc/shard_group.cu, NCCL owned by the library).  The numpy functions
below restate the key layout and the merge so the host logic can be exercised on CPU with gloo (tests/test_sharding_gloo.py).
"""
import ctypes as C

import numpy as np

INVALID_ID = 0xFFFFFFFF
NCCL_UNIQUE_ID_BYTES = 128


def shard_range(n_rows, world, rank):
    """contiguous row range [row0, row0+n) of `rank`; sizes differ by at most one row"""
    base, rem = divmod(int(n_rows), int(world))
    n = base + (1 if rank < rem else 0)
    row0 = rank * base + min(rank, rem)
    return row0, n


# ----------------------------------------------------------------------------- key layout (host mirror of common.cuh)
def order_key_np(metric, score_bits):
    """f32::total_cmp as an unsigned key; distance-like metrics (1 Euclidean, 2 Hamming) reversed: larger = better"""
    b = np.asarray(score_bits, dtype=np.uint32)
    key = np.where(b & np.uint32(0x80000000), ~b, b | np.uint32(0x80000000)).astype(np.uint32)
    return (~key).astype(np.uint32) if metric in (1, 2) else key


def pack_keys(ids, scores, metric=0):
    """[.., k] global ids (u32, INVALID_ID = empty) + f32 scores -> u64 selection keys (0 = empty)"""
    ids = np.asarray(ids, dtype=np.uint32)
    ok = order_key_np(metric, np.ascontiguousarray(scores, dtype=np.float32).view(np.uint32)).astype(np.uint64)
    keys = (ok << np.uint64(32)) | (~ids).astype(np.uint64)
    return np.where(ids == INVALID_ID, np.uint64(0), keys).astype(np.uint64)


def unpack_keys(keys, metric=0):
    keys = np.asarray(keys, dtype=np.uint64)
    ids = (~(keys & np.uint64(0xFFFFFFFF)).astype(np.uint32)).astype(np.uint32)
    k32 = (keys >> np.uint64(32)).astype(np.uint32)
    if metric in (1, 2):
        k32 = ~k32
    bits = np.where(k32 & np.uint32(0x80000000), k32 & np.uint32(0x7FFFFFFF), ~k32).astype(np.uint32)
    ids = np.where(keys == 0, np.uint32(INVALID_ID), ids)
    scores = np.where(keys == 0, np.float32(0), bits.view(np.float32))
    return ids.astype(np.uint32), scores.astype(np.float32)


def merge_packed(gathered, k, metric=0):
    """gathered: [world, B, k] keys (the all-gather result) -> (ids[B,k], scores[B,k], counts[B]); keys are unique"""
    world, b, kk = gathered.shape
    allk = np.transpose(gathered, (1, 0, 2)).reshape(b, world * kk)
    order = np.argsort(allk, axis=1)[:, ::-1][:, :k]                  # u64 keys: descending
    best = np.take_along_axis(allk, order, axis=1)
    ids, scores = unpack_keys(best, metric)
    return ids, scores, (best != 0).sum(axis=1).astype(np.uint32)


def merge_runs(gathered, metric=0):
    """the top_k None merge of the sharded dense search.  gathered: [world, B, w] keys, every rank's whole sorted list
    (descending, unique, zero padded) -> (ids u32[B, world*w], scores f32[B, world*w], counts u32[B]).  An entry's position
    is its index in its run plus, for every other run, the number of that run's keys greater than it."""
    gathered = np.asarray(gathered, dtype=np.uint64)
    world, b, w = gathered.shape
    out = np.zeros((b, world * w), np.uint64)
    for q in range(b):
        runs = [gathered[r, q][gathered[r, q] != 0] for r in range(world)]
        asc = [np.sort(x) for x in runs]
        for r, x in enumerate(runs):
            pos = np.arange(len(x), dtype=np.int64)
            for o in range(world):
                if o != r:
                    pos += len(asc[o]) - np.searchsorted(asc[o], x, side="right")
            out[q, pos] = x
    ids, scores = unpack_keys(out, metric)
    return ids, scores, (out != 0).sum(axis=1).astype(np.uint32)


def gather_and_merge(local_ids, local_scores, world, all_gather_fn, k=None, metric=0):
    """host logic of the sharded search: pack -> ONE all-gather of B*k u64 -> merge.
    all_gather_fn(x: u64[B,k]) -> u64[world,B,k] stacked over ranks."""
    keys = pack_keys(local_ids, local_scores, metric)
    k = keys.shape[1] if k is None else k
    if world == 1:
        return merge_packed(keys[None], k, metric)[:2]
    return merge_packed(all_gather_fn(keys), k, metric)[:2]


# ----------------------------------------------------------------------------- sparse and TF-IDF shards (host mirrors)
def sparse_keys(ids, sims):
    """[.., m] global ids (INVALID_ID = empty) + u32 similarities -> u64 selection keys sim << 32 | ~id (0 = empty)"""
    ids = np.asarray(ids, dtype=np.uint32)
    keys = (np.asarray(sims, dtype=np.uint64) << np.uint64(32)) | (~ids).astype(np.uint64)
    return np.where(ids == INVALID_ID, np.uint64(0), keys).astype(np.uint64)


def _key_ids(keys):
    return (~(keys & np.uint64(0xFFFFFFFF)).astype(np.uint32)).astype(np.uint32)


def merge_sparse(gathered, k, rerank_fn=None):
    """cdb_sparse_search_batch_sharded's merge.  gathered: [world, B, m] u64 keys, every rank's top m (all-gather #1).
    The group's top m per query are the best m of the world * m keys.  Without rerank_fn (m = k) they are the results,
    scored by similarity as f32.  With rerank_fn(q, ids) -> f32 dot products of those global ids for query q (each rank
    re-ranks the ids it owns; here one function stands for all of them), the m candidates are rekeyed by the total_cmp
    order of the dp (NaN canonicalised) then the smaller id, and the best k kept.
    -> (ids u32[B, k], scores f32[B, k], counts u32[B])"""
    world, b, m = gathered.shape
    allk = np.transpose(gathered, (1, 0, 2)).reshape(b, world * m)
    top = np.take_along_axis(allk, np.argsort(allk, axis=1)[:, ::-1][:, :m], axis=1)
    ids = np.full((b, k), INVALID_ID, np.uint32)
    scores = np.zeros((b, k), np.float32)
    counts = np.zeros(b, np.uint32)
    for q in range(b):
        cand = top[q][top[q] != 0]
        if rerank_fn is None:
            best = cand[:k]
            ids[q, :len(best)] = _key_ids(best)
            scores[q, :len(best)] = (best >> np.uint64(32)).astype(np.float64).astype(np.float32)
        else:
            cid = _key_ids(cand)
            dp = np.asarray(rerank_fn(q, cid), dtype=np.float32).reshape(-1)
            dbits = np.where(np.isnan(dp), np.uint32(0xFFC00000), dp.view(np.uint32)).astype(np.uint32)
            rk = (order_key_np(0, dbits).astype(np.uint64) << np.uint64(32)) | (~cid).astype(np.uint64)
            best = np.sort(rk)[::-1][:k]
            ids[q, :len(best)], scores[q, :len(best)] = unpack_keys(best)
        counts[q] = len(best)
    return ids, scores, counts


def merge_runs_var(keys, counts):
    """the top_k None merge of the sharded sparse search.  keys[r]: rank r's sorted keys of a batch of queries, query after
    query (descending within a query, unique across ranks); counts: u32[world, B], rank r's keys of each query.  ->
    (offsets u64[B+1], merged keys u64[total]).  An entry's position is its query's output offset, plus its index in its
    run, plus for every other rank the number of that rank's keys of the query greater than it."""
    counts = np.asarray(counts, dtype=np.int64)
    world, b = counts.shape
    pre = np.zeros((world, b + 1), np.int64)
    pre[:, 1:] = np.cumsum(counts, axis=1)
    offsets = np.zeros(b + 1, np.uint64)
    offsets[1:] = np.cumsum(counts.sum(axis=0))
    out = np.zeros(int(offsets[-1]), np.uint64)
    for q in range(b):
        runs = [np.asarray(keys[r], dtype=np.uint64)[pre[r, q]:pre[r, q + 1]] for r in range(world)]
        asc = [np.sort(x) for x in runs]
        for r, x in enumerate(runs):
            pos = int(offsets[q]) + np.arange(len(x), dtype=np.int64)
            for o in range(world):
                if o != r:
                    pos += len(asc[o]) - np.searchsorted(asc[o], x, side="right")
            out[pos] = x
    return offsets, out


def key_batches(counts, budget=256 << 20):
    """the key exchange of one scoring chunk of a sharded top_k None sparse search, from the all-gathered counts
    u32[world, c] alone: consecutive queries [a, b) whose largest rank total `words` keeps world * words * 8 bytes within
    the budget (at least one query each), sub-batches without a key dropped -> [(a, b, words)]"""
    counts = np.asarray(counts, dtype=np.int64)
    world, c = counts.shape
    cap = budget // (8 * world)
    out, a = [], 0
    while a < c:
        tot, words, b = np.zeros(world, np.int64), 0, a
        while b < c:
            w = int((tot + counts[:, b]).max())
            if b > a and w > cap:
                break
            tot += counts[:, b]
            words, b = w, b + 1
        if words:
            out.append((a, b, words))
        a = b
    return out


def merge_buckets(g_ids, g_scores, k=0):
    """cdb_tfidf_search_batch_sharded's merge.  g_ids / g_scores: [world, B, 512] every rank's bucket winners
    (INVALID_ID = empty bucket; all-gathered).  Per bucket the best of the ranks by `score > best`, equal scores (+0 and -0
    too) going to the smaller id; the winners sorted by total_cmp descending, ties to the smaller id, truncated to
    kout = 512 for k = 0 or k > 512, else k.  -> (ids u32[B, kout], scores f32[B, kout], counts u32[B])"""
    g_ids = np.asarray(g_ids, dtype=np.uint32)
    g_scores = np.asarray(g_scores, dtype=np.float32)
    world, b, nb = g_ids.shape
    kout = nb if k == 0 or k > nb else k
    best = np.full((b, nb), -np.inf, np.float32)
    bid = np.full((b, nb), INVALID_ID, np.uint32)
    for r in range(world):
        i, s = g_ids[r], g_scores[r]
        take = (i != INVALID_ID) & ((s > best) | ((s == best) & (i < bid)))
        best = np.where(take, s, best)
        bid = np.where(take, i, bid)
    keys = pack_keys(bid, best)
    top = np.take_along_axis(keys, np.argsort(keys, axis=1)[:, ::-1][:, :kout], axis=1)
    ids, scores = unpack_keys(top)
    return ids, scores, (top != 0).sum(axis=1).astype(np.uint32)


# ----------------------------------------------------------------------------- C ABI wrapper
class ShardGroup:
    """cdb_shard_group: the NCCL communicator + gather buffers owned by the library."""

    def __init__(self, handle, lib):
        self._h, self._lib = handle, lib
        self._shards = []
        self._ranks_elsewhere = False        # a per-rank group of world > 1: the other ranks' shards are not visible here
        self._text_shards = []              # sparse and TF-IDF shards, kept alive as long as the group

    @staticmethod
    def unique_id():
        from . import _lib
        from .api import _check
        buf = (C.c_uint8 * NCCL_UNIQUE_ID_BYTES)()
        _check(_lib.load().cdb_nccl_unique_id(buf))
        return bytes(buf)

    @classmethod
    def local(cls, devices):
        """one process driving len(devices) GPUs (a device listed twice -> copy-based loopback gather, single-GPU tests)"""
        from . import _lib
        from .api import _check
        lib = _lib.load()
        arr = (C.c_int32 * len(devices))(*devices)
        h = C.c_void_p()
        _check(lib.cdb_shard_group_create(arr, len(devices), C.byref(h)))
        return cls(h, lib)

    @classmethod
    def rank(cls, unique_id, world, rank, device):
        """one process per GPU; every rank passes the id rank 0 created (None when world == 1)"""
        from . import _lib
        from .api import _check
        lib = _lib.load()
        buf = (C.c_uint8 * NCCL_UNIQUE_ID_BYTES).from_buffer_copy(unique_id) if unique_id is not None else None
        h = C.c_void_p()
        _check(lib.cdb_shard_group_create_rank(buf, world, rank, device, C.byref(h)))
        g = cls(h, lib)
        g._ranks_elsewhere = world > 1
        return g

    @property
    def world(self):
        return int(self._lib.cdb_shard_group_world(self._h))

    def attach(self, local_slot, index):
        from .api import _check
        _check(self._lib.cdb_shard_group_attach(self._h, local_slot, index._h))
        self._shards.append(index)          # keep the shard alive as long as the group

    def all_width(self, width=None):
        """row width W of a top_k None search over this group.  Every rank must pass the same W, a multiple of the world size
        with W / world >= every shard's (num_levels + 1) * 100: ranks that disagree run all-gathers of different sizes, and a
        rank that refuses leaves the others waiting in theirs.  A local group sees every shard, so W defaults to world * the
        largest (num_levels + 1) * 100; a per-rank group of more than one rank must pass `width` (the same on every rank)."""
        if width is not None:
            return int(width)
        if self._ranks_elsewhere:
            raise ValueError("a per-rank group's top_k None search needs width= (the same W on every rank)")
        return self.world * max(s.hnsw_out_cap() for s in self._shards)

    def search(self, queries, k, mode=0, width=None, **kw):
        """host queries -> merged (ids u32[B,k], scores f32[B,k], counts u32[B], err u8[B]).
        k=None (top_k None, HNSW): every shard's candidates, merged best first, in rows of all_width(width) columns"""
        from .api import _check, _ptr
        q = np.ascontiguousarray(queries, dtype=np.float32)
        b = q.shape[0]
        if k is None:
            k, kw["all_candidates"] = self.all_width(width), True
        ids = np.zeros((b, k), dtype=np.uint32)
        scores = np.zeros((b, k), dtype=np.float32)
        counts = np.zeros(b, dtype=np.uint32)
        err = np.zeros(b, dtype=np.uint8)
        p = self._shards[0].params(k, mode, **kw)
        _check(self._lib.cdb_search_batch_sharded(self._h, _ptr(q), b, C.byref(p), _ptr(ids), _ptr(scores), _ptr(counts), _ptr(err)))
        return ids, scores, counts, err

    def search_device(self, d_queries, nq, k, d_ids, d_scores, d_counts=None, d_err=None, stream_ptr=None, mode=0, **kw):
        """per-rank groups: device pointers (ints), asynchronous on the stream"""
        from .api import _check
        p = self._shards[0].params(k, mode, **kw)
        _check(self._lib.cdb_search_batch_sharded_device(self._h, C.c_void_p(d_queries), nq, C.byref(p), C.c_void_p(d_ids),
                                                         C.c_void_p(d_scores), C.c_void_p(d_counts) if d_counts else None,
                                                         C.c_void_p(d_err) if d_err else None,
                                                         C.c_void_p(stream_ptr) if stream_ptr else None))

    def search_filtered(self, queries, filters, k, width=None, **kw):
        """DenseIndex.batch_search_filtered over the group (every shard a graph with metadata of one md_dims): filters[q] is
        None or a list of int8[md_dims] -> (replica ids u32[B,k], scores f32[B,k], counts u32[B], err u8[B]); k=None: top_k None"""
        from .api import SearchMode, _check, _ptr
        q = np.ascontiguousarray(queries, dtype=np.float32)
        if q.ndim == 1:
            q = q[None]
        b = q.shape[0]
        offs, dims, has = self._shards[0].pack_filters(filters)
        if dims.shape[0] == 0:
            dims = np.zeros((1, self._shards[0].md_dims), dtype=np.int8)
        if k is None:
            k, kw["all_candidates"] = self.all_width(width), True
        ids = np.zeros((b, k), dtype=np.uint32)
        scores = np.zeros((b, k), dtype=np.float32)
        counts = np.zeros(b, dtype=np.uint32)
        err = np.zeros(b, dtype=np.uint8)
        p = self._shards[0].params(k, SearchMode.HNSW, **kw)
        _check(self._lib.cdb_search_batch_filtered_sharded(self._h, _ptr(q), b, C.byref(p), _ptr(offs), _ptr(dims), _ptr(has), _ptr(ids),
                                                           _ptr(scores), _ptr(counts), _ptr(err)))
        return ids, scores, counts, err

    def search_filtered_device(self, d_queries, nq, k, d_offsets, d_dims, n_filter_rows, d_has, d_ids, d_scores, d_counts=None,
                               d_err=None, stream_ptr=None, **kw):
        """per-rank groups: search_filtered on device pointers (ints), the filters in the CSR form of DenseIndex.pack_filters
        (d_has None: no query has a filter); asynchronous on the stream.  all_candidates=True: top_k None, k = the row width"""
        from .api import SearchMode, _check
        p = self._shards[0].params(k, SearchMode.HNSW, **kw)
        _check(self._lib.cdb_search_batch_filtered_sharded_device(self._h, d_queries, nq, C.byref(p), d_offsets, d_dims, n_filter_rows,
                                                                  d_has, d_ids, d_scores, d_counts, d_err,
                                                                  C.c_void_p(stream_ptr) if stream_ptr else None))

    def attach_sparse(self, local_slot, index):
        """a SparseIndex shard (id_base = its first global id) into local slot `local_slot`, next to any dense shard"""
        from .api import _check
        _check(self._lib.cdb_shard_group_attach_sparse(self._h, local_slot, index.h))
        self._text_shards.append(index)

    def attach_tfidf(self, local_slot, index):
        """a TfIdfIndex shard (id_base = its first global id) into local slot `local_slot`"""
        from .api import _check
        _check(self._lib.cdb_shard_group_attach_tfidf(self._h, local_slot, index.h))
        self._text_shards.append(index)

    def search_sparse(self, queries, options):
        """SparseIndex.batch_search over the whole group -> ids u32[B, k], scores f32[B, k], counts u32[B]"""
        from .api import _as_csr, _check, _ptr
        o, d, v = _as_csr(queries)
        nq, k = len(o) - 1, int(options.top_k or 0)
        ids = np.zeros((nq, max(k, 1)), np.uint32)
        scores = np.zeros((nq, max(k, 1)), np.float32)
        counts = np.zeros(max(nq, 1), np.uint32)
        p = options.params()
        _check(self._lib.cdb_sparse_search_batch_sharded(self._h, _ptr(o), _ptr(d), _ptr(v), nq, C.byref(p), _ptr(ids), _ptr(scores),
                                                         _ptr(counts)))
        return ids[:, :k], scores[:, :k], counts[:nq]

    def search_sparse_all(self, queries, options):
        """SparseIndex.batch_search_all over the whole group (top_k None: options.top_k None or 0) -> (offsets u64[B+1],
        ids u32[total], scores f32[total]); query q's results are ids[offsets[q]:offsets[q+1]], best first"""
        from .api import SparseResults, _as_csr, _check, _ptr
        o, d, v = _as_csr(queries)
        p = options.params()
        h = C.c_void_p()
        _check(self._lib.cdb_sparse_search_batch_all_sharded(self._h, _ptr(o), _ptr(d), _ptr(v), len(o) - 1, C.byref(p), C.byref(h)))
        r = SparseResults(h)
        try:
            off = r.offsets()
            ids, scores = r.read(0, len(off) - 1)
        finally:
            r.close()
        return off, ids, scores

    def search_sparse_device(self, d_offsets, d_dims, d_values, nq, options, d_ids, d_scores, d_counts, stream_ptr=None):
        """per-rank groups: the sparse search on device pointers (ints), asynchronous on the stream"""
        from .api import _check
        p = options.params()
        _check(self._lib.cdb_sparse_search_batch_sharded_device(self._h, d_offsets, d_dims, d_values, nq, C.byref(p), d_ids, d_scores,
                                                                d_counts, C.c_void_p(stream_ptr) if stream_ptr else None))

    def search_tfidf(self, queries, top_k=None):
        """TfIdfIndex.batch_search over the whole group (global N and df) -> ids u32[B, kout], scores f32[B, kout], counts u32[B]"""
        from .api import _check, _ptr, _query_csr
        o, h = _query_csr(queries)
        nq, k = len(o) - 1, int(top_k or 0)
        kout = 512 if k == 0 or k > 512 else k
        ids = np.zeros((max(nq, 1), kout), np.uint32)
        scores = np.zeros((max(nq, 1), kout), np.float32)
        counts = np.zeros(max(nq, 1), np.uint32)
        _check(self._lib.cdb_tfidf_search_batch_sharded(self._h, _ptr(o), _ptr(h), nq, k, _ptr(ids), _ptr(scores), _ptr(counts)))
        return ids[:nq], scores[:nq], counts[:nq]

    def search_tfidf_device(self, d_offsets, d_hashes, nq, n_hashes, top_k, d_ids, d_scores, d_counts, stream_ptr=None):
        """search_tfidf on device pointers (ints), asynchronous on the stream: d_offsets u64[nq + 1] with d_offsets[0] = 0 and
        d_offsets[nq] = n_hashes, d_hashes u32[n_hashes], d_ids / d_scores [nq, kout], d_counts u32[nq].  Groups whose local
        slots share the arrays' device: per-rank, one-slot and loopback groups."""
        from .api import _check
        _check(self._lib.cdb_tfidf_search_batch_sharded_device(self._h, d_offsets, d_hashes, nq, n_hashes, int(top_k or 0), d_ids,
                                                               d_scores, d_counts, C.c_void_p(stream_ptr) if stream_ptr else None))

    def _hybrid_sources(self, dense, sparse, tfidf, dense_id_stride, host):
        """cdb_hybrid_group_sources -> (struct, arrays to keep alive, n_queries or None).  Host form: dense = (queries f32[B, dim],
        DenseIndex.params keywords or None), sparse = (queries as for SparseIndex.batch_search, SparseSearchOptions or None),
        tfidf = queries as for TfIdfIndex.batch_search.  Device form: the queries are device pointers (ints): dense =
        (d_queries, kw), sparse = ((d_offsets, d_dims, d_values), options), tfidf = (d_offsets, d_hashes)."""
        from . import _lib
        from .api import SparseSearchOptions, _as_csr, _ptr, _query_csr
        src, keep, nqs = _lib.HybridGroupSources(), [], []
        if dense is not None:
            q, opts = (tuple(dense) + (None,))[:2]
            if host:
                q = np.ascontiguousarray(q, dtype=np.float32)
                q = q[None] if q.ndim == 1 else q
                keep.append(q)
                nqs.append(q.shape[0])
            src.use_dense, src.dense_queries = 1, _ptr(q) if host else q
            src.dense_params = self._shards[0].params(0, **(opts or {}))
            src.dense_id_stride = int(dense_id_stride)
        if sparse is not None:
            q, opts = (tuple(sparse) + (None,))[:2]
            if host:
                q = _as_csr(q)
                keep += list(q)
                nqs.append(len(q[0]) - 1)
            src.use_sparse = 1
            src.sparse_offsets, src.sparse_dims, src.sparse_values = [_ptr(a) for a in q] if host else q
            src.sparse_params = (opts or SparseSearchOptions(0)).params()
        if tfidf is not None:
            q = _query_csr(tfidf) if host else tuple(tfidf)
            if host:
                keep += list(q)
                nqs.append(len(q[0]) - 1)
            src.use_tfidf = 1
            src.tfidf_offsets, src.tfidf_hashes = [_ptr(a) for a in q] if host else q
        if len(set(nqs)) > 1:
            raise ValueError("every source needs the same number of queries")
        return src, keep, (nqs[0] if nqs else 0)

    def hybrid_search(self, top_k=10, fusion_constant_k=60.0, dense=None, sparse=None, tfidf=None, dense_id_stride=1):
        """batch_hybrid_search over the group's shards of two kinds (cdb_hybrid_search_batch_sharded): dense = (queries,
        DenseIndex.params keywords), sparse = (queries, SparseSearchOptions), tfidf = queries.  dense_id_stride =
        max_replica_per_node for replica graphs.  -> ids u32[B, 6 * top_k], scores f32[B, 6 * top_k], counts u32[B] (the
        whole fused union), dense err flags u8[B] (zeros without a dense source)"""
        from .api import _check, _ptr
        src, keep, nq = self._hybrid_sources(dense, sparse, tfidf, dense_id_stride, True)
        w = 6 * int(top_k)
        ids = np.zeros((max(nq, 1), max(w, 1)), np.uint32)
        scores = np.zeros((max(nq, 1), max(w, 1)), np.float32)
        counts = np.zeros(max(nq, 1), np.uint32)
        err = np.zeros(max(nq, 1), np.uint8)
        _check(self._lib.cdb_hybrid_search_batch_sharded(self._h, C.byref(src), nq, int(top_k), float(fusion_constant_k), _ptr(ids),
                                                         _ptr(scores), _ptr(counts), _ptr(err)))
        return ids[:nq, :w], scores[:nq, :w], counts[:nq], err[:nq]

    def hybrid_search_device(self, nq, d_ids, d_scores, d_counts, d_err=None, stream_ptr=None, top_k=10, fusion_constant_k=60.0,
                             dense=None, sparse=None, tfidf=None, dense_id_stride=1):
        """groups of one local slot: hybrid_search on device pointers (ints), asynchronous on the stream; see _hybrid_sources
        for the source forms.  A TF-IDF source is refused (CDB_UNSUPPORTED): the host sizes the TF-IDF idf exchange by the
        batch's term count, which cdb_hybrid_group_sources does not carry."""
        from .api import _check
        src, keep, _ = self._hybrid_sources(dense, sparse, tfidf, dense_id_stride, False)
        _check(self._lib.cdb_hybrid_search_batch_sharded_device(self._h, C.byref(src), nq, int(top_k), float(fusion_constant_k), d_ids,
                                                                d_scores, d_counts, d_err, C.c_void_p(stream_ptr) if stream_ptr else None))

    def _mixed_sources(self, kinds, dense, sparse, tfidf, dense_id_stride):
        """cdb_hybrid_group_mixed_sources of kinds (host) and every source's params; queries are set by the caller"""
        from . import _lib
        from .api import HYBRID_KIND_SOURCES, SparseSearchOptions, _ptr
        kinds = np.ascontiguousarray(kinds, dtype=np.uint8).reshape(-1)
        src = _lib.HybridGroupMixedSources()
        src.kinds = _ptr(kinds)
        src.n_dense, src.n_sparse, src.n_tfidf = (sum(name in HYBRID_KIND_SOURCES[k] for k in kinds.tolist() if k <= 2)
                                                  for name in ("dense", "sparse", "tfidf"))
        if dense is not None:
            src.dense_params = self._shards[0].params(0, **((tuple(dense) + (None,))[1] or {}))
        if sparse is not None:
            src.sparse_params = ((tuple(sparse) + (None,))[1] or SparseSearchOptions(0)).params()
        src.dense_id_stride = int(dense_id_stride)
        return src, kinds

    def hybrid_search_mixed(self, kinds, top_k=10, fusion_constant_k=60.0, dense=None, sparse=None, tfidf=None, dense_id_stride=1):
        """batch_hybrid_search over a batch that mixes kinds (cdb_hybrid_search_batch_mixed_sharded): kinds[q] names query q's
        pair (0 dense + sparse, 1 dense + tfidf, 2 sparse + tfidf); dense = (per-query vectors [B][dim], DenseIndex.params
        keywords), sparse = (per-query sparse queries [B], SparseSearchOptions), tfidf = per-query hash lists [B]; entries of
        queries whose kind does not name the source are ignored.  -> ids u32[B, 6 * top_k], scores, counts u32[B], err u8[B]
        (the dense search's flags OR-ed over the ranks; 0 for sparse + tfidf queries)"""
        from .api import _check, _ptr, _query_csr, sparse_csr, split_mixed
        kinds, batches = split_mixed(kinds, None if dense is None else tuple(dense)[0], None if sparse is None else tuple(sparse)[0], tfidf)
        src, kinds = self._mixed_sources(kinds, dense, sparse, tfidf, dense_id_stride)
        keep = [kinds]
        if "dense" in batches:
            q = np.ascontiguousarray(batches["dense"], dtype=np.float32)
            src.dense_queries = _ptr(q)
            keep.append(q)
        if "sparse" in batches:
            q = sparse_csr(batches["sparse"])
            src.sparse_offsets, src.sparse_dims, src.sparse_values = [_ptr(a) for a in q]
            keep += list(q)
        if "tfidf" in batches:
            q = _query_csr(batches["tfidf"])
            src.tfidf_offsets, src.tfidf_hashes = [_ptr(a) for a in q]
            src.n_tfidf_hashes = int(q[0][-1])
            keep += list(q)
        nq, w = kinds.size, 6 * int(top_k)
        ids = np.zeros((max(nq, 1), max(w, 1)), np.uint32)
        scores = np.zeros((max(nq, 1), max(w, 1)), np.float32)
        counts = np.zeros(max(nq, 1), np.uint32)
        err = np.zeros(max(nq, 1), np.uint8)
        _check(self._lib.cdb_hybrid_search_batch_mixed_sharded(self._h, C.byref(src), nq, int(top_k), float(fusion_constant_k), _ptr(ids),
                                                               _ptr(scores), _ptr(counts), _ptr(err)))
        return ids[:nq, :w], scores[:nq, :w], counts[:nq], err[:nq]

    def hybrid_search_mixed_device(self, kinds, d_ids, d_scores, d_counts, d_err=None, stream_ptr=None, top_k=10, fusion_constant_k=60.0,
                                   dense=None, sparse=None, tfidf=None, dense_id_stride=1):
        """groups of one local slot: hybrid_search_mixed on device pointers (ints), asynchronous on the stream.  kinds stays
        a host array; each source's queries are already its batch in request order, on the device: dense = (d_queries,
        kw), sparse = ((d_offsets, d_dims, d_values), options), tfidf = (d_offsets, d_hashes, n_hashes)."""
        from .api import _check
        src, kinds = self._mixed_sources(kinds, dense, sparse, tfidf, dense_id_stride)
        if dense is not None:
            src.dense_queries = tuple(dense)[0]
        if sparse is not None:
            src.sparse_offsets, src.sparse_dims, src.sparse_values = tuple(sparse)[0]
        if tfidf is not None:
            src.tfidf_offsets, src.tfidf_hashes, src.n_tfidf_hashes = tfidf
        _check(self._lib.cdb_hybrid_search_batch_mixed_sharded_device(self._h, C.byref(src), kinds.size, int(top_k), float(fusion_constant_k),
                                                                      d_ids, d_scores, d_counts, d_err,
                                                                      C.c_void_p(stream_ptr) if stream_ptr else None))

    def close(self):
        if self._h:
            self._lib.cdb_shard_group_destroy(self._h)
            self._h = None
        self._shards = []
        self._text_shards = []

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def cuda_merge_fn(lib, device, metric, stream_ptr):
    """merge of gathered (ids, scores) arrays through cdb_merge_topk_device (torch tensors on `device`); kept for callers that
    exchange ids/scores themselves -- cdb_search_batch_sharded does not need it"""
    import torch

    def merge(g_ids, g_scores):
        world, b, k = g_ids.shape
        out_ids = torch.empty((b, k), dtype=torch.int32, device=g_ids.device)
        out_scores = torch.empty((b, k), dtype=torch.float32, device=g_ids.device)
        rc = lib.cdb_merge_topk_device(device, int(metric), g_ids.data_ptr(), g_scores.data_ptr(), world, b, k,
                                       out_ids.data_ptr(), out_scores.data_ptr(), stream_ptr)
        if rc != 0:
            raise RuntimeError(f"cdb_merge_topk_device failed: {rc}")
        return out_ids.view(torch.uint32), out_scores      # ids are u32 (>= 2^31 for large id_base shards; 0xFFFFFFFF = empty)

    return merge
