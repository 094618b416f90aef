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


def gather_and_merge(local_ids, local_scores, world, all_gather_fn, k=None, metric=0):
    """host logic of the sharded search: pack -> ONE all-gather of B*k u64 -> merge.
    all_gather_fn(x: u64[B,k]) -> u64[world,B,k] stacked over ranks."""
    keys = pack_keys(local_ids, local_scores, metric)
    k = keys.shape[1] if k is None else k
    if world == 1:
        return merge_packed(keys[None], k, metric)[:2]
    return merge_packed(all_gather_fn(keys), k, metric)[:2]


# ----------------------------------------------------------------------------- C ABI wrapper
class ShardGroup:
    """cdb_shard_group: the NCCL communicator + gather buffers owned by the library."""

    def __init__(self, handle, lib):
        self._h, self._lib = handle, lib
        self._shards = []

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
        return cls(h, lib)

    @property
    def world(self):
        return int(self._lib.cdb_shard_group_world(self._h))

    def attach(self, local_slot, index):
        from .api import _check
        _check(self._lib.cdb_shard_group_attach(self._h, local_slot, index._h))
        self._shards.append(index)          # keep the shard alive as long as the group

    def search(self, queries, k, mode=0, **kw):
        """host queries -> merged (ids u32[B,k], scores f32[B,k], counts u32[B], err u8[B])"""
        from .api import _check, _ptr
        q = np.ascontiguousarray(queries, dtype=np.float32)
        b = q.shape[0]
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

    def close(self):
        if self._h:
            self._lib.cdb_shard_group_destroy(self._h)
            self._h = None
        self._shards = []

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
