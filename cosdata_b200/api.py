"""Host-side mirror of the reference's operator surface for the distance hot path.

Same names / argument meaning / error behaviour as the Rust traits, implemented
as thin calls into the C ABI (include/cosdata_b200.h) -- nothing is computed in
Python:

  StorageType, Storage           src/quantization/mod.rs:19-25, src/storage/mod.rs:7-25
  ScalarQuantization.quantize    src/quantization/scalar.rs:10-52
  DistanceMetric.calculate       src/models/types.rs:460-496 (DistanceFunction, src/distance/mod.rs:8-16)
  DistanceError                  src/distance/mod.rs:18-22
  DenseIndex.batch_search        IndexOps::batch_search, src/indexes/mod.rs:260-272
  DenseIndex.score_ids           neighbour expansion, src/vector_store.rs:1161-1191
  DenseIndex.rerank              finalize_ann_results, src/vector_store.rs:404-445
"""
import ctypes as C
import enum
import os

import numpy as np

from . import _lib
from ._lib import BuildParams, GraphDesc, GraphMetadata, IndexDesc, SearchParams, VectorDataBatch

INVALID_ID = 0xFFFFFFFF
SEARCH_TENSOR_WITH_DELETED = 1      # cdb_search_params.flags bit CDB_SEARCH_TENSOR_WITH_DELETED
SEARCH_ALL_CANDIDATES = 2           # cdb_search_params.flags bit CDB_SEARCH_ALL_CANDIDATES (top_k None; k = the row width)


class Status(enum.IntEnum):
    OK = 0
    STORAGE_MISMATCH = 1
    CALCULATION_ERROR = 2
    INVALID_PARAMS = 3
    CUDA_ERROR = 4
    NCCL_ERROR = 5
    UNSUPPORTED = 6
    UNREACHABLE_ARM = 7


class StorageType(enum.IntEnum):
    """StorageType; SubByte(r) is SUB1..SUB3."""
    UnsignedByte = 0
    SubByte1 = 1
    SubByte2 = 2
    SubByte3 = 3
    HalfPrecisionFP = 4
    FullPrecisionFP = 5
    BFloat16 = 6          # labelled extension (CDB_ST_BF16), not a reference StorageType


class DistanceMetricKind(enum.IntEnum):
    Cosine = 0
    Euclidean = 1
    Hamming = 2
    DotProduct = 3


class SearchMode(enum.IntEnum):
    BRUTE_RAW = 0
    BRUTE_CODES = 1
    HNSW = 2


class CosdataError(RuntimeError):
    def __init__(self, status, msg=""):
        try:
            self.status = Status(status)
            name = self.status.name
        except ValueError:          # a status this mirror does not know yet: keep the number
            self.status = int(status)
            name = f"status {int(status)}"
        super().__init__(f"{name}: {msg}")


class DistanceError(CosdataError):
    """DistanceError::{StorageMismatch, CalculationError}"""


def _check(rc):
    if rc != 0:
        msg = _lib.load().cdb_last_error_string().decode("utf-8", "replace")
        raise CosdataError(rc, msg)


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def device_count():
    n = C.c_int32(0)
    rc = _lib.load().cdb_device_count(C.byref(n))
    return n.value if rc == 0 else 0


def debug_set_hnsw_flags(flags=0xFFFFFFFF):
    """former kernel-variant switch of CDB_MODE_HNSW searches: every value is accepted and selects nothing (HNSW search
    has one kernel per graph kind)"""
    _check(_lib.load().cdb_debug_set_hnsw_flags(flags & 0xFFFFFFFF))


def tensor_peak(kind_i8=True, device=0, iters=0):
    """dense wgmma issue-rate probe -> (TOP/s or TFLOP/s, ms); the measured peak of u8 / f16 MMAs"""
    tops, ms = C.c_double(0), C.c_float(0)
    _check(_lib.load().cdb_debug_tensor_peak(device, 1 if kind_i8 else 0, iters, C.byref(tops), C.byref(ms)))
    return tops.value, ms.value


def kernel_launch_count():
    return int(_lib.load().cdb_kernel_launch_count())


def synth_matrix(seed, n, dim, first_row=0):
    out = np.empty((n, dim), dtype=np.float32)
    _check(_lib.load().cdb_synth_fill_host(seed, first_row * dim, n * dim, _ptr(out)))
    return out


def code_bytes(storage_type, dim):
    return int(_lib.load().cdb_code_bytes(int(storage_type), dim))


class Storage:
    """enum Storage: one quantized vector = (variant, mag, payload bytes)."""

    __slots__ = ("storage_type", "mag", "code", "dim")

    def __init__(self, storage_type, mag, code, dim):
        self.storage_type = StorageType(storage_type)
        self.mag = np.float32(mag)
        self.code = np.ascontiguousarray(code, dtype=np.uint8)
        self.dim = int(dim)


class ScalarQuantization:
    """impl Quantization for ScalarQuantization"""

    def __init__(self, device=0):
        self.device = device

    def quantize_batch(self, vectors, storage_type, value_range=(-1.0, 1.0)):
        v = np.ascontiguousarray(vectors, dtype=np.float32)
        if v.ndim == 1:
            v = v[None]
        n, dim = v.shape
        codes = np.zeros((n, code_bytes(storage_type, dim)), dtype=np.uint8)
        mags = np.zeros(n, dtype=np.float32)
        _check(_lib.load().cdb_quantize_batch(self.device, int(storage_type), float(value_range[0]), float(value_range[1]),
                                              _ptr(v), n, dim, _ptr(codes), _ptr(mags)))
        return codes, mags

    def quantize(self, vector, storage_type, value_range=(-1.0, 1.0)):
        codes, mags = self.quantize_batch(vector, storage_type, value_range)
        return Storage(storage_type, mags[0], codes[0], np.asarray(vector).size)

    def train(self, vectors):  # scalar.rs:54-57: nothing to train
        return None


def sample_values_range(vectors, clamp_margin_percent=1.0, prior_counts=None, prior_values=0, device=0):
    """HNSWIndex::sample_embedding + finalize_sampling (`quantization: auto`) -> (counts u64[14], (range_start, range_end))"""
    v = np.ascontiguousarray(vectors, dtype=np.float32)
    if v.ndim == 1:
        v = v[None]
    n, dim = v.shape
    prior = None if prior_counts is None else np.ascontiguousarray(prior_counts, dtype=np.uint64)
    counts = np.zeros(14, dtype=np.uint64)
    rng = np.zeros(2, dtype=np.float32)
    _check(_lib.load().cdb_sample_values_range(device, _ptr(v), n, dim, float(clamp_margin_percent), _ptr(prior),
                                               int(prior_values), _ptr(counts), _ptr(rng)))
    return counts, (np.float32(rng[0]), np.float32(rng[1]))


def sample_values_range_device(d_ptr, n, dim, clamp_margin_percent=1.0, device=0, stream=None):
    counts = np.zeros(14, dtype=np.uint64)
    rng = np.zeros(2, dtype=np.float32)
    _check(_lib.load().cdb_sample_values_range_device(device, C.c_void_p(d_ptr), n, dim, float(clamp_margin_percent), None, 0,
                                                      _ptr(counts), _ptr(rng), C.c_void_p(stream) if stream else None))
    return counts, (np.float32(rng[0]), np.float32(rng[1]))


def prop_file_scan(path):
    """prop.data (file_persist.rs:58-108) -> (records, StorageType or None, elems per vector, code bytes per record)"""
    n, st, el, cb = C.c_uint64(0), C.c_int32(-1), C.c_uint32(0), C.c_uint64(0)
    _check(_lib.load().cdb_prop_file_scan(os.fsencode(path), C.byref(n), C.byref(st), C.byref(el), C.byref(cb)))
    return n.value, (StorageType(st.value) if st.value >= 0 else None), el.value, cb.value


def prop_file_load(path, first_record=0, max_records=None):
    """-> dict(ids u32[n], codes u8[n, code_bytes], mags f32[n], offsets u64[n], lengths u32[n], storage_type)"""
    total, st, _, cb = prop_file_scan(path)
    n = max(0, total - first_record) if max_records is None else min(max_records, max(0, total - first_record))
    ids = np.zeros(n, dtype=np.uint32)
    codes = np.zeros((n, cb), dtype=np.uint8)
    mags = np.zeros(n, dtype=np.float32)
    offsets = np.zeros(n, dtype=np.uint64)
    lengths = np.zeros(n, dtype=np.uint32)
    got = C.c_uint64(0)
    _check(_lib.load().cdb_prop_file_load(os.fsencode(path), first_record, n, _ptr(ids), _ptr(codes), _ptr(mags),
                                          _ptr(offsets), _ptr(lengths), C.byref(got)))
    assert got.value == n
    return {"ids": ids, "codes": codes, "mags": mags, "offsets": offsets, "lengths": lengths, "storage_type": st}


def prop_file_load_metadata(path):
    """replica Metadata records of a prop.data file -> dict(replica_ids, mags, mbits i32[n, md_dims], offsets, lengths)"""
    n, dims = C.c_uint64(0), C.c_uint32(0)
    _check(_lib.load().cdb_prop_file_scan_metadata(os.fsencode(path), C.byref(n), C.byref(dims)))
    n, dims = n.value, dims.value
    ids = np.zeros(n, dtype=np.uint32)
    mags = np.zeros(n, dtype=np.float32)
    mbits = np.zeros((n, dims), dtype=np.int32)
    offsets = np.zeros(n, dtype=np.uint64)
    lengths = np.zeros(n, dtype=np.uint32)
    got = C.c_uint64(0)
    _check(_lib.load().cdb_prop_file_load_metadata(os.fsencode(path), n, dims, _ptr(ids), _ptr(mags), _ptr(mbits), _ptr(offsets),
                                                   _ptr(lengths), C.byref(got)))
    assert got.value == n
    return {"replica_ids": ids, "mags": mags, "mbits": mbits, "offsets": offsets, "lengths": lengths}


class HnswFiles:
    """the reference's on-disk HNSW index (prop.data, nodes.ptr, <id>.index) flattened to the set_graph arrays"""

    def __init__(self, index_dir, root_link_offset, pseudo_root_link_offset=INVALID_ID, latest_version=None):
        """latest_version: bound for the "<region>-<version>.ptr" layout of enable_context_history (None = newest)"""
        self._lib = _lib.load()
        self._h = C.c_void_p()
        if latest_version is None:
            _check(self._lib.cdb_hnsw_files_open(os.fsencode(index_dir), int(root_link_offset), int(pseudo_root_link_offset), C.byref(self._h)))
        else:
            _check(self._lib.cdb_hnsw_files_open_versioned(os.fsencode(index_dir), int(root_link_offset), int(pseudo_root_link_offset),
                                                           int(latest_version), C.byref(self._h)))
        info = np.zeros(8, dtype=np.uint32)
        counts = np.zeros(33, dtype=np.uint32)
        _check(self._lib.cdb_hnsw_files_info(self._h, _ptr(info), _ptr(counts)))
        (self.num_levels, self.neighbors_count, self.level0_neighbors_count, self.entry, self.pseudo_entry, self.root_row,
         self.md_dims, self.n_md) = (int(x) for x in info)
        self.level_counts = counts[: self.num_levels + 1].copy()
        self.node_row, self.node_id, self.node_md, self.adj, self.child = [], [], [], [], []
        for lv in range(self.num_levels + 1):
            c = int(self.level_counts[lv])
            nb = self.level0_neighbors_count if lv == 0 else self.neighbors_count
            arrs = [np.zeros(c, np.uint32), np.zeros(c, np.uint32), np.zeros(c, np.uint32), np.zeros(c * nb, np.uint32), np.zeros(c, np.uint32)]
            _check(self._lib.cdb_hnsw_files_level(self._h, lv, *[_ptr(a) for a in arrs]))
            for dst, a in zip((self.node_row, self.node_id, self.node_md, self.adj, self.child), arrs):
                dst.append(a)
        self.md_bits = np.zeros((self.n_md, max(self.md_dims, 1)), dtype=np.int32)
        self.md_mags = np.zeros(self.n_md, dtype=np.float32)
        _check(self._lib.cdb_hnsw_files_metadata(self._h, _ptr(self.md_bits), _ptr(self.md_mags)))
        # the MetricResult stored with each slot, parallel to adj: value (empty slot 0) and tag (empty slot 0xFF)
        self.slot_scores, self.slot_tags = [], []
        for lv in range(self.num_levels + 1):
            sc, tg = np.zeros(self.adj[lv].size, np.float32), np.zeros(self.adj[lv].size, np.uint8)
            _check(self._lib.cdb_hnsw_files_slot_scores(self._h, lv, _ptr(sc), _ptr(tg)))
            self.slot_scores.append(sc)
            self.slot_tags.append(tg)

    def apply(self, index, slot_scores=False):
        """cdb_index_set_graph_from_files; slot_scores=True also attaches the stored slot similarities
        (cdb_index_set_graph_slot_scores), so the graph takes insert_graph_replicas / delete_rows_replicas"""
        _check(self._lib.cdb_index_set_graph_from_files(index._h, self._h))
        index.md_dims = max(self.md_dims, 1)
        if slot_scores:
            index.set_graph_slot_scores(self.slot_scores, self.slot_tags)

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._lib.cdb_hnsw_files_close(self._h)
            self._h = C.c_void_p()

    __del__ = close


def itoe_scan(collection_dir):
    """itoe.dim / itoe.<version>.data (collection.rs:149-164) -> (live dense embeddings, dim, max internal id)"""
    n, dim, mx = C.c_uint64(0), C.c_uint32(0), C.c_uint64(0)
    _check(_lib.load().cdb_itoe_scan(os.fsencode(collection_dir), C.byref(n), C.byref(dim), C.byref(mx)))
    return n.value, dim.value, mx.value


def itoe_load(collection_dir, first_entry=0, max_entries=None):
    """-> (internal ids u32[n] ascending, vectors f32[n, dim])"""
    total, dim, _ = itoe_scan(collection_dir)
    n = max(0, total - first_entry) if max_entries is None else min(max_entries, max(0, total - first_entry))
    ids = np.zeros(n, dtype=np.uint32)
    vecs = np.zeros((n, dim), dtype=np.float32)
    got = C.c_uint64(0)
    _check(_lib.load().cdb_itoe_load(os.fsencode(collection_dir), first_entry, n, _ptr(ids), _ptr(vecs), C.byref(got)))
    assert got.value == n
    return ids, vecs


def itoe_get(collection_dir, internal_id, capacity=65536):
    """Collection::get_raw_emb_by_internal_id -> f32[dim] or None"""
    out = np.zeros(capacity, dtype=np.float32)
    n = C.c_uint32(0)
    _check(_lib.load().cdb_itoe_get(os.fsencode(collection_dir), int(internal_id), _ptr(out), capacity, C.byref(n)))
    return out[: n.value].copy() if n.value else None


class DistanceMetric:
    """enum DistanceMetric + impl DistanceFunction (pairwise; batched here over pairs)."""

    def __init__(self, kind, device=0):
        self.kind = DistanceMetricKind(kind)
        self.device = device

    def calculate_pairs(self, storage_type, dim, x_codes, x_mags, y_codes, y_mags):
        """-> (values f32[n], status int32[n]); status mirrors Result<_, DistanceError> per pair."""
        x = np.ascontiguousarray(x_codes, dtype=np.uint8)
        y = np.ascontiguousarray(y_codes, dtype=np.uint8)
        xm = np.ascontiguousarray(x_mags, dtype=np.float32)
        ym = np.ascontiguousarray(y_mags, dtype=np.float32)
        n = xm.size
        out = np.zeros(n, dtype=np.float32)
        st = np.zeros(n, dtype=np.int32)
        _check(_lib.load().cdb_distance_pairs(self.device, int(self.kind), int(storage_type), dim, _ptr(x), _ptr(xm),
                                              _ptr(y), _ptr(ym), n, _ptr(out), _ptr(st)))
        return out, st

    def calculate_pairs_md(self, storage_type, dim, md_dims, x, y):
        """DistanceFunction::calculate over pairs of VectorData { id, quantized_vec, metadata } (cosine.rs:34-102).
        x / y: dict(codes, mags, ids=None, has_id=None, md_bits=None, md_mags=None, has_md=None); x is the query side.
        -> (values f32[n], status int32[n])"""
        keep = []

        def side(v):
            def arr(key, dt):
                a = v.get(key)
                if a is None:
                    return None
                a = np.ascontiguousarray(a, dtype=dt)
                keep.append(a)
                return a.ctypes.data
            return VectorDataBatch(arr("codes", np.uint8), arr("mags", np.float32), arr("ids", np.uint32), arr("has_id", np.uint8),
                                   arr("md_bits", np.int32), arr("md_mags", np.float32), arr("has_md", np.uint8))
        bx, by = side(x), side(y)
        n = np.asarray(x["mags"]).size
        out = np.zeros(n, dtype=np.float32)
        st = np.zeros(n, dtype=np.int32)
        _check(_lib.load().cdb_distance_pairs_md(self.device, int(self.kind), int(storage_type), dim, md_dims, C.byref(bx), C.byref(by),
                                                 n, _ptr(out), _ptr(st)))
        return out, st

    def calculate(self, x: Storage, y: Storage):
        """DistanceFunction::calculate(x, y) -> f32 or raises DistanceError."""
        if x.storage_type != y.storage_type:
            raise DistanceError(Status.STORAGE_MISMATCH, "storage variants differ")  # cosine.rs:214
        out, st = self.calculate_pairs(x.storage_type, x.dim, x.code[None], [x.mag], y.code[None], [y.mag])
        if st[0] != 0:
            raise DistanceError(int(st[0]), "pair")
        return out[0]


class DenseIndex:
    """Device-resident dense index shard: the GPU counterpart of what HNSWIndex +
    Collection hold for this path (quantized rows + mags, optional raw f32 rows)."""

    def __init__(self, dim, storage_type=StorageType.FullPrecisionFP, metric=DistanceMetricKind.Cosine,
                 value_range=(-1.0, 1.0), capacity=1, device=0, keep_raw_f32=False, id_base=0,
                 tensor_prefilter=True):
        self._lib = _lib.load()
        self.desc = IndexDesc(dim, int(storage_type), int(metric), float(value_range[0]), float(value_range[1]),
                              int(capacity), int(device), 1 if keep_raw_f32 else 0, int(id_base),
                              1 if tensor_prefilter else 0)
        self._h = C.c_void_p()
        _check(self._lib.cdb_index_create(C.byref(self.desc), C.byref(self._h)))
        self.dim = dim
        self.storage_type = StorageType(storage_type)
        self.metric = DistanceMetricKind(metric)

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._lib.cdb_index_destroy(self._h)
            self._h = C.c_void_p()

    __del__ = close

    def __len__(self):
        return int(self._lib.cdb_index_size(self._h))

    # -- ingest
    def append(self, vectors):
        v = np.ascontiguousarray(vectors, dtype=np.float32)
        assert v.ndim == 2 and v.shape[1] == self.dim
        _check(self._lib.cdb_index_append_f32(self._h, _ptr(v), v.shape[0]))

    def append_codes(self, codes, mags):
        c = np.ascontiguousarray(codes, dtype=np.uint8)
        m = np.ascontiguousarray(mags, dtype=np.float32)
        _check(self._lib.cdb_index_append_codes(self._h, _ptr(c), _ptr(m), m.size))

    def append_prop_file(self, path, max_ids=0):
        """append every Storage record of a reference prop.data file (row = record number) -> (n, ids u32[min(n, max_ids)])"""
        ids = np.zeros(max_ids, dtype=np.uint32)
        n = C.c_uint64(0)
        _check(self._lib.cdb_index_append_prop_file(self._h, os.fsencode(path), _ptr(ids) if max_ids else None, max_ids, C.byref(n)))
        return n.value, ids[: min(n.value, max_ids)]

    def append_itoe(self, collection_dir, max_ids=0):
        """append every live raw embedding of a reference collection directory, ascending internal id -> (n, internal ids)"""
        ids = np.zeros(max_ids, dtype=np.uint32)
        n = C.c_uint64(0)
        _check(self._lib.cdb_index_append_itoe(self._h, os.fsencode(collection_dir), _ptr(ids) if max_ids else None, max_ids, C.byref(n)))
        return n.value, ids[: min(n.value, max_ids)]

    def set_raw(self, first_row, vectors):
        """raw f32 rows for rows that were appended as codes (keep_raw_f32 index)"""
        v = np.ascontiguousarray(vectors, dtype=np.float32)
        _check(self._lib.cdb_index_set_raw_f32(self._h, first_row, _ptr(v), v.shape[0]))

    @property
    def raw_missing(self):
        return int(self._lib.cdb_index_raw_missing(self._h))

    def fill_raw_from_itoe(self, collection_dir, row_ids):
        """row r <- embedding of internal id row_ids[r] (INVALID_ID: none by design) -> (filled, missing)"""
        ids = np.ascontiguousarray(row_ids, dtype=np.uint32)
        f, m = C.c_uint64(0), C.c_uint64(0)
        _check(self._lib.cdb_index_fill_raw_from_itoe(self._h, os.fsencode(collection_dir), _ptr(ids), ids.size, C.byref(f), C.byref(m)))
        return f.value, m.value

    def append_synthetic(self, seed, n, first_row=None):
        """rows [first_row, first_row+n) of synthetic stream `seed` (default: continue at len(self))"""
        first_row = len(self) if first_row is None else first_row
        _check(self._lib.cdb_index_append_synthetic(self._h, seed, first_row, n))

    def read_codes(self, first, n):
        codes = np.zeros((n, code_bytes(self.storage_type, self.dim)), dtype=np.uint8)
        mags = np.zeros(n, dtype=np.float32)
        _check(self._lib.cdb_index_read_codes(self._h, first, n, _ptr(codes), _ptr(mags)))
        return codes, mags

    # -- S1
    @property
    def size(self):
        return int(self._lib.cdb_index_size(self._h))

    def params(self, k, mode=SearchMode.BRUTE_RAW, ef_search=256, shortlist_size=64, exact_only=False, prefilter_k=0,
               tensor_with_deleted=False, all_candidates=False):
        """tensor_with_deleted: brute-force searches may take the tensor-core paths while rows are deleted (the kernels skip
        them; results are identical, CDB_SEARCH_TENSOR_WITH_DELETED).  all_candidates: top_k None, k is the row width
        (CDB_SEARCH_ALL_CANDIDATES)"""
        flags = (SEARCH_TENSOR_WITH_DELETED if tensor_with_deleted else 0) | (SEARCH_ALL_CANDIDATES if all_candidates else 0)
        return SearchParams(k, int(mode), ef_search, shortlist_size, 1 if exact_only else 0, prefilter_k, flags, 0)

    def hnsw_out_cap(self):
        """(num_levels + 1) * 100: the most candidates one HNSW search reports per query, the row width of a top_k None search"""
        info = np.zeros(5, dtype=np.uint32)
        counts = np.zeros(32, dtype=np.uint32)
        _check(self._lib.cdb_index_graph_info(self._h, _ptr(info), _ptr(counts)))
        return (int(info[0]) + 1) * 100

    def _width(self, k, mode):
        """k=None (top_k None): (row width, True), the width that of the graph (1 for a brute-force mode, which refuses it)"""
        if k is not None:
            return k, False
        return (self.hnsw_out_cap() if int(mode) == SearchMode.HNSW else 1), True

    def batch_search(self, queries, k, mode=SearchMode.BRUTE_RAW, **kw):
        """IndexOps::batch_search -> (ids u32[B,k], scores f32[B,k], counts u32[B], err u8[B]).
        k=None (top_k None, HNSW only): every candidate, best first, in rows of hnsw_out_cap() columns"""
        q = np.ascontiguousarray(queries, dtype=np.float32)
        if q.ndim == 1:
            q = q[None]
        b = q.shape[0]
        k, all_candidates = self._width(k, mode)
        if all_candidates:
            kw["all_candidates"] = True
        ids = np.zeros((b, k), dtype=np.uint32)
        scores = np.zeros((b, k), dtype=np.float32)
        counts = np.zeros(b, dtype=np.uint32)
        err = np.zeros(b, dtype=np.uint8)
        p = self.params(k, mode, **kw)
        _check(self._lib.cdb_search_batch(self._h, _ptr(q), b, C.byref(p), _ptr(ids), _ptr(scores), _ptr(counts), _ptr(err)))
        return ids, scores, counts, err

    def batch_search_device(self, d_queries_ptr, b, k, d_ids_ptr, d_scores_ptr, d_counts_ptr=None, d_err_ptr=None,
                            stream_ptr=None, mode=SearchMode.BRUTE_RAW, **kw):
        """All pointers are device addresses (ints), asynchronous on stream_ptr."""
        p = self.params(k, mode, **kw)
        _check(self._lib.cdb_search_batch_device(self._h, d_queries_ptr, b, C.byref(p), d_ids_ptr, d_scores_ptr,
                                                 d_counts_ptr, d_err_ptr, stream_ptr))

    # -- S2
    def score_ids(self, query, ids):
        q = np.ascontiguousarray(query, dtype=np.float32)
        i = np.ascontiguousarray(ids, dtype=np.uint32)
        out = np.zeros(i.size, dtype=np.float32)
        st = np.zeros(i.size, dtype=np.int32)
        _check(self._lib.cdb_score_ids(self._h, _ptr(q), _ptr(i), i.size, _ptr(out), _ptr(st)))
        return out, st

    # -- S3
    def rerank(self, query, cand_ids, k):
        q = np.ascontiguousarray(query, dtype=np.float32)
        c = np.ascontiguousarray(cand_ids, dtype=np.uint32)
        ids = np.zeros(k, dtype=np.uint32)
        scores = np.zeros(k, dtype=np.float32)
        cnt = np.zeros(1, dtype=np.uint32)
        _check(self._lib.cdb_rerank_f32(self._h, _ptr(q), _ptr(c), c.size, k, _ptr(ids), _ptr(scores), _ptr(cnt)))
        return ids, scores, int(cnt[0])

    def last_kernel_ms(self):
        a, b = C.c_float(0), C.c_float(0)
        _check(self._lib.cdb_index_last_kernel_ms(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def scan_ms_history(self, n=64):
        out = np.zeros(n, dtype=np.float32)
        m = C.c_uint32(0)
        _check(self._lib.cdb_index_scan_ms_history(self._h, n, _ptr(out), C.byref(m)))
        return out[: m.value].copy()

    def hnsw_profile(self, enable=True, read=True):
        """per-phase clock64 sums of the HNSW search kernel (see cdb_index_hnsw_profile); returns a dict or None"""
        out = np.zeros(16, dtype=np.uint64) if read else None
        _check(self._lib.cdb_index_hnsw_profile(self._h, 1 if enable else 0, _ptr(out)))
        if out is None:
            return None
        names = ["adjacency", "fixed_set", "stage_issue", "stage_wait", "chains", "queue", "level_sort", "levels_total", "pops",
                 "trims", "exact_selections"]
        return {n: int(v) for n, v in zip(names, out)}

    def stats(self):
        out = np.zeros(8, dtype=np.uint64)
        _check(self._lib.cdb_index_stats_ex(self._h, _ptr(out), 8))
        return {"tensor_searches": int(out[0]), "fallbacks": int(out[1]), "zero_rows": int(out[2]), "odd_rows": int(out[3]),
                "has_shadow": bool(out[4]), "fallback_queries": int(out[5]), "s8_searches": int(out[6]),
                "tensor_deleted_searches": int(out[7])}

    def last_candidate_counts(self, n):
        out = np.zeros(n, dtype=np.uint32)
        _check(self._lib.cdb_index_last_candidate_counts(self._h, n, _ptr(out)))
        return out

    # -- HNSW graph
    def set_graph(self, num_levels, neighbors_count, level0_neighbors_count, entry, root_row, node_row, adjacency, child):
        """flat graph arrays per level (lists of uint32 numpy arrays), see include/cosdata_b200.h"""
        L1 = num_levels + 1
        nr = [np.ascontiguousarray(a, dtype=np.uint32) for a in node_row]
        ad = [np.ascontiguousarray(a, dtype=np.uint32) for a in adjacency]
        ch = [np.ascontiguousarray(a, dtype=np.uint32) for a in child]
        cnt = np.array([a.size for a in nr], dtype=np.uint32)
        t_nr = (C.c_void_p * L1)(*[a.ctypes.data for a in nr])
        t_ad = (C.c_void_p * L1)(*[a.ctypes.data for a in ad])
        t_ch = (C.c_void_p * L1)(*[a.ctypes.data for a in ch])
        gd = GraphDesc(num_levels, neighbors_count, level0_neighbors_count, entry, root_row, cnt.ctypes.data,
                       C.cast(t_nr, C.c_void_p), C.cast(t_ad, C.c_void_p), C.cast(t_ch, C.c_void_p))
        _check(self._lib.cdb_index_set_graph(self._h, C.byref(gd)))

    def set_graph_metadata(self, md_bits, md_mags, node_id, node_md, pseudo_entry):
        """replica ids / metadata rows per graph node + the metadata table + the pseudo root (include/cosdata_b200.h)"""
        bits = np.ascontiguousarray(md_bits, dtype=np.int32)
        mags = np.ascontiguousarray(md_mags, dtype=np.float32)
        ni = [np.ascontiguousarray(a, dtype=np.uint32) for a in node_id]
        nm = [np.ascontiguousarray(a, dtype=np.uint32) for a in node_md]
        t_ni = (C.c_void_p * len(ni))(*[a.ctypes.data for a in ni])
        t_nm = (C.c_void_p * len(nm))(*[a.ctypes.data for a in nm])
        md = GraphMetadata(bits.shape[1], bits.shape[0], bits.ctypes.data, mags.ctypes.data, C.cast(t_ni, C.c_void_p),
                           C.cast(t_nm, C.c_void_p), int(pseudo_entry))
        _check(self._lib.cdb_index_set_graph_metadata(self._h, C.byref(md)))
        self.md_dims = bits.shape[1]

    def set_graph_slot_scores(self, scores, tags=None):
        """cdb_index_set_graph_slot_scores: the similarity stored with every slot of a graph with uploaded metadata (one f32
        array of level_counts[L] * neighbours per level, the graph's upload order) and optionally the MetricResult tags
        (u8, same shape; checked against the index's metric).  The graph then takes insert_graph_replicas /
        delete_rows_replicas."""
        info = np.zeros(5, dtype=np.uint32)
        counts = np.zeros(32, dtype=np.uint32)
        _check(self._lib.cdb_index_graph_info(self._h, _ptr(info), _ptr(counts)))
        L1 = int(info[0]) + 1
        shapes = [int(counts[lv]) * int(info[2] if lv == 0 else info[1]) for lv in range(L1)]
        sc = [np.ascontiguousarray(a, dtype=np.float32).ravel() for a in scores]
        tg = None if tags is None else [np.ascontiguousarray(a, dtype=np.uint8).ravel() for a in tags]
        if len(sc) != L1 or (tg is not None and len(tg) != L1):
            raise ValueError(f"need one array per level ({L1})")
        for lv in range(L1):
            if sc[lv].size != shapes[lv] or (tg is not None and tg[lv].size != shapes[lv]):
                raise ValueError(f"level {lv} needs {shapes[lv]} slot values")
        t_sc = (C.c_void_p * L1)(*[a.ctypes.data for a in sc])
        t_tg = None if tg is None else (C.c_void_p * L1)(*[a.ctypes.data for a in tg])
        _check(self._lib.cdb_index_set_graph_slot_scores(self._h, C.cast(t_sc, C.c_void_p),
                                                         None if t_tg is None else C.cast(t_tg, C.c_void_p)))

    def pack_filters(self, filters):
        """filters[q]: None (no filter) or a list of int8[md_dims] (QueryFilterDimensions) -> the CSR form of the C API:
        (offsets u32[B+1], dims i8[rows, md_dims], has_filter u8[B])"""
        offs, rows, has = [0], [], []
        for f in filters:
            has.append(0 if f is None else 1)
            for dims in (f or []):
                rows.append(np.asarray(dims, dtype=np.int8).reshape(self.md_dims))
            offs.append(len(rows))
        dims = np.ascontiguousarray(np.stack(rows)) if rows else np.zeros((0, self.md_dims), dtype=np.int8)
        return np.array(offs, dtype=np.uint32), dims, np.array(has, dtype=np.uint8)

    def batch_search_filtered(self, queries, filters, k, **kw):
        """search_internal with per-query metadata filters: filters[q] is None or a list of int8[md_dims] (QueryFilterDimensions)
        -> (replica ids u32[B,k], scores f32[B,k], counts u32[B], err u8[B]); k=None (top_k None): rows of hnsw_out_cap()"""
        q = np.ascontiguousarray(queries, dtype=np.float32)
        if q.ndim == 1:
            q = q[None]
        b = q.shape[0]
        k, all_candidates = self._width(k, SearchMode.HNSW)
        if all_candidates:
            kw["all_candidates"] = True
        offs, dims, has = self.pack_filters(filters)
        if dims.shape[0] == 0:
            dims = np.zeros((1, self.md_dims), dtype=np.int8)
        ids = np.zeros((b, k), dtype=np.uint32)
        scores = np.zeros((b, k), dtype=np.float32)
        counts = np.zeros(b, dtype=np.uint32)
        err = np.zeros(b, dtype=np.uint8)
        p = self.params(k, SearchMode.HNSW, **kw)
        _check(self._lib.cdb_search_batch_filtered(self._h, _ptr(q), b, C.byref(p), _ptr(offs), _ptr(dims), _ptr(has), _ptr(ids),
                                                   _ptr(scores), _ptr(counts), _ptr(err)))
        return ids, scores, counts, err

    def batch_search_filtered_device(self, d_queries_ptr, b, k, d_offsets_ptr, d_dims_ptr, n_filter_rows, d_has_ptr, d_ids_ptr,
                                     d_scores_ptr, d_counts_ptr=None, d_err_ptr=None, stream_ptr=None, **kw):
        """batch_search_filtered on device buffers (cdb_search_batch_filtered_device): every pointer is a device address (int),
        the filters in the CSR form of pack_filters (d_has_ptr None = no query has a filter); asynchronous on stream_ptr.
        A query whose offsets are out of order or past n_filter_rows gets err flag 8 (BAD_FILTER) and count 0."""
        p = self.params(k, SearchMode.HNSW, **kw)
        _check(self._lib.cdb_search_batch_filtered_device(self._h, d_queries_ptr, b, C.byref(p), d_offsets_ptr, d_dims_ptr,
                                                          n_filter_rows, d_has_ptr, d_ids_ptr, d_scores_ptr, d_counts_ptr, d_err_ptr,
                                                          stream_ptr))

    def hnsw_counters(self):
        out = np.zeros(2, dtype=np.uint64)
        _check(self._lib.cdb_index_hnsw_counters(self._h, _ptr(out)))
        return int(out[0]), int(out[1])

    def build_graph(self, num_levels=9, neighbors_count=32, level0_neighbors_count=64, ef_construction=128,
                    shortlist_size=64, max_batch=4096, seed=1):
        """GPU-side index_embeddings: appends the root row and builds the HNSW graph (reference defaults)"""
        bp = BuildParams(num_levels, neighbors_count, level0_neighbors_count, ef_construction, shortlist_size, max_batch, seed)
        _check(self._lib.cdb_index_build_graph(self._h, C.byref(bp)))

    def insert_graph(self, ef_construction=128, shortlist_size=64, max_batch=4096, seed=1, max_level=None):
        """GPU-side index_embeddings on the live graph (cdb_index_insert_graph): inserts every row appended since the graph was
        built or uploaded.  num_levels and the neighbour counts are the graph's.  max_level: the caller's
        get_max_insert_level draws (u8 per new row) or None for the seeded counter RNG.  -> failed u8[n_new]"""
        check_insert_args(ef_construction, shortlist_size, max_batch)
        info = np.zeros(5, dtype=np.uint32)
        counts = np.zeros(32, dtype=np.uint32)
        _check(self._lib.cdb_index_graph_info(self._h, _ptr(info), _ptr(counts)))
        n_new = self.size - int(counts[0])
        lv = check_insert_args(ef_construction, shortlist_size, max_batch, max_level, n_new)
        failed = np.zeros(max(n_new, 1), dtype=np.uint8)
        done = C.c_uint64(0)
        bp = BuildParams(int(info[0]), int(info[1]), int(info[2]), ef_construction, shortlist_size, max_batch, seed)
        _check(self._lib.cdb_index_insert_graph(self._h, C.byref(bp), _ptr(lv) if lv is not None else None, _ptr(failed),
                                                C.byref(done)))
        return failed[: done.value]

    def delete_rows(self, rows, shortlist_size=64, max_batch=0):
        """delete_embedding on the GPU (cdb_index_delete_rows) for local row numbers -> status u8[len(rows)]: 0 deleted,
        1 already deleted, 2 deleted but an Err stopped some relinks"""
        r = np.asarray(rows)
        if r.ndim != 1:
            raise ValueError(f"rows must be one-dimensional, got shape {r.shape}")
        if r.size and (r.min() < 0 or r.max() >= self.size):
            raise ValueError(f"rows must be in 0..{self.size - 1}")
        check_insert_args(1, shortlist_size, max_batch)
        r = np.ascontiguousarray(r, dtype=np.uint32)
        status = np.zeros(max(r.size, 1), dtype=np.uint8)
        _check(self._lib.cdb_index_delete_rows(self._h, _ptr(r), r.size, shortlist_size, max_batch, _ptr(status), None))
        return status[: r.size]

    def delete_rows_replicas(self, rows, shortlist_size=64, max_batch=0):
        """delete_embedding on a graph that build_graph_replicas built (cdb_index_delete_rows_replicas): every node of each
        row, its base replica and its Metadata replicas, is deleted -> status u8[len(rows)]: 0 deleted, 1 already deleted,
        2 deleted but an Err hit one of the row's nodes"""
        r = np.asarray(rows)
        if r.ndim != 1:
            raise ValueError(f"rows must be one-dimensional, got shape {r.shape}")
        if r.size and (r.min() < 0 or r.max() >= self.size):
            raise ValueError(f"rows must be in 0..{self.size - 1}")
        check_insert_args(1, shortlist_size, max_batch)
        r = np.ascontiguousarray(r, dtype=np.uint32)
        status = np.zeros(max(r.size, 1), dtype=np.uint8)
        _check(self._lib.cdb_index_delete_rows_replicas(self._h, _ptr(r), r.size, shortlist_size, max_batch, _ptr(status), None))
        return status[: r.size]

    def read_replica_slot_scores(self):
        """-> [f32[level_counts[L] * neighbours]] per level of a graph that build_graph_replicas built: the similarity its
        builder keeps with each neighbour slot (0 = empty slot)"""
        info = np.zeros(5, dtype=np.uint32)
        counts = np.zeros(32, dtype=np.uint32)
        _check(self._lib.cdb_index_graph_info(self._h, _ptr(info), _ptr(counts)))
        out = []
        for lv in range(int(info[0]) + 1):
            a = np.zeros(int(counts[lv]) * int(info[2] if lv == 0 else info[1]), dtype=np.float32)
            _check(self._lib.cdb_index_read_replica_slot_scores(self._h, lv, _ptr(a)))
            out.append(a)
        return out

    def deleted_rows(self):
        """-> bool[size]: True where the row is deleted"""
        out = np.zeros(max(self.size, 1), dtype=np.uint8)
        _check(self._lib.cdb_index_deleted_rows(self._h, 0, self.size, _ptr(out), None))
        return out[: self.size].astype(bool)

    def read_graph_slot_scores(self):
        """-> [f32[level_counts[L] * neighbours]] per level: the similarity stored with each neighbour slot (0 = empty slot)"""
        info = np.zeros(5, dtype=np.uint32)
        counts = np.zeros(32, dtype=np.uint32)
        _check(self._lib.cdb_index_graph_info(self._h, _ptr(info), _ptr(counts)))
        out = []
        for lv in range(int(info[0]) + 1):
            a = np.zeros(int(counts[lv]) * int(info[2] if lv == 0 else info[1]), dtype=np.float32)
            _check(self._lib.cdb_index_read_graph_slot_scores(self._h, lv, _ptr(a)))
            out.append(a)
        return out

    def build_graph_replicas(self, row, node_id, base_id, md_row, max_level, md_bits, md_mags, main_root_md, pseudo_root_md,
                             num_levels=9, neighbors_count=32, level0_neighbors_count=64, ef_construction=128, shortlist_size=64,
                             max_batch=4096, seed=1):
        """GPU-side index_embeddings for a collection with a metadata schema (cdb_index_build_graph_replicas): one entry per
        graph node to create; row 0xFFFFFFFF = the pseudo root's vector.  -> failed u8[n_nodes]"""
        from ._lib import ReplicaBuild
        arrs = [np.ascontiguousarray(a, dtype=np.uint32) for a in (row, node_id, base_id, md_row)]
        lv = np.ascontiguousarray(max_level, dtype=np.uint8)
        bits = np.ascontiguousarray(md_bits, dtype=np.int32)
        mags = np.ascontiguousarray(md_mags, dtype=np.float32)
        n = arrs[0].size
        assert all(a.size == n for a in arrs) and lv.size == n and bits.ndim == 2 and mags.size == bits.shape[0]
        rb = ReplicaBuild(n, *[a.ctypes.data for a in arrs], lv.ctypes.data, bits.shape[1], bits.shape[0], bits.ctypes.data,
                          mags.ctypes.data, int(main_root_md) & 0xFFFFFFFF, int(pseudo_root_md))
        bp = BuildParams(num_levels, neighbors_count, level0_neighbors_count, ef_construction, shortlist_size, max_batch, seed)
        failed = np.zeros(max(n, 1), dtype=np.uint8)
        _check(self._lib.cdb_index_build_graph_replicas(self._h, C.byref(bp), C.byref(rb), _ptr(failed)))
        self.md_dims = bits.shape[1]
        return failed[:n]

    def insert_graph_replicas(self, row, node_id, base_id, md_row, max_level, md_bits_new=None, md_mags_new=None,
                              ef_construction=128, shortlist_size=64, max_batch=4096):
        """GPU-side index_embeddings on a graph that build_graph_replicas built (cdb_index_insert_graph_replicas): one entry per
        graph node to create, rows already appended; row 0xFFFFFFFF = the pseudo root's vector.  md_bits_new / md_mags_new:
        rows appended to the graph's metadata table (md_row may name them).  num_levels and the neighbour counts are the
        graph's.  -> failed u8[n_nodes]"""
        from ._lib import ReplicaInsert
        check_insert_args(ef_construction, shortlist_size, max_batch)
        # without a graph with metadata there is no md_dims: the library refuses the call (CDB_INVALID_PARAMS)
        md_dims = getattr(self, "md_dims", None) or (np.asarray(md_bits_new).shape[-1] if md_bits_new is not None else 1)
        arrs = [np.ascontiguousarray(a, dtype=np.uint32) for a in (row, node_id, base_id, md_row)]
        n = arrs[0].size
        if max_level is None:
            raise ValueError("max_level (the caller's get_max_insert_level draws) is required")
        lv = check_insert_args(ef_construction, shortlist_size, max_batch, max_level, n)
        if any(a.ndim != 1 or a.size != n for a in arrs):
            raise ValueError("row, node_id, base_id, md_row and max_level need one entry per node")
        bits = np.zeros((0, md_dims), np.int32) if md_bits_new is None else np.ascontiguousarray(md_bits_new, dtype=np.int32)
        mags = np.zeros(0, np.float32) if md_mags_new is None else np.ascontiguousarray(md_mags_new, dtype=np.float32)
        if bits.ndim != 2 or bits.shape[1] != md_dims or mags.shape != (bits.shape[0],):
            raise ValueError(f"md_bits_new must be [n, {md_dims}] with one md_mags_new entry per row")
        info = np.zeros(5, dtype=np.uint32)
        _check(self._lib.cdb_index_graph_info(self._h, _ptr(info), None))
        ri = ReplicaInsert(n, *[a.ctypes.data for a in arrs], lv.ctypes.data, md_dims, bits.shape[0], bits.ctypes.data, mags.ctypes.data)
        bp = BuildParams(int(info[0]), int(info[1]), int(info[2]), ef_construction, shortlist_size, max_batch, 0)
        failed = np.zeros(max(n, 1), dtype=np.uint8)
        done = C.c_uint64(0)
        _check(self._lib.cdb_index_insert_graph_replicas(self._h, C.byref(bp), C.byref(ri), _ptr(failed), C.byref(done)))
        return failed[: done.value]

    def read_graph_metadata(self):
        """-> (node_id[], node_md[]) per level of a graph with replica nodes"""
        info = np.zeros(5, dtype=np.uint32)
        counts = np.zeros(32, dtype=np.uint32)
        _check(self._lib.cdb_index_graph_info(self._h, _ptr(info), _ptr(counts)))
        ids, mds = [], []
        for lv in range(int(info[0]) + 1):
            a, b = np.zeros(int(counts[lv]), np.uint32), np.zeros(int(counts[lv]), np.uint32)
            _check(self._lib.cdb_index_read_graph_metadata_level(self._h, lv, _ptr(a), _ptr(b)))
            ids.append(a); mds.append(b)
        return ids, mds

    def read_graph(self):
        """-> dict(num_levels, neighbors_count, level0_neighbors_count, entry, root_row, node_row[], adj[], child[])"""
        info = np.zeros(5, dtype=np.uint32)
        counts = np.zeros(32, dtype=np.uint32)
        _check(self._lib.cdb_index_graph_info(self._h, _ptr(info), _ptr(counts)))
        L1 = int(info[0]) + 1
        node_row, adj, child = [], [], []
        for lv in range(L1):
            c = int(counts[lv])
            nb = int(info[2]) if lv == 0 else int(info[1])
            nr, ad, ch = np.zeros(c, np.uint32), np.zeros(c * nb, np.uint32), np.full(c, 0xFFFFFFFF, np.uint32)
            _check(self._lib.cdb_index_read_graph_level(self._h, lv, _ptr(nr), _ptr(ad), _ptr(ch)))
            node_row.append(nr); adj.append(ad); child.append(ch)
        return dict(num_levels=int(info[0]), neighbors_count=int(info[1]), level0_neighbors_count=int(info[2]),
                    entry=int(info[3]), root_row=int(info[4]), node_row=node_row, adj=adj, child=child)

    def append_device(self, d_ptr, n):
        """rows already on the index's device: d_ptr = address of n*dim contiguous f32"""
        _check(self._lib.cdb_index_append_f32_device(self._h, d_ptr, n))


def check_insert_args(ef_construction, shortlist_size, max_batch, max_level=None, n_new=None):
    """argument checks of DenseIndex.insert_graph (the ranges cdb_index_insert_graph accepts) -> max_level as u8 or None"""
    if not 1 <= int(ef_construction) <= 4096:
        raise ValueError(f"ef_construction must be in 1..4096, got {ef_construction}")
    if not 1 <= int(shortlist_size) <= 64:
        raise ValueError(f"shortlist_size must be in 1..64, got {shortlist_size}")
    if not 0 <= int(max_batch) <= 0xFFFFFFFF:
        raise ValueError(f"max_batch must be a u32 (0 = 4096), got {max_batch}")
    if max_level is None:
        return None
    lv = np.asarray(max_level)
    if lv.ndim != 1 or (n_new is not None and lv.size != n_new):
        raise ValueError(f"max_level needs one draw per new row ({n_new}), got shape {lv.shape}")
    if lv.size and (lv.min() < 0 or lv.max() > 255):
        raise ValueError("max_level draws must fit in u8")
    return np.ascontiguousarray(lv, dtype=np.uint8)


# ----------------------------------------------------------------------------- level draws (host side of the builders)
def level_probs(num_levels, factor=4.0):
    """generate_level_probs (src/models/common.rs:421-429; factor 4, api_service.rs:109): [(1 - factor^-n, n)] for n = num_levels..0"""
    return [(1.0 - float(factor) ** (-n), n) for n in range(int(num_levels), -1, -1)]


def pseudo_level_probs(num_levels, num_pseudo_nodes):
    """pseudo_level_probs (src/metadata/mod.rs:182-211): pseudo replicas are spread over the top ilog10(n)+1 levels"""
    higher = len(str(int(num_pseudo_nodes)))             # ilog10 + 1
    if higher > num_levels:
        higher, lower = 0, int(num_levels)
    else:
        lower = int(num_levels) - higher
    out = [(p, lower + lv) for p, lv in level_probs(higher, 10.0) if lv != 0] if higher > 0 else []
    return out + [(0.0, i) for i in range(lower, -1, -1)]


def max_insert_level(x, probs):
    """get_max_insert_level (src/models/common.rs:373-379): level of the first entry with x >= prob"""
    for p, lv in probs:
        if x >= p:
            return lv
    raise ValueError("No matching element found")


# ---------------------------------------------------------------- sparse inverted index (InvertedIndex)
def sparse_csr(rows):
    """list of [(dim, value), ...] per row -> (offsets u64[n+1], dims u32, values f32)"""
    off = np.zeros(len(rows) + 1, np.uint64)
    if rows:
        off[1:] = np.cumsum([len(r) for r in rows])
    dims = np.array([d for r in rows for d, _ in r], np.uint32)
    vals = np.array([v for r in rows for _, v in r], np.float32)
    return off, dims, vals


def _as_csr(x):
    if isinstance(x, tuple) and len(x) == 3:
        o, d, v = x
        return (np.ascontiguousarray(o, dtype=np.uint64), np.ascontiguousarray(d, dtype=np.uint32),
                np.ascontiguousarray(v, dtype=np.float32))
    return sparse_csr(x)


class SparseSearchOptions:
    """SparseSearchOptions (inverted/mod.rs:29-32) plus the config values search_internal reads: top_k (None = every
    candidate, SparseIndex.batch_search_all; batch_search needs a number),
    early_terminate_threshold (None = config.search.early_terminate_threshold, 0.0), rerank_sparse_with_raw_values and
    sparse_raw_values_reranking_factor (config.toml:5-6)"""

    def __init__(self, top_k, early_terminate_threshold=None, rerank=False, reranking_factor=5, config_threshold=0.0):
        self.top_k = top_k
        self.early_terminate_threshold = early_terminate_threshold
        self.rerank = rerank
        self.reranking_factor = reranking_factor
        self.config_threshold = config_threshold

    def params(self):
        thr = self.config_threshold if self.early_terminate_threshold is None else self.early_terminate_threshold
        return _lib.SparseSearchParams(int(self.top_k or 0), float(thr), 1 if self.rerank else 0, int(self.reranking_factor))


class SparseIndex:
    """InvertedIndex's IndexOps surface on one GPU (cdb_sparse_index).  Row r has id id_base + r."""

    def __init__(self, quantization_bits=4, values_upper_bound=1.0, capacity_rows=1 << 20, capacity_pairs=1 << 27, id_base=0,
                 device=0):
        L = _lib.load()
        d = _lib.SparseIndexDesc(device, quantization_bits, values_upper_bound, capacity_rows, capacity_pairs, id_base)
        h = C.c_void_p()
        _check(L.cdb_sparse_index_create(C.byref(d), C.byref(h)))
        self.h, self.desc = h, d
        self.sampling_counts, self.values_collected = np.zeros(9, np.uint64), 0

    def close(self):
        if getattr(self, "h", None):
            _lib.load().cdb_sparse_index_destroy(self.h)
            self.h = None

    __del__ = close

    def __len__(self):
        return int(_lib.load().cdb_sparse_index_size(self.h))

    def append(self, rows):
        """rows: list of pair lists, or a CSR triple (offsets, dims, values)"""
        o, d, v = _as_csr(rows)
        _check(_lib.load().cdb_sparse_index_append(self.h, _ptr(o), _ptr(d), _ptr(v), len(o) - 1))

    index_embeddings = append

    def delete_embedding(self, rows):
        """tombstones local rows (delete_embedding with the inserted pairs removes the row from every list)"""
        r = np.ascontiguousarray(np.atleast_1d(rows), dtype=np.uint32)
        _check(_lib.load().cdb_sparse_index_delete_rows(self.h, _ptr(r), r.size))

    def deleted_rows(self, first=0, n=None):
        n = len(self) - first if n is None else n
        out = np.zeros(max(n, 1), np.uint8)
        tot = C.c_uint64(0)
        _check(_lib.load().cdb_sparse_index_deleted_rows(self.h, first, n, _ptr(out), C.byref(tot)))
        return out[:n], tot.value

    def batch_search(self, queries, options):
        """-> ids u32[B, k], scores f32[B, k], counts u32[B]"""
        o, d, v = _as_csr(queries)
        nq, k = len(o) - 1, int(options.top_k or 0)
        ids = np.zeros((nq, max(k, 1)), np.uint32)
        scores = np.zeros((nq, max(k, 1)), np.float32)
        counts = np.zeros(max(nq, 1), np.uint32)
        p = options.params()
        _check(_lib.load().cdb_sparse_search_batch(self.h, _ptr(o), _ptr(d), _ptr(v), nq, C.byref(p), _ptr(ids), _ptr(scores),
                                                   _ptr(counts)))
        return ids[:, :k], scores[:, :k], counts[:nq]

    def search(self, query, options):
        if options.top_k is None:
            _, ids, scores = self.batch_search_all([list(query)], options)
            return list(zip(ids.tolist(), scores.tolist()))
        ids, scores, counts = self.batch_search([list(query)], options)
        c = int(counts[0])
        return list(zip(ids[0, :c].tolist(), scores[0, :c].tolist()))

    def search_all_results(self, queries, options):
        """top_k None (options.top_k = None): every candidate of every query -> a SparseResults handle"""
        o, d, v = _as_csr(queries)
        p = options.params()
        h = C.c_void_p()
        _check(_lib.load().cdb_sparse_search_batch_all(self.h, _ptr(o), _ptr(d), _ptr(v), len(o) - 1, C.byref(p), C.byref(h)))
        return SparseResults(h)

    def batch_search_all(self, queries, options):
        """top_k None: every candidate of every query, best first -> (offsets u64[B+1], ids u32[total], scores f32[total]);
        query q's results are ids[offsets[q]:offsets[q+1]]"""
        r = self.search_all_results(queries, options)
        try:
            off = r.offsets()
            ids, scores = r.read(0, len(off) - 1)
        finally:
            r.close()
        return off, ids, scores

    def sample_embedding(self, pairs, device=None):
        """accumulates the sampling counters over the pair values (sample_embedding)"""
        v = np.ascontiguousarray([x for _, x in pairs], dtype=np.float32)
        self.sampling_counts, _ = sparse_sample_upper_bound(v, 1.0, self.sampling_counts, self.values_collected,
                                                            self.desc.device if device is None else device)
        self.values_collected += v.size

    def finalize_sampling(self, clamp_margin_percent=1.0):
        """-> values_upper_bound (for an index created after sampling, as the reference's is_configured gate orders it)"""
        _, ub = sparse_sample_upper_bound(np.zeros(0, np.float32), clamp_margin_percent, self.sampling_counts, self.values_collected,
                                          self.desc.device)
        return ub

    def append_itoe(self, collection_dir):
        """cdb_sparse_index_append_itoe -> internal ids of the appended rows"""
        n, _, _ = itoe_scan_sparse(collection_dir)
        ids = np.zeros(max(n, 1), np.uint32)
        got = C.c_uint64(0)
        _check(_lib.load().cdb_sparse_index_append_itoe(self.h, os.fsencode(collection_dir), _ptr(ids), n, C.byref(got)))
        return ids[: got.value]


class SparseResults:
    """The results of a top_k None sparse search (cdb_sparse_results), held by the library in host memory"""

    def __init__(self, h):
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            _lib.load().cdb_sparse_results_destroy(self.h)
            self.h = None

    __del__ = close

    def offsets(self):
        """-> u64[n_queries + 1]"""
        L = _lib.load()
        n = C.c_uint32(0)
        _check(L.cdb_sparse_results_offsets(self.h, C.byref(n), None))
        off = np.zeros(n.value + 1, np.uint64)
        _check(L.cdb_sparse_results_offsets(self.h, C.byref(n), _ptr(off)))
        return off

    def read(self, first, n):
        """entries of queries [first, first + n) -> (ids u32, scores f32)"""
        off = self.offsets()
        m = int(off[first + n] - off[first]) if first + n < len(off) else 0
        ids = np.zeros(max(m, 1), np.uint32)
        scores = np.zeros(max(m, 1), np.float32)
        _check(_lib.load().cdb_sparse_results_read(self.h, first, n, _ptr(ids), _ptr(scores)))
        return ids[:m], scores[:m]


def sparse_sample_upper_bound(values, clamp_margin_percent=1.0, prior_counts=None, prior_values=0, device=0):
    """-> (counts u64[9] of values > 1..9, values_upper_bound)"""
    v = np.ascontiguousarray(values, dtype=np.float32)
    out = np.zeros(9, np.uint64)
    pr = None if prior_counts is None else np.ascontiguousarray(prior_counts, dtype=np.uint64)
    ub = C.c_float(0)
    _check(_lib.load().cdb_sparse_sample_upper_bound(device, _ptr(v), v.size, float(clamp_margin_percent), _ptr(pr), prior_values,
                                                     _ptr(out), C.byref(ub)))
    return out, ub.value


def itoe_scan_sparse(collection_dir):
    """-> (live embeddings with sparse values, their pairs, max internal id)"""
    n, p, mx = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
    _check(_lib.load().cdb_itoe_scan_sparse(os.fsencode(collection_dir), C.byref(n), C.byref(p), C.byref(mx)))
    return n.value, p.value, mx.value


def itoe_load_sparse(collection_dir):
    """-> (internal ids u32[n] ascending, (offsets u64[n+1], dims u32, values f32))"""
    n, p, _ = itoe_scan_sparse(collection_dir)
    ids = np.zeros(max(n, 1), np.uint32)
    off = np.zeros(n + 1, np.uint64)
    dims = np.zeros(max(p, 1), np.uint32)
    vals = np.zeros(max(p, 1), np.float32)
    got = C.c_uint64(0)
    _check(_lib.load().cdb_itoe_load_sparse(os.fsencode(collection_dir), 0, n, p, _ptr(ids), _ptr(off), _ptr(dims), _ptr(vals),
                                            C.byref(got)))
    return ids[:n], (off, dims[:p], vals[:p])


# ---------------------------------------------------------------- TF-IDF / BM25 index (TFIDFIndex)
def _u_to_f32(x):
    """Rust's `u32 as f32` / `u64 as f32` on an array: round to nearest, ties to even (exact for every u64)"""
    x = np.asarray(x, dtype=np.uint64)
    small = x < np.uint64(1 << 53)          # exact in f64, so one rounding to f32
    out = x.astype(np.float64).astype(np.float32)
    for i in np.flatnonzero(~small):
        v = int(x.flat[i])
        shift = v.bit_length() - 24
        m, rem = v >> shift, v & ((1 << shift) - 1)
        half = 1 << (shift - 1)
        if rem > half or (rem == half and m & 1):
            m += 1
        out.flat[i] = np.float32(m * 2.0 ** shift)
    return out


def bm25_term_frequency(count, doc_len, avgdl, k1, b):
    """compute_bm25_term_frequency (tf_idf/mod.rs:362-371) in f32, one rounding per operation, no FMA:
    count as f32 * (k1 + 1.0) / (count as f32 + k1 * (1.0 - b + b * (document_length as f32 / average_document_length)))"""
    f32 = np.float32
    c = _u_to_f32(np.asarray(count, dtype=np.uint32))
    dl = _u_to_f32(np.asarray(doc_len, dtype=np.uint32))
    k1, b, avgdl = f32(k1), f32(b), f32(avgdl)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        num = c * (k1 + f32(1.0))
        den = c + k1 * ((f32(1.0) - b) + b * (dl / avgdl))
        return (num / den).astype(np.float32)


def average_document_length(total_len, count):
    """finalize_sampling (tf_idf/mod.rs:187-207): total_documents_length (u64) as f32 / total_documents_count (u32) as f32"""
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.float32(_u_to_f32(np.uint64(total_len)) / _u_to_f32(np.uint32(count)))


def _tfidf_csr(rows):
    """list of [(hash, tf), ...] per row, or (offsets, hashes, tfs) -> CSR triple"""
    if isinstance(rows, tuple) and len(rows) == 3:
        o, h, v = rows
        return (np.ascontiguousarray(o, dtype=np.uint64), np.ascontiguousarray(h, dtype=np.uint32),
                np.ascontiguousarray(v, dtype=np.float32))
    return sparse_csr(rows)


def _query_csr(queries):
    """list of hash lists, or (offsets, hashes) -> (offsets u64, hashes u32)"""
    if isinstance(queries, tuple) and len(queries) == 2:
        return np.ascontiguousarray(queries[0], dtype=np.uint64), np.ascontiguousarray(queries[1], dtype=np.uint32)
    off = np.zeros(len(queries) + 1, np.uint64)
    if queries:
        off[1:] = np.cumsum([len(q) for q in queries])
    return off, np.array([h for q in queries for h in q], np.uint32)


def debug_bm25_host(x=(), n_docs=(), df=()):
    """the library's host copy of csrc/bm25_idf.h, the one a shard group's host form runs
    -> (bm25_log1pf(x) f32[n], bm25_idf(n_docs, df) f32[m])"""
    x = np.ascontiguousarray(x, dtype=np.float32)
    n_docs, df = np.ascontiguousarray(n_docs, dtype=np.uint32), np.ascontiguousarray(df, dtype=np.uint32)
    if n_docs.shape != df.shape:
        raise ValueError("n_docs and df differ in length")
    out_log1p, out_idf = np.empty_like(x), np.empty(df.shape, np.float32)
    _check(_lib.load().cdb_debug_bm25(0, _ptr(x), x.size, _ptr(out_log1p), _ptr(n_docs), _ptr(df), df.size, _ptr(out_idf), None))
    return out_log1p, out_idf


def debug_bm25_device(d_x, n, d_out_log1p, d_n_docs, d_df, n_pairs, d_out_idf, stream_ptr=None):
    """the library's device copy of csrc/bm25_idf.h, the one the idf kernels inline, on device pointers (ints) of the current
    device: bm25_log1pf(d_x[:n]) -> d_out_log1p, bm25_idf(d_n_docs, d_df)[:n_pairs] -> d_out_idf; asynchronous on the stream"""
    _check(_lib.load().cdb_debug_bm25(1, d_x, n, d_out_log1p, d_n_docs, d_df, n_pairs, d_out_idf, stream_ptr))


class TfIdfIndex:
    """TFIDFIndex's IndexOps surface on one GPU (cdb_tfidf_index) from (term_hash, tf) pairs.  Row r has id id_base + r."""

    def __init__(self, capacity_rows=1 << 20, capacity_pairs=1 << 26, id_base=0, device=0):
        L = _lib.load()
        d = _lib.TfIdfIndexDesc(device, capacity_rows, capacity_pairs, id_base)
        h = C.c_void_p()
        _check(L.cdb_tfidf_index_create(C.byref(d), C.byref(h)))
        self.h, self.desc = h, d

    def close(self):
        if getattr(self, "h", None):
            _lib.load().cdb_tfidf_index_destroy(self.h)
            self.h = None

    __del__ = close

    def __len__(self):
        return int(_lib.load().cdb_tfidf_index_size(self.h))

    def append(self, rows, version=0, counted=None):
        """rows: list of (hash, tf) lists or a CSR triple; counted: per-row flags (False = an id without text, empty row)"""
        o, h, v = _tfidf_csr(rows)
        c = None if counted is None else np.ascontiguousarray(counted, dtype=np.uint8)
        _check(_lib.load().cdb_tfidf_index_append(self.h, _ptr(o), _ptr(h), _ptr(v), _ptr(c), len(o) - 1, version))

    index_embeddings = append

    def delete_embedding(self, rows, version=0):
        """deletes local rows at `version` (mark_embedding_as_deleted)"""
        r = np.ascontiguousarray(np.atleast_1d(rows), dtype=np.uint32)
        _check(_lib.load().cdb_tfidf_index_delete_rows(self.h, _ptr(r), r.size, version))

    def deleted_rows(self, first=0, n=None):
        n = len(self) - first if n is None else n
        out = np.zeros(max(n, 1), np.uint8)
        tot = C.c_uint64(0)
        _check(_lib.load().cdb_tfidf_index_deleted_rows(self.h, first, n, _ptr(out), C.byref(tot)))
        return out[:n], tot.value

    def term_stats(self, hashes):
        """-> (df u32[n], idf f32[n] as the device holds it, N); unseen hashes get df 0 and idf NaN"""
        hs = np.ascontiguousarray(np.atleast_1d(hashes), dtype=np.uint32)
        df = np.zeros(max(hs.size, 1), np.uint32)
        idf = np.zeros(max(hs.size, 1), np.float32)
        n = C.c_uint32(0)
        _check(_lib.load().cdb_tfidf_index_term_stats(self.h, _ptr(hs), hs.size, _ptr(df), _ptr(idf), C.byref(n)))
        return df[:hs.size], idf[:hs.size], n.value

    def batch_search(self, queries, top_k=None):
        """queries: list of hash lists or (offsets, hashes); top_k None = all bucket winners (up to 512)
        -> ids u32[B, kout], scores f32[B, kout], counts u32[B] with kout = min(top_k, 512) (512 for None)"""
        o, h = _query_csr(queries)
        nq, k = len(o) - 1, int(top_k or 0)
        kout = 512 if k == 0 or k > 512 else k
        ids = np.zeros((max(nq, 1), kout), np.uint32)
        scores = np.zeros((max(nq, 1), kout), np.float32)
        counts = np.zeros(max(nq, 1), np.uint32)
        _check(_lib.load().cdb_tfidf_search_batch(self.h, _ptr(o), _ptr(h), nq, k, _ptr(ids), _ptr(scores), _ptr(counts)))
        return ids[:nq], scores[:nq], counts[:nq]

    def search(self, query, top_k=None):
        """-> [(id, score)] best first (search_internal's result order)"""
        ids, scores, counts = self.batch_search([list(query)], top_k)
        c = int(counts[0])
        return list(zip(ids[0, :c].tolist(), scores[0, :c].tolist()))


# ---------------------------------------------------------------- hybrid search (reciprocal-rank fusion)
def rrf_fuse(first_ids, first_counts, second_ids, second_counts, fusion_constant_k=60.0, id_strides=(1, 1), device=0):
    """batch_hybrid_search's fusion of two ranked id lists per query (cdb_rrf_fuse): ids u32[B, ld], counts u32[B] per list,
    id_strides = the max_replica_per_node of each list (0 or 1: ids are keys)
    -> ids u32[B, ld_first + ld_second], scores f32[B, ...], counts u32[B]: every distinct key, total_cmp descending"""
    a = np.ascontiguousarray(first_ids, dtype=np.uint32)
    b = np.ascontiguousarray(second_ids, dtype=np.uint32)
    if a.ndim == 1:
        a = a[None]
    if b.ndim == 1:
        b = b[None]
    ca = np.ascontiguousarray(np.atleast_1d(first_counts), dtype=np.uint32)
    cb = np.ascontiguousarray(np.atleast_1d(second_counts), dtype=np.uint32)
    nq, ld_a, ld_b = a.shape[0], a.shape[1], b.shape[1]
    if b.shape[0] != nq or ca.size != nq or cb.size != nq:
        raise ValueError("both lists need the same number of queries")
    ld = ld_a + ld_b
    ids = np.zeros((max(nq, 1), max(ld, 1)), np.uint32)
    scores = np.zeros((max(nq, 1), max(ld, 1)), np.float32)
    counts = np.zeros(max(nq, 1), np.uint32)
    _check(_lib.load().cdb_rrf_fuse(device, _ptr(a), _ptr(ca), ld_a, int(id_strides[0]), _ptr(b), _ptr(cb), ld_b, int(id_strides[1]),
                                    nq, float(fusion_constant_k), ld, _ptr(ids), _ptr(scores), _ptr(counts)))
    return ids[:nq, :ld], scores[:nq, :ld], counts[:nq]


def hybrid_sources(dense=None, sparse=None, tfidf=None):
    """the cdb_hybrid_sources of host queries -> (struct, arrays to keep alive, n_queries)
    dense = (DenseIndex, queries f32[B, dim], DenseIndex.params keywords or None)
    sparse = (SparseIndex, queries as for SparseIndex.batch_search, SparseSearchOptions or None)
    tfidf = (TfIdfIndex, queries as for TfIdfIndex.batch_search[, None])"""
    src, keep, nqs = _lib.HybridSources(), [], []
    if dense is not None:
        ix, q, opts = (tuple(dense) + (None,))[:3]
        q = np.ascontiguousarray(q, dtype=np.float32)
        if q.ndim == 1:
            q = q[None]
        src.dense, src.dense_queries, src.dense_params = ix._h, _ptr(q), ix.params(0, **(opts or {}))
        keep.append(q)
        nqs.append(q.shape[0])
    if sparse is not None:
        ix, q, opts = (tuple(sparse) + (None,))[:3]
        o, d, v = _as_csr(q)
        src.sparse, src.sparse_offsets, src.sparse_dims, src.sparse_values = ix.h, _ptr(o), _ptr(d), _ptr(v)
        src.sparse_params = (opts or SparseSearchOptions(0)).params()
        keep += [o, d, v]
        nqs.append(len(o) - 1)
    if tfidf is not None:
        ix, q = tuple(tfidf)[:2]
        o, h = _query_csr(q)
        src.tfidf, src.tfidf_offsets, src.tfidf_hashes = ix.h, _ptr(o), _ptr(h)
        keep += [o, h]
        nqs.append(len(o) - 1)
    if len(set(nqs)) > 1:
        raise ValueError("every source needs the same number of queries")
    return src, keep, (nqs[0] if nqs else 0)


def hybrid_batch_search(top_k=10, fusion_constant_k=60.0, dense=None, sparse=None, tfidf=None):
    """batch_hybrid_search over two of the three sources (cdb_hybrid_search_batch); see hybrid_sources for their form.
    -> ids u32[B, 6 * top_k], scores f32[B, 6 * top_k], counts u32[B] (the whole fused union, not truncated to top_k, as in
    the reference), dense err flags u8[B] (zeros without a dense source)"""
    src, keep, nq = hybrid_sources(dense, sparse, tfidf)
    w = 6 * int(top_k)
    ids = np.zeros((max(nq, 1), max(w, 1)), np.uint32)
    scores = np.zeros((max(nq, 1), max(w, 1)), np.float32)
    counts = np.zeros(max(nq, 1), np.uint32)
    err = np.zeros(max(nq, 1), np.uint8)
    _check(_lib.load().cdb_hybrid_search_batch(C.byref(src), nq, int(top_k), float(fusion_constant_k), _ptr(ids), _ptr(scores),
                                               _ptr(counts), _ptr(err)))
    return ids[:nq, :w], scores[:nq, :w], counts[:nq], err[:nq]


# which sources each kind of a mixed batch names (CDB_HYBRID_DENSE_SPARSE, _DENSE_TFIDF, _SPARSE_TFIDF), first list first
HYBRID_KIND_SOURCES = (("dense", "sparse"), ("dense", "tfidf"), ("sparse", "tfidf"))


def split_mixed(kinds, dense=None, sparse=None, tfidf=None):
    """batch_hybrid_search's query_mapping: per-query inputs (row or entry q is query q's input for that source; entries of
    queries whose kind does not name the source are ignored and may be None) -> (kinds u8[B], {source: its queries in
    request order}), dense as f32[n, dim], sparse and tfidf as lists"""
    kinds = np.ascontiguousarray(kinds, dtype=np.uint8).reshape(-1)
    if kinds.size and int(kinds.max()) > 2:
        raise ValueError("a kind is 0 (dense + sparse), 1 (dense + tfidf) or 2 (sparse + tfidf)")
    given = {"dense": dense, "sparse": sparse, "tfidf": tfidf}
    out = {}
    for name, q in given.items():
        rows = [i for i, k in enumerate(kinds.tolist()) if name in HYBRID_KIND_SOURCES[k]]
        if not rows:
            continue
        if q is None:
            raise ValueError(f"queries of kinds that name {name} need {name} inputs")
        if len(q) != kinds.size:
            raise ValueError(f"{name}: one input per query ({kinds.size})")
        out[name] = np.stack([np.asarray(q[i], np.float32) for i in rows]) if name == "dense" else [q[i] for i in rows]
    return kinds, out


def hybrid_batch_search_mixed(kinds, top_k=10, fusion_constant_k=60.0, dense=None, sparse=None, tfidf=None):
    """batch_hybrid_search over a batch that mixes kinds (cdb_hybrid_search_batch_mixed): kinds[q] names query q's pair
    (CDB_HYBRID_*: 0 dense + sparse, 1 dense + tfidf, 2 sparse + tfidf); dense = (DenseIndex, per-query vectors [B][dim],
    DenseIndex.params keywords or None), sparse = (SparseIndex, per-query sparse queries [B], SparseSearchOptions or None),
    tfidf = (TfIdfIndex, per-query hash lists [B]); entries of queries whose kind does not name the source are ignored.
    Each source is searched once over the queries that name it.  -> ids u32[B, 6 * top_k], scores f32[B, 6 * top_k],
    counts u32[B] (the whole fused union), err u8[B] (the dense search's flags; 0 for sparse + tfidf queries)"""
    ins = {n: (tuple(x) + (None,))[:3] for n, x in (("dense", dense), ("sparse", sparse), ("tfidf", tfidf)) if x is not None}
    kinds, batches = split_mixed(kinds, *(ins[n][1] if n in ins else None for n in ("dense", "sparse", "tfidf")))
    nq = kinds.size
    src, keep = _lib.HybridMixedSources(), [kinds]
    src.kinds = _ptr(kinds)
    if "dense" in ins:
        ix, _, opts = ins["dense"]
        src.dense, src.dense_params = ix._h, ix.params(0, **(opts or {}))
    if "sparse" in ins:
        src.sparse, src.sparse_params = ins["sparse"][0].h, (ins["sparse"][2] or SparseSearchOptions(0)).params()
    if "tfidf" in ins:
        src.tfidf = ins["tfidf"][0].h
    if "dense" in batches:
        q = np.ascontiguousarray(batches["dense"], dtype=np.float32)
        src.n_dense, src.dense_queries = q.shape[0], _ptr(q)
        keep.append(q)
    if "sparse" in batches:
        o, d, v = sparse_csr(batches["sparse"])
        src.n_sparse, src.sparse_offsets, src.sparse_dims, src.sparse_values = len(o) - 1, _ptr(o), _ptr(d), _ptr(v)
        keep += [o, d, v]
    if "tfidf" in batches:
        o, h = _query_csr(batches["tfidf"])
        src.n_tfidf, src.tfidf_offsets, src.tfidf_hashes = len(o) - 1, _ptr(o), _ptr(h)
        keep += [o, h]
    w = 6 * int(top_k)
    ids = np.zeros((max(nq, 1), max(w, 1)), np.uint32)
    scores = np.zeros((max(nq, 1), max(w, 1)), np.float32)
    counts = np.zeros(max(nq, 1), np.uint32)
    err = np.zeros(max(nq, 1), np.uint8)
    _check(_lib.load().cdb_hybrid_search_batch_mixed(C.byref(src), nq, int(top_k), float(fusion_constant_k), _ptr(ids), _ptr(scores),
                                                     _ptr(counts), _ptr(err)))
    return ids[:nq, :w], scores[:nq, :w], counts[:nq], err[:nq]
