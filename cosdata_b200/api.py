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
    """kernel-variant switch of CDB_MODE_HNSW searches (measurement only; results are identical); default restores"""
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

    def apply(self, index):
        """cdb_index_set_graph_from_files"""
        _check(self._lib.cdb_index_set_graph_from_files(index._h, self._h))
        index.md_dims = max(self.md_dims, 1)

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

    def params(self, k, mode=SearchMode.BRUTE_RAW, ef_search=256, shortlist_size=64, exact_only=False, prefilter_k=0):
        return SearchParams(k, int(mode), ef_search, shortlist_size, 1 if exact_only else 0, prefilter_k, 0, 0)

    def batch_search(self, queries, k, mode=SearchMode.BRUTE_RAW, **kw):
        """IndexOps::batch_search -> (ids u32[B,k], scores f32[B,k], counts u32[B], err u8[B])"""
        q = np.ascontiguousarray(queries, dtype=np.float32)
        if q.ndim == 1:
            q = q[None]
        b = q.shape[0]
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
        names = ["adjacency", "fixed_set", "stage_issue", "stage_wait", "chains", "merge", "level_sort", "levels_total", "pops",
                 "speculation", "chain_phases", "speculative_evals"]
        return {n: int(v) for n, v in zip(names, out)}

    def stats(self):
        out = np.zeros(6, dtype=np.uint64)
        _check(self._lib.cdb_index_stats_ex(self._h, _ptr(out), 6))
        return {"tensor_searches": int(out[0]), "fallbacks": int(out[1]), "zero_rows": int(out[2]), "odd_rows": int(out[3]),
                "has_shadow": bool(out[4]), "fallback_queries": int(out[5])}

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

    def batch_search_filtered(self, queries, filters, k, **kw):
        """search_internal with per-query metadata filters: filters[q] is None or a list of int8[md_dims] (QueryFilterDimensions)
        -> (replica ids u32[B,k], scores f32[B,k], counts u32[B], err u8[B])"""
        q = np.ascontiguousarray(queries, dtype=np.float32)
        if q.ndim == 1:
            q = q[None]
        b = q.shape[0]
        offs, rows, has = [0], [], []
        for f in filters:
            has.append(0 if f is None else 1)
            for dims in (f or []):
                rows.append(np.asarray(dims, dtype=np.int8).reshape(self.md_dims))
            offs.append(len(rows))
        offs = np.array(offs, dtype=np.uint32)
        has = np.array(has, dtype=np.uint8)
        dims = np.ascontiguousarray(np.stack(rows)) if rows else np.zeros((1, self.md_dims), dtype=np.int8)
        ids = np.zeros((b, k), dtype=np.uint32)
        scores = np.zeros((b, k), dtype=np.float32)
        counts = np.zeros(b, dtype=np.uint32)
        err = np.zeros(b, dtype=np.uint8)
        p = self.params(k, SearchMode.HNSW, **kw)
        _check(self._lib.cdb_search_batch_filtered(self._h, _ptr(q), b, C.byref(p), _ptr(offs), _ptr(dims), _ptr(has), _ptr(ids),
                                                   _ptr(scores), _ptr(counts), _ptr(err)))
        return ids, scores, counts, err

    def hnsw_counters(self):
        out = np.zeros(2, dtype=np.uint64)
        _check(self._lib.cdb_index_hnsw_counters(self._h, _ptr(out)))
        return int(out[0]), int(out[1])

    def build_graph(self, num_levels=9, neighbors_count=32, level0_neighbors_count=64, ef_construction=128,
                    shortlist_size=64, max_batch=4096, seed=1):
        """GPU-side index_embeddings: appends the root row and builds the HNSW graph (reference defaults)"""
        bp = BuildParams(num_levels, neighbors_count, level0_neighbors_count, ef_construction, shortlist_size, max_batch, seed)
        _check(self._lib.cdb_index_build_graph(self._h, C.byref(bp)))

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
