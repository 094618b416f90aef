"""CPU-side checks of dense search without top_k (CDB_SEARCH_ALL_CANDIDATES) and of the filtered sharded entries: the flag and
the new prototypes are bound, the refusals that need no device come first (handles here are never dereferenced before
them), and the numpy mirror of the sharded run merge equals a plain sort of the concatenated keys."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import cosdata_b200 as cdb
from cosdata_b200 import _lib
from cosdata_b200.sharding import INVALID_ID, merge_runs, pack_keys, unpack_keys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HNSW, BRUTE_RAW, BRUTE_CODES = int(cdb.SearchMode.HNSW), int(cdb.SearchMode.BRUTE_RAW), int(cdb.SearchMode.BRUTE_CODES)
ALL = 2
INV = cdb.Status.INVALID_PARAMS
FAKE = C.c_void_p(16)                    # a handle or device address the host never dereferences before these refusals
ALL_ONLY_HNSW = "CDB_SEARCH_ALL_CANDIDATES (top_k None) applies to CDB_MODE_HNSW"


def params(k, mode=HNSW, flags=0):
    return _lib.SearchParams(k, mode, 64, 64, 0, 0, flags, 0)


def last_error():
    return _lib.load().cdb_last_error_string().decode()


def test_flag_prototypes_and_bindings():
    hdr = open(os.path.join(ROOT, "include", "cosdata_b200.h")).read()
    assert re.search(r"#define CDB_SEARCH_ALL_CANDIDATES 2u", hdr)
    assert cdb.api.SEARCH_ALL_CANDIDATES == ALL
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    for name, n in (("cdb_search_batch_filtered_sharded", 11), ("cdb_search_batch_filtered_sharded_device", 13)):
        assert name in _lib.PROTOTYPES and len(_lib.PROTOTYPES[name][1]) == n
        assert hasattr(_lib.load(), name)
        assert re.search(r"pub fn " + name + r"\(", doc)
    assert "match options.top_k" in doc


@pytest.mark.parametrize("mode", [BRUTE_RAW, BRUTE_CODES])
def test_flag_with_a_brute_force_mode_is_refused(mode):
    L = _lib.load()
    out = np.zeros(4, np.uint32)
    p = params(1, mode, ALL)
    assert L.cdb_search_batch_sharded(FAKE, FAKE, 1, C.byref(p), out.ctypes.data, out.ctypes.data, None, None) == INV
    assert last_error() == ALL_ONLY_HNSW
    # the filtered entries refuse any brute-force mode first, flag or not
    assert L.cdb_search_batch_filtered_device(None, FAKE, 4, C.byref(p), FAKE, FAKE, 1, FAKE, FAKE, FAKE, FAKE, FAKE, None) == INV
    assert last_error() == "metadata filters apply to CDB_MODE_HNSW"


def test_flag_in_hybrid_dense_params_is_refused():
    L = _lib.load()
    out = np.zeros(8, np.uint32)
    cnt = np.zeros(1, np.uint32)
    for flags, want in ((ALL, "CDB_SEARCH_ALL_CANDIDATES (top_k None) has no hybrid form: the dense sub-search takes k = 3 * top_k"),):
        s = _lib.HybridSources()
        s.dense, s.dense_queries, s.dense_params = FAKE, FAKE, params(0, HNSW, flags)
        s.sparse, s.sparse_offsets = FAKE, FAKE
        assert L.cdb_hybrid_search_batch(C.byref(s), 1, 2, 60.0, out.ctypes.data, out.ctypes.data, cnt.ctypes.data, None) == INV
        assert last_error() == want
        assert L.cdb_hybrid_search_batch_device(C.byref(s), 1, 2, 60.0, out.ctypes.data, out.ctypes.data, cnt.ctypes.data, None,
                                                None) == INV
        assert last_error() == want


def test_k_bounds_without_the_flag_are_unchanged():
    L = _lib.load()
    out = np.zeros(4, np.uint32)
    for k in (0, 1025):
        p = params(k)
        assert L.cdb_search_batch_sharded(FAKE, FAKE, 1, C.byref(p), out.ctypes.data, out.ctypes.data, None, None) == INV
        assert last_error() == "k must be in 1..1024"
        assert L.cdb_search_batch_filtered_device(None, FAKE, 4, C.byref(p), FAKE, FAKE, 1, FAKE, FAKE, FAKE, FAKE, FAKE, None) == INV
        assert last_error() == "k must be in 1..1024"
        assert L.cdb_search_batch_filtered_sharded(FAKE, FAKE, 1, C.byref(p), FAKE, FAKE, FAKE, out.ctypes.data, out.ctypes.data,
                                                   None, None) == INV
        assert last_error() == "k must be in 1..1024"
        assert L.cdb_search_batch_filtered_sharded_device(None, FAKE, 1, C.byref(p), FAKE, FAKE, 1, FAKE, FAKE, FAKE, FAKE, FAKE,
                                                          None) == INV
        assert last_error() == "k must be in 1..1024"
    # under the flag k is a width: 0 and 4096 pass these checks and reach the handle (null here)
    for k in (0, 4096):
        p = params(k, HNSW, ALL)
        assert L.cdb_search_batch_filtered_sharded_device(None, FAKE, 1, C.byref(p), FAKE, FAKE, 1, FAKE, FAKE, FAKE, FAKE, FAKE,
                                                          None) == INV
        assert last_error() == "null argument"


def test_filtered_sharded_refusals_before_any_device_work():
    L = _lib.load()
    ok = params(10)
    out = np.zeros(4, np.uint32)

    def host(g=FAKE, q=FAKE, p=ok, offs=FAKE, dims=FAKE, has=FAKE, ids=out.ctypes.data, scores=out.ctypes.data):
        rc = L.cdb_search_batch_filtered_sharded(g, q, 4, None if p is None else C.byref(p), offs, dims, has, ids, scores, None, None)
        return rc, last_error()

    def dev(g=None, p=ok, offs=FAKE, dims=FAKE, n_rows=1, has=FAKE):
        rc = L.cdb_search_batch_filtered_sharded_device(g, FAKE, 4, None if p is None else C.byref(p), offs, dims, n_rows, has, FAKE,
                                                        FAKE, FAKE, FAKE, None)
        return rc, last_error()

    for kw in ({"g": None}, {"q": None}, {"p": None}, {"ids": None}, {"scores": None}):
        assert host(**kw) == (INV, "null argument")
    assert host(p=params(10, BRUTE_RAW)) == (INV, "metadata filters apply to CDB_MODE_HNSW")
    assert host(p=params(10, BRUTE_RAW, ALL)) == (INV, "metadata filters apply to CDB_MODE_HNSW")
    assert host(offs=None) == (INV, "has_filter needs filter_offsets")
    assert dev(p=None) == (INV, "null params")
    assert dev(p=params(10, BRUTE_CODES)) == (INV, "metadata filters apply to CDB_MODE_HNSW")
    assert dev(offs=None) == (INV, "has_filter needs filter_offsets")
    assert dev(dims=None, n_rows=3) == (INV, "n_filter_rows > 0 needs filter_dims")
    assert dev() == (INV, "null argument")


def sorted_runs(rng, world, b, w, lens, dup_scores=False):
    """[world, b, w] u64 keys: run (r, q) holds lens[r][q] keys, descending, unique over the whole query, zero padded"""
    g = np.zeros((world, b, w), np.uint64)
    for q in range(b):
        n = sum(lens[r][q] for r in range(world))
        ids = rng.choice(1 << 20, size=n, replace=False).astype(np.uint32)
        sc = rng.normal(size=n).astype(np.float32)
        if dup_scores:
            sc = np.round(sc, 1).astype(np.float32)
            sc[: n // 3] = np.float32(0.0)
            sc[n // 3: n // 2] = np.float32(-0.0)
        keys = pack_keys(ids, sc)
        at = 0
        for r in range(world):
            m = lens[r][q]
            g[r, q, :m] = np.sort(keys[at:at + m])[::-1]
            at += m
    return g


@pytest.mark.parametrize("world,w", [(1, 7), (2, 5), (3, 16), (8, 40)])
def test_run_merge_equals_a_sort_of_the_concatenated_keys(world, w):
    rng = np.random.default_rng(world * 100 + w)
    b = 24
    lens = [[int(x) for x in rng.integers(0, w + 1, b)] for _ in range(world)]
    lens[0][0] = 0                                                      # an empty run
    for r in range(world):
        lens[r][1] = 0                                                  # every run empty
        lens[r][2] = w                                                  # every run full
    for dup in (False, True):
        g = sorted_runs(rng, world, b, w, lens, dup)
        ids, scores, counts = merge_runs(g)
        allk = np.transpose(g, (1, 0, 2)).reshape(b, world * w)
        want = np.sort(allk, axis=1)[:, ::-1]
        w_ids, w_scores = unpack_keys(want)
        assert np.array_equal(ids, w_ids)
        assert np.array_equal(scores.view(np.uint32), w_scores.view(np.uint32))
        assert np.array_equal(counts, (allk != 0).sum(axis=1))
        assert counts[1] == 0 and (ids[1] == INVALID_ID).all()
        assert counts[2] == world * w
