"""Reading the sparse pairs of the itoe store (cdb_itoe_scan_sparse / cdb_itoe_load_sparse): the reader parses past the
metadata fields (raw_vector_embedding.rs:34-64, 91-132) and returns the live embeddings that have sparse values, newest
version, ascending internal id.  Written with the test writer of tests/test_itoe_file.py.  CPU only; the sparse index
parameters are checked before any device is touched."""
import os

import numpy as np
import pytest

import cosdata_b200 as cdb
from cosdata_b200 import _lib
from tests.test_itoe_file import TreeMapWriter, raw_embedding


def f32(x):
    return float(np.float32(x))


def store(tmp_path):
    w = TreeMapWriter()
    want = {}
    rng = np.random.default_rng(2)
    for i, key in enumerate(rng.choice(300_000, 500, replace=False).tolist()):
        sp = [(int(d), f32(v)) for d, v in zip(rng.integers(0, 1 << 20, i % 7), rng.random(i % 7))] or None
        md = [None, {"age": -i, "tag": "t" * (i % 140)}, {"name": "x" * 200}][i % 3]   # both FieldValue variants, long strings
        dense = [0.25] * 3 if i % 2 else None
        w.insert(1, key, raw_embedding(f"id{i}", dense, doc_id="doc" if i % 5 == 0 else None, metadata=md, sparse=sp,
                                       text="body" if i % 4 == 0 else None))
        if sp:
            want[key] = sp
    keys = sorted(want)
    for key in keys[:10]:                                    # deleted keys
        w.delete(2, key)
        del want[key]
    for key in keys[10:20]:                                  # newer versions replace the pairs
        want[key] = [(key % 1000, 0.5), (3, -1.0)]
        w.insert(3, key, raw_embedding("new", None, metadata={"a": 1}, sparse=want[key]))
    for key in keys[20:25]:                                  # a newer version without sparse values drops the row
        w.insert(3, key, raw_embedding("dense-only", [1.0, 2.0, 3.0]))
        del want[key]
    w.serialize(str(tmp_path))
    return want


def test_sparse_pairs_read_as_the_reference_would(tmp_path):
    want = store(tmp_path)
    n, pairs, mx = cdb.itoe_scan_sparse(str(tmp_path))
    keys = sorted(want)
    assert n == len(keys) and pairs == sum(len(v) for v in want.values()) and mx == keys[-1]
    ids, (off, dims, vals) = cdb.itoe_load_sparse(str(tmp_path))
    assert ids.tolist() == keys
    for r, key in enumerate(keys):
        got = list(zip(dims[off[r]:off[r + 1]].tolist(), vals[off[r]:off[r + 1]].tolist()))
        assert got == want[key]
    # the dense reader is unchanged by the sparse fields
    dn, ddim, _ = cdb.itoe_scan(str(tmp_path))
    assert ddim == 3 and dn > 0


def test_damaged_sparse_records_fail_with_an_error(tmp_path):
    w = TreeMapWriter()
    w.insert(1, 5, raw_embedding("a", None, metadata={"k": 1}, sparse=[(1, 0.5), (2, 0.25)]))
    w.serialize(str(tmp_path))
    data = os.path.join(tmp_path, "itoe.1.data")
    raw = bytearray(open(data, "rb").read())
    with open(data, "wb") as f:                              # pairs cut short
        f.write(raw[:-6])
    with pytest.raises(cdb.CosdataError):
        cdb.itoe_scan_sparse(str(tmp_path))
    bad = bytes(raw).replace(b"\x01k\x00", b"\x01k\x07")     # FieldValue variant 7
    with open(data, "wb") as f:
        f.write(bad)
    with pytest.raises(cdb.CosdataError) as e:
        cdb.itoe_scan_sparse(str(tmp_path))
    assert "variant" in str(e.value)
    with pytest.raises(cdb.CosdataError):
        cdb.itoe_scan_sparse(str(tmp_path / "missing"))


def test_load_respects_max_pairs(tmp_path):
    store(tmp_path)
    n, pairs, _ = cdb.itoe_scan_sparse(str(tmp_path))
    import ctypes as C
    off = np.zeros(n + 1, np.uint64)
    d, v = np.zeros(pairs, np.uint32), np.zeros(pairs, np.float32)
    got = C.c_uint64(0)
    rc = _lib.load().cdb_itoe_load_sparse(os.fsencode(str(tmp_path)), 0, n, pairs - 1, None, off.ctypes.data, d.ctypes.data,
                                          v.ctypes.data, C.byref(got))
    assert rc == cdb.Status.INVALID_PARAMS


def test_sparse_index_params_are_checked_before_the_device():
    import ctypes as C
    L = _lib.load()
    h = C.c_void_p()
    for bits, cap, base in ((3, 10, 0), (9, 10, 0), (4, 0, 0), (4, 10, 0xFFFFFFF8)):
        d = _lib.SparseIndexDesc(0, bits, 1.0, cap, 10, base)
        assert L.cdb_sparse_index_create(C.byref(d), C.byref(h)) == cdb.Status.INVALID_PARAMS
    assert L.cdb_sparse_index_create(None, C.byref(h)) == cdb.Status.INVALID_PARAMS


def test_no_cpu_fallback_without_device():
    if cdb.device_count() > 0:
        pytest.skip("CUDA device present")
    with pytest.raises(cdb.CosdataError) as e:
        cdb.SparseIndex(capacity_rows=10, capacity_pairs=10)
    assert e.value.status == cdb.Status.CUDA_ERROR
    with pytest.raises(cdb.CosdataError) as e:
        cdb.sparse_sample_upper_bound(np.ones(4, np.float32))
    assert e.value.status == cdb.Status.CUDA_ERROR
