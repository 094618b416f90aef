"""The reader of the reference's TF-IDF index files (cdb_tfidf_files_*): the Python restatement of the reference's writer
and reader (tests/tfidf_files.py) round-trips, the quirk of serialize shows, the library's reader equals the Python
deserialize on every corner of the format, and malformed files are refused with CDB_INVALID_PARAMS, never a crash."""
import os
import struct
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import cosdata_b200 as cdb
from tests import tfidf_files as tff

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref", "tf_idf_index")


def library_view(d):
    """cdb_tfidf_files_* over directory d -> (info, N, {hash: (df, [(doc, tf bits, version)])})"""
    with cdb.TfIdfFiles(d) as f:
        hs, df, off, ids, tfs, ver = f.read()
        info = f.info
    bits = tfs.view(np.uint32)
    out = {int(h): (int(df[t]), [(int(ids[p]), int(bits[p]), int(ver[p])) for p in range(int(off[t]), int(off[t + 1]))])
           for t, h in enumerate(hs)}
    assert list(hs) == sorted(out)
    return info, info["n_docs"], out


def python_view(d):
    return tff.deserialize(*tff.read_dir(d))


def check_reader(d):
    info, n, got = library_view(d)
    want_n, want = python_view(d)
    assert n == want_n
    assert got == want
    live = [w for _, ws in want.values() for w in ws]
    assert info["terms"] == len(want) and info["live"] == len(live)
    assert info["id_end"] == (max(w[0] for w in live) + 1 if live else 0)
    return info


@pytest.mark.parametrize("seed", range(6))
def test_round_trip_of_histories_without_the_quirk(seed, tmp_path):
    hist, _, _ = tff.seeded_history(seed, flush_after={1, 3} if seed % 2 else None)
    hist.save(str(tmp_path))
    n, terms = python_view(str(tmp_path))
    assert n == hist.root.n_docs
    assert terms == hist.root.terms()
    check_reader(str(tmp_path))


def test_quirk_a_same_version_delete_after_a_flush_survives_the_reload(tmp_path):
    h = tff.History()
    a, b = 0x0001_0005, 0x0002_0005
    h.insert(0, [(a, 1.0), (b, 2.0)], 1)
    h.insert(1, [(a, 3.0)], 1)
    h.flush()
    h.delete(0, 1)                      # same version as the insert, after the record of version 1 was written
    h.insert(2, [(b, 4.0)], 2)
    h.flush()
    h.save(str(tmp_path))
    mem = h.root.terms()
    n, disk = python_view(str(tmp_path))
    assert n == h.root.n_docs == 2
    # in memory the entries of document 0 are gone (df - 1); after the reload they are live again with the old df
    assert mem[a] == (1, [(1, tff.tf_bits(3.0), 1)])
    assert disk[a] == (2, [(0, tff.tf_bits(1.0), 1), (1, tff.tf_bits(3.0), 1)])
    assert mem[b] == (1, [(2, tff.tf_bits(4.0), 2)])
    assert disk[b] == (2, [(0, tff.tf_bits(2.0), 1), (2, tff.tf_bits(4.0), 2)])
    check_reader(str(tmp_path))


def corner_history():
    """every corner of the format in one directory"""
    h = tff.History()
    dims = [0, 1, 4 ** 7, 65535, 5, 21]
    quots = [0, 1, 2, 3, 4, 5, 7, 0x7FFF, 0xFFFF]          # more than 4 quotients in one node: overflow chunks
    hashes = [q << 16 | d for d in dims for q in quots]
    tfs = [0.0, -0.0, np.inf, -np.inf, 1.5, float(np.frombuffer(struct.pack("<I", 0x7FC0_1234), np.float32)[0])]
    doc = 0
    for v in (1, 2, 3):
        for i in range(12):
            pairs = [(hh, tfs[(i + j) % len(tfs)]) for j, hh in enumerate(hashes) if (i + j + v) % 3 == 0]
            h.insert(doc, pairs, v)
            doc += 1
        h.delete(doc - 5, v)                 # in the insert's version
        if v > 1:
            h.delete(doc - 13, v)            # in a later one
        h.flush()
    # every document of one term deleted: a term with no live word
    lone = 9 << 16 | 65535
    h.insert(doc, [(lone, 2.0)], 4)
    h.delete(doc, 5)
    doc += 1
    # ids up to 2^31 - 1, and an id whose word is tombstone-shaped (bit 63 set): deserialize reads it as a tombstone
    h.docs[2 ** 31 - 1] = ([(hashes[0], 7.0)], True)
    h.root.n_docs += 1
    h.root.insert(hashes[0], tff.tf_bits(7.0), 2 ** 31 - 1, 5)
    h.root.insert(hashes[1], 0, 2 ** 31 | 1, 5)     # "tombstone" of version 1, index 0
    h.flush()
    return h


def test_reader_equals_deserialize_on_every_corner(tmp_path):
    h = corner_history()
    h.save(str(tmp_path))
    assert len([f for f in os.listdir(tmp_path) if f.endswith(".idat")]) == 5
    info = check_reader(str(tmp_path))
    n, terms = python_view(str(tmp_path))
    assert info["max_version"] == 5
    assert terms[9 << 16 | 65535][1] == [] and terms[9 << 16 | 65535][0] == 2
    assert max(w[0] for _, ws in terms.values() for w in ws) == 2 ** 31 - 1
    # the tombstone-shaped word marked word 0 of hashes[1]'s version-1 record
    mem = h.root.terms()
    assert len(terms[1 << 16][1]) == len(mem[1 << 16][1]) - 1


def test_reader_equals_deserialize_on_seeded_histories(tmp_path):
    for seed in range(10, 16):
        d = str(tmp_path / str(seed))
        hist, _, _ = tff.seeded_history(seed, n_versions=4, vocab_size=40, flush_after={2})
        hist.save(d)
        check_reader(d)


def test_list_scorer_equals_the_oracle(tmp_path):
    """tfidf_files.search_lists, which the GPU quirk test scores with, equals the C oracle fed the same history"""
    from tests import pytfidf as pt
    from tests.tfidf_data import query_csr, random_queries
    for seed in (30, 31, 32):
        hist, ops, vocab = tff.seeded_history(seed, n_versions=4, docs_per_version=50, vocab_size=12,
                                              flush_after={2} if seed % 2 else None)
        d = str(tmp_path / str(seed))
        hist.save(d)
        n_docs, terms = python_view(d)
        orc = pt.Oracle()
        for op in ops:
            if op[0] == "append":
                rows, counted, v = op[1], op[2], op[3]
                off = np.zeros(len(rows) + 1, np.uint64)
                off[1:] = np.cumsum([len(r) for r in rows])
                orc.append((off, np.array([h for r in rows for h, _ in r], np.uint32),
                            np.array([t for r in rows for _, t in r], np.float32)), v, counted)
            else:
                orc.delete(op[1], op[2])
        qs = random_queries(np.random.default_rng(seed), vocab, 40)
        for k in (1, 10, 512, 0):
            wi, ws, wc, _ = orc.search(query_csr(qs), k)
            gi, gs, gc = tff.search_lists(n_docs, terms, qs, k)
            assert np.array_equal(gc, wc) and np.array_equal(gi, wi) and np.array_equal(gs.view(np.uint32), ws.view(np.uint32)), (seed, k)
        orc.close()


# ---------------------------------------------------------------- refusals
def small_dir(tmp_path):
    h = tff.History()
    h.insert(0, [(0x0003_0001, 1.0), (0x0004_0001, 2.0)], 1)
    h.insert(1, [(0x0003_0001, 1.0)], 2)
    h.flush()
    h.save(str(tmp_path))
    return str(tmp_path), h


def refused(d, what):
    with pytest.raises(cdb.CosdataError) as e:
        cdb.TfIdfFiles(d)
    assert e.value.status == cdb.Status.INVALID_PARAMS
    msg = cdb.last_error() if hasattr(cdb, "last_error") else str(e.value)
    assert what in msg, msg


def patch(path, off, b):
    data = bytearray(open(path, "rb").read())
    data[off:off + len(b)] = b
    open(path, "wb").write(bytes(data))


def child_offset(h, dim):
    """the file offset of the node of `dim` and of its parent's child slot"""
    n, slot = h.root.root, None
    for i in tff.calculate_path(dim):
        slot = n.offset + 50 + 4 * i
        n = n.children[i]
    return n.offset, slot


def test_refuses_missing_files(tmp_path):
    d, _ = small_dir(tmp_path)
    os.remove(os.path.join(d, "2.idat"))
    refused(d, "missing")
    os.remove(os.path.join(d, "index-tree.dim"))
    refused(d, "missing")


def test_refuses_truncated_nodes_and_records(tmp_path):
    d, h = small_dir(tmp_path / "a")
    dim = os.path.join(d, "index-tree.dim")
    off, _ = child_offset(h, 1)
    data = open(dim, "rb").read()
    open(dim, "wb").write(data[:off + 60])
    refused(d, "past the end")
    d, h = small_dir(tmp_path / "b")
    p = os.path.join(d, "1.idat")
    data = open(p, "rb").read()
    open(p, "wb").write(data[:-4])
    refused(d, "truncated")


def test_refuses_offsets_past_the_end(tmp_path):
    d, h = small_dir(tmp_path / "a")
    _, slot = child_offset(h, 1)
    patch(os.path.join(d, "index-tree.dim"), slot, struct.pack("<I", 1 << 20))
    refused(d, "past the end")
    d, h = small_dir(tmp_path / "b")
    off, _ = child_offset(h, 1)
    patch(os.path.join(d, "index-tree.dim"), off + 6 + 2, struct.pack("<I", 1 << 20))   # first slot's list offset
    refused(d, "past its end")


def test_refuses_cycles(tmp_path):
    d, h = small_dir(tmp_path / "a")
    off, _ = child_offset(h, 1)
    patch(os.path.join(d, "index-tree.dim"), off + 50, struct.pack("<I", 4))           # child 0 of dim 1 -> the root
    refused(d, "")
    d, h = small_dir(tmp_path / "b")
    # the head record of 0x0003_0001 (version 1, offset 0) points to itself
    patch(os.path.join(d, "1.idat"), 0, struct.pack("<II", 0, 1))
    refused(d, "cycle")


def test_refuses_a_wrong_dim_and_a_missing_head_version(tmp_path):
    d, h = small_dir(tmp_path / "a")
    off, _ = child_offset(h, 1)
    patch(os.path.join(d, "index-tree.dim"), off, struct.pack("<I", 2))
    refused(d, "dim")
    d, h = small_dir(tmp_path / "b")
    off, _ = child_offset(h, 1)
    # the slot names version 3, and 3.idat holds a copy of the version-1 records: no record of version 3 (the reference panics)
    patch(os.path.join(d, "index-tree.dim"), off + 6 + 6, struct.pack("<I", 3))
    open(os.path.join(d, "3.idat"), "wb").write(open(os.path.join(d, "1.idat"), "rb").read())
    refused(d, "no record of its slot's version")


def test_null_arguments_and_close(tmp_path):
    from cosdata_b200 import _lib
    L = _lib.load()
    assert L.cdb_tfidf_files_open(None, None) == cdb.Status.INVALID_PARAMS
    assert L.cdb_tfidf_files_info(None, None) == cdb.Status.INVALID_PARAMS
    assert L.cdb_tfidf_files_read(None, None, None, None, None, None, None) == cdb.Status.INVALID_PARAMS
    assert L.cdb_tfidf_files_close(None) == cdb.Status.OK
    assert L.cdb_tfidf_index_load_files(None, None, 0, None, 1) == cdb.Status.INVALID_PARAMS
    d, _ = small_dir(tmp_path)
    f = cdb.TfIdfFiles(d)
    assert f.info == {"n_docs": 2, "terms": 2, "records": 3, "live": 3, "id_end": 2, "max_version": 2}
    f.close()
    f.close()


def check_reference_script(d):
    """directory d holds the files of tools/ref_fixtures' TF-IDF script: the library's reader, the Python deserialize and
    the in-memory state of the script's history agree"""
    h = tff.reference_fixture_script()
    info = check_reader(d)
    n, terms = python_view(d)
    assert n == h.root.n_docs == 12
    assert terms == h.root.terms()
    assert info["max_version"] == 3


def test_reference_fixture_script_through_the_python_writer(tmp_path):
    h = tff.reference_fixture_script()
    h.save(str(tmp_path))
    assert sorted(os.listdir(tmp_path)) == ["1.idat", "2.idat", "3.idat", "index-tree.dim"]
    check_reference_script(str(tmp_path))


@pytest.mark.skipif(not os.path.isdir(GOLDEN), reason="reference-written TF-IDF fixtures not present: tools/ref_fixtures/README.md")
def test_reference_written_files():
    check_reference_script(GOLDEN)


# ---------------------------------------------------------------- fuzz
CHILD = textwrap.dedent('''
    import os, shutil, sys
    import numpy as np
    sys.path.insert(0, sys.argv[1])
    import cosdata_b200 as cdb
    from tests import tfidf_files as tff

    tmp = sys.argv[2]
    rng = np.random.default_rng(4321)
    def mutate(path):
        b = bytearray(open(path, "rb").read())
        if not b:
            return
        kind = rng.integers(0, 3)
        if kind == 0:
            b = b[: int(rng.integers(0, len(b)))]
        elif kind == 1:
            for _ in range(int(rng.integers(1, 8))):
                b[int(rng.integers(0, len(b)))] = int(rng.integers(0, 256))
        else:
            p = int(rng.integers(0, len(b)))
            b[p:p + 4] = bytes(rng.integers(0, 256, 4, dtype=np.uint8))
        open(path, "wb").write(bytes(b))
    outcomes = [0, 0]
    hist, _, _ = tff.seeded_history(7, n_versions=3, docs_per_version=20, vocab_size=30, flush_after={1})
    for it in range(300):
        d = os.path.join(tmp, "tf")
        shutil.rmtree(d, ignore_errors=True)
        hist.save(d)
        names = sorted(os.listdir(d))
        mutate(os.path.join(d, names[int(rng.integers(0, len(names)))]))
        try:
            with cdb.TfIdfFiles(d) as f:
                f.read()
            outcomes[0] += 1
        except cdb.CosdataError as e:
            assert e.status == cdb.Status.INVALID_PARAMS
            outcomes[1] += 1
    print("outcomes", outcomes)
''')


def test_reader_fuzz_truncations_and_byte_flips(tmp_path):
    r = subprocess.run([sys.executable, "-c", CHILD, ROOT, str(tmp_path)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    ok, bad = (int(x) for x in r.stdout.split("outcomes [")[1].split("]")[0].split(","))
    assert ok + bad == 300 and bad > 0
