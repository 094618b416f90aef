"""The library's own copies of the BM25 idf (csrc/bm25_idf.h) against the C library's log1pf, over the whole argument domain
and at production document counts.

Every TF-IDF score goes through bm25_idf, in two compiled copies: the device one the idf kernels inline (a single index's
table, a shard group's idf in both forms) and the same source compiled for the host.  tests/test_bm25_idf.py checks the
header's arithmetic through a separate g++ build; here cdb_debug_bm25 runs the library's own copies:

  - the device bm25_log1pf on every non-negative finite float (2^31 - 2^23 of them), compared as checksums of blocks of
    2^16 results with the C library's, block by block;
  - bm25_idf through both copies on N around 2^24 and 2^25, where N - df and df stop converting to f32 exactly, on
    production N with sampled df, and on the u32 sums a group of up to 8 ranks forms;
  - the host bm25_log1pf on every 61st float;
  - one TF-IDF index of more than 2^24 documents, end to end: its idf table, a batch against tests/pytfidf.py fed the whole
    corpus, and the same corpus over a two-slot loopback group in the host and the device form.

The reference outputs come from tests/bm25_driver.py, the C library side of the g++ driver."""
import time

import numpy as np
import pytest

import cosdata_b200 as cdb
from cosdata_b200.sharding import ShardGroup
from tests import bm25_driver
from tests import pytfidf as pt
from tests.test_bm25_idf import idf_pairs
from tests.test_gpu_tfidf_sharded_device import check, device_search
from tests.tfidf_data import query_csr

pytestmark = pytest.mark.gpu

FINITE, BLOCK = bm25_driver.FINITE, bm25_driver.BLOCK
CHUNK = 1 << 26          # floats per device launch of the sweep


@pytest.fixture(scope="module")
def driver():
    return bm25_driver.build()


def _hex(u):
    return f"{int(u):#010x}"


def device_log1pf(first, n):
    """the device bm25_log1pf of the floats with bits first .. first + n - 1 -> u32 bits (numpy)"""
    import torch
    dev = torch.device("cuda", 0)
    x = torch.arange(first, first + n, dtype=torch.int32, device=dev)
    out = torch.empty(n, dtype=torch.float32, device=dev)
    s = torch.cuda.current_stream(dev)
    cdb.debug_bm25_device(x.data_ptr(), n, out.data_ptr(), None, None, 0, None, s.cuda_stream)
    s.synchronize()
    return out.cpu().numpy().view(np.uint32)


def test_device_log1pf_equals_the_c_librarys_log1pf_on_every_non_negative_float(driver):
    """every non-negative finite float through the device copy in chunks on one stream; each block of 2^16 results is
    reduced on the device to sum((i + 1) * bits) mod 2^64 and compared with the driver's same sum of log1pf"""
    import torch
    assert FINITE == (1 << 31) - (1 << 23) and FINITE % BLOCK == 0
    want = np.array(bm25_driver.run(driver, "sums", 1, FINITE).split(), np.uint64)
    assert want.size == FINITE // BLOCK
    dev = torch.device("cuda", 0)
    s = torch.cuda.Stream(dev)
    w = torch.arange(1, BLOCK + 1, dtype=torch.int64, device=dev)
    out = torch.empty(CHUNK, dtype=torch.float32, device=dev)
    sums = torch.empty(FINITE // BLOCK, dtype=torch.int64, device=dev)
    t0 = time.perf_counter()
    with torch.cuda.stream(s):
        for c0 in range(0, FINITE, CHUNK):
            n = min(CHUNK, FINITE - c0)
            x = torch.arange(c0, c0 + n, dtype=torch.int32, device=dev)
            cdb.debug_bm25_device(x.data_ptr(), n, out.data_ptr(), None, None, 0, None, s.cuda_stream)
            bits = out[:n].view(torch.int32).to(torch.int64) & 0xFFFFFFFF
            sums[c0 // BLOCK:(c0 + n) // BLOCK] = (bits.view(-1, BLOCK) * w).sum(1)
    s.synchronize()
    print(f"\ndevice bm25_log1pf sweep: {FINITE} inputs in {FINITE // CHUNK + 1} launches, "
          f"{time.perf_counter() - t0:.2f} s with the checksums")
    got = sums.cpu().numpy().view(np.uint64)
    bad = np.flatnonzero(got != want)
    if bad.size:
        b = int(bad[0])
        dev_bits = device_log1pf(b * BLOCK, BLOCK)
        libc_bits = np.array(bm25_driver.run(driver, "dump", 1, b * BLOCK, BLOCK).split(), np.uint64).astype(np.uint32)
        i = int(np.flatnonzero(dev_bits != libc_bits)[0])
        pytest.fail(f"the device bm25_log1pf differs from the C library's log1pf in {bad.size} blocks of {BLOCK}; the first "
                    f"input is {_hex(b * BLOCK + i)}: device {_hex(dev_bits[i])}, log1pf {_hex(libc_bits[i])}")


def test_the_sweep_reaches_every_branch_of_bm25_log1pf(driver):
    """how many of the swept floats take each branch (by the header's thresholds): every branch is reached, and the five
    exclusive ones partition the domain"""
    counts = {k: int(v) for k, v in (line.split() for line in bm25_driver.run(driver, "branches").splitlines())}
    print("\nbm25_log1pf branches over the sweep:", counts)
    exclusive = ("tiny_below_2^-54", "tiny_below_2^-29", "unsplit", "split_below_sqrt2", "split_at_or_above_sqrt2")
    assert sum(counts[k] for k in exclusive) == FINITE
    assert all(v > 0 for v in counts.values()), counts


def production_pairs(rng):
    """(N, df) u32: every N in [2^24 - 4, 2^24 + 64] and [2^25 - 4, 2^25 + 4] against df 0..3, odd values near N / 2,
    N - 1, N and N + 1 (the first inexact u32 -> f32 conversions, ties to even included); then N of 8.8M (MS MARCO), 10M,
    100M, 2^31 and 2^32 - 1 with 10^4 sampled df each, some past N (u32 wrapping N - df)"""
    ns, dfs = [], []
    for lo, hi in ((2**24 - 4, 2**24 + 64), (2**25 - 4, 2**25 + 4)):
        for n in range(lo, hi + 1):
            d = [0, 1, 2, 3, n - 1, n, n + 1] + [v for v in range(n // 2 - 9, n // 2 + 10) if v & 1]
            ns += [n] * len(d)
            dfs += d
    for n in (8_841_823, 10_000_000, 100_000_000, 1 << 31, (1 << 32) - 1):
        d = np.concatenate([rng.integers(0, n + 1, 4000), (2.0 ** rng.uniform(0, np.log2(n), 4000)).astype(np.int64),
                            n - rng.integers(0, 1000, 1000), n + rng.integers(1, 1000, 1000)])
        ns += [n] * d.size
        dfs += d.tolist()
    return np.array(ns, np.uint64).astype(np.uint32), (np.array(dfs, np.int64) % (1 << 32)).astype(np.uint32)


def group_pairs(rng, groups=5000):
    """(N, df) as a shard group of 2..8 ranks forms them: each rank's N and df summed in u32, wrapping
    (tf_group_idf_kernel's arithmetic).  Ranks hold up to 2^31 documents, so many sums wrap."""
    world = rng.integers(2, 9, groups)
    live = np.arange(8)[None, :] < world[:, None]
    n_r = np.where(live, rng.integers(0, 1 << 31, (groups, 8)), 0).astype(np.uint64)
    df_r = (n_r * rng.uniform(0, 1.02, (groups, 8))).astype(np.uint64)     # a little past N: later-version deletes
    n = n_r.astype(np.uint32).sum(axis=1, dtype=np.uint32)
    df = df_r.astype(np.uint32).sum(axis=1, dtype=np.uint32)
    assert (n_r.sum(axis=1) >= 1 << 32).sum() > groups // 4 and (df_r.sum(axis=1) >= 1 << 32).sum() > groups // 8
    return n, df


def device_idf(n_docs, df):
    import torch
    dev = torch.device("cuda", 0)
    d_n = torch.from_numpy(n_docs.view(np.int32)).to(dev)
    d_df = torch.from_numpy(df.view(np.int32)).to(dev)
    out = torch.empty(n_docs.size, dtype=torch.float32, device=dev)
    s = torch.cuda.current_stream(dev)
    cdb.debug_bm25_device(None, 0, None, d_n.data_ptr(), d_df.data_ptr(), n_docs.size, out.data_ptr(), s.cuda_stream)
    s.synchronize()
    return out.cpu().numpy().view(np.uint32)


def test_bm25_idf_through_the_device_and_host_copies(driver):
    rng = np.random.default_rng(41)
    edge = np.array(idf_pairs(), np.uint64).astype(np.uint32)
    sets = {"edge and sampled": (edge[:, 0], edge[:, 1]), "production N": production_pairs(rng), "group sums": group_pairs(rng)}
    total, failures = 0, []
    for name, (n_docs, df) in sets.items():
        n_docs, df = np.ascontiguousarray(n_docs), np.ascontiguousarray(df)
        gxx, libc = bm25_driver.pairs(driver, n_docs, df)
        assert np.array_equal(gxx, libc), name
        for copy, got in (("device", device_idf(n_docs, df)), ("host", cdb.debug_bm25_host(n_docs=n_docs, df=df)[1].view(np.uint32))):
            bad = np.flatnonzero(got != libc)
            if bad.size:
                failures.append(f"{copy} bm25_idf differs from get_idf with log1pf on {bad.size} of {n_docs.size} {name} pairs "
                                f"({(n_docs[bad] > 1 << 24).sum()} with N > 2^24), the first (N, df) = ({n_docs[bad[0]]}, "
                                f"{df[bad[0]]}): {_hex(got[bad[0]])}, log1pf {_hex(libc[bad[0]])}")
        total += n_docs.size
    assert not failures, "\n".join(failures)
    big = sets["production N"][0] > 1 << 24
    assert big.sum() > 30000
    print(f"\nbm25_idf pairs: {total} through each copy ({', '.join(f'{k} {v[0].size}' for k, v in sets.items())}; "
          f"{big.sum()} with N > 2^24)")


def test_host_log1pf_on_every_61st_float(driver):
    count = -(-FINITE // 61)
    x = (np.arange(count, dtype=np.uint64) * 61).astype(np.uint32).view(np.float32)
    got = cdb.debug_bm25_host(x)[0].view(np.uint32)
    want = np.array(bm25_driver.run(driver, "sums", 61, count).split(), np.uint64)
    bad = np.flatnonzero(bm25_driver.block_sums(got) != want)
    if bad.size:
        b = int(bad[0])
        libc_bits = np.array(bm25_driver.run(driver, "dump", 61, b * BLOCK, BLOCK).split(), np.uint64).astype(np.uint32)
        mine = got[b * BLOCK:(b + 1) * BLOCK]
        i = int(np.flatnonzero(mine != libc_bits[:mine.size])[0])
        pytest.fail(f"the host bm25_log1pf differs from the C library's log1pf in {bad.size} blocks; the first input is "
                    f"{_hex((b * BLOCK + i) * 61)}: host {_hex(mine[i])}, log1pf {_hex(libc_bits[i])}")
    print(f"\nhost bm25_log1pf: {count} inputs (every 61st float)")


# ---------------------------------------------------------------- one index past 2^24 documents
N_DOCS = (1 << 24) + (1 << 20) + 2     # even: N - df is odd, so not an f32, for every odd df below 2^24
# df of each term: N - df rounds to even up (df 3, 7, ...) or down (df 1, 5, ...); 2^24 + 3 is itself inexact and rounds up
DFS = (1, 3, 2, 5, 7, 1001, 12345, 65537, (1 << 19) + 1, (1 << 24) + 3)
UNCOUNTED = 777                        # rows without text: ids, but not documents
SPLIT = 7_000_003                      # the two-slot group's shard boundary (not on a 2^15-row tile)


def production_corpus(seed=23):
    """one-term documents: term j in DFS[j] rows, the other counted rows empty, UNCOUNTED empty rows not counted, all
    shuffled -> (offsets, hashes, tfs), counted, term hashes"""
    rng = np.random.default_rng(seed)
    hashes = rng.choice(1 << 32, len(DFS), replace=False).astype(np.uint32)
    label = np.concatenate([np.repeat(np.arange(len(DFS)), DFS), np.full(N_DOCS - sum(DFS), -1), np.full(UNCOUNTED, -2)])
    label = label[rng.permutation(label.size)]
    has = label >= 0
    off = np.zeros(label.size + 1, np.uint64)
    np.cumsum(has, out=off[1:])
    tfs = (rng.integers(1, 64, int(has.sum())) * 0.125).astype(np.float32)    # few values: many equal scores
    return (off, hashes[label[has]], tfs), (label != -2).astype(np.uint8), hashes


def test_an_index_past_2_24_documents_end_to_end(driver):
    import torch
    (off, hs, tfs), counted, terms = production_corpus()
    rows = counted.size
    t0 = time.perf_counter()
    whole = cdb.TfIdfIndex(capacity_rows=rows, capacity_pairs=hs.size)
    whole.append((off, hs, tfs), 1, counted)
    torch.cuda.synchronize()
    ingest = time.perf_counter() - t0
    print(f"\n{rows} rows, {N_DOCS} documents, {hs.size} pairs ingested in {ingest:.2f} s (one append)")

    # the idf table the device computed after the append
    df, idf, n_docs = whole.term_stats(terms)
    assert n_docs == N_DOCS and df.tolist() == list(DFS)
    inexact = [d for d in DFS if int(np.float32(N_DOCS - d)) != N_DOCS - d or int(np.float32(d)) != d]
    assert len(inexact) >= 6
    _, libc = bm25_driver.pairs(driver, np.full(len(DFS), N_DOCS, np.uint32), df)
    assert np.array_equal(idf.view(np.uint32), libc), [(d, _hex(a), _hex(b)) for d, a, b in zip(DFS, idf.view(np.uint32), libc) if a != b]

    # a batch against the oracle fed the whole corpus
    t1 = time.perf_counter()
    orc = pt.Oracle()
    orc.append((off, hs, tfs), 1, counted)
    t = [int(h) for h in terms]
    qs = [[h] for h in t] + [t, t[::-1], [t[-1], t[-1]], [t[0], t[-1], 12345], [7], []]
    qo, qh = query_csr(qs)
    for k in (0, 10):
        got = whole.batch_search(qs, k)
        want = orc.search((qo, qh), k)
        check(got, want)
        assert got[2][len(DFS) - 1] == (k or 512) and got[2][0] == 1
    orc.close()
    print(f"oracle: the whole corpus replayed and searched in {time.perf_counter() - t1:.2f} s")

    # the same corpus over a two-slot loopback group, in both forms
    g = ShardGroup.local([0, 0])
    parts = []
    for r, (a, b) in enumerate(((0, SPLIT), (SPLIT, rows))):
        p = cdb.TfIdfIndex(capacity_rows=b - a, capacity_pairs=int(off[b] - off[a]), id_base=a)
        p.append((off[a:b + 1] - off[a], hs[off[a]:off[b]], tfs[off[a]:off[b]]), 1, counted[a:b])
        g.attach_tfidf(r, p)
        parts.append(p)
    assert sum(int(p.term_stats(terms)[0][-1]) for p in parts) == DFS[-1]
    for k in (0, 10):
        want = whole.batch_search(qs, k)
        check(g.search_tfidf(qs, k), want)
        check(device_search(g, qs, k), want)
    g.close()
    for x in parts + [whole]:
        x.close()
