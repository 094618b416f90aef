"""Committed known-answer vectors (tests/golden/hotpath_v1.npz, made by tests/golden/make_golden.py).

CPU (not gpu): the oracle still reproduces every stored byte, and a subset is re-derived independently of the oracle's C
code (exact-integer f32 emulation, numpy integer arithmetic) so the fixture is not only self-consistent.
GPU: the CUDA path reproduces the same bytes through the C ABI (quantize, pairwise distances incl. error arms, brute-force
top-k over raw f32 and over codes, HNSW search on the stored graph, sequential GPU build == stored graph)."""
import os

import numpy as np
import pytest

import oracle as orc
from oracle import pyhnsw
from tests import f32emu
from tests.golden import make_golden as mg

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "hotpath_v1.npz")


@pytest.fixture(scope="module")
def gold():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def fbits(u):
    return np.ascontiguousarray(u, dtype=np.uint32).view(np.float32)


# ------------------------------------------------------------------ CPU: fixture <-> oracle <-> independent derivation

def test_manifest_matches_fixture(gold):
    with open(os.path.join(os.path.dirname(GOLDEN), "MANIFEST.txt")) as f:
        assert f.read() == mg.manifest(gold)


def test_oracle_reproduces_every_golden_array(gold):
    fresh = mg.generate()
    assert sorted(fresh) == sorted(gold)
    for k in gold:
        assert fresh[k].dtype == gold[k].dtype and np.array_equal(fresh[k], gold[k]), k


@pytest.mark.parametrize("dim", [8, 31, 33])
def test_f32_cosine_rederived_with_exact_integer_emulation(gold, dim):
    m, q = gold[f"d{dim}/corpus"], gold[f"d{dim}/queries"]
    val = fbits(gold[f"d{dim}/st5/m0/value_bits"])
    status = gold[f"d{dim}/st5/m0/status"]
    for i in range(q.shape[0]):
        qm = f32emu.sqrt32(f32emu.sumsq_sequential(q[i]))
        for j in range(m.shape[0]):
            xm = f32emu.sqrt32(f32emu.sumsq_sequential(m[j]))
            den = f32emu.mul32(qm, xm)
            if den == 0.0:
                assert status[i, j] == 2                            # cosine.rs:230-231
                continue
            dot = f32emu.dot_f32_simd_order([float(x) for x in q[i]], [float(x) for x in m[j]])
            want = np.float32(f32emu.div32(dot, den))
            assert status[i, j] == 0 and bits(want) == bits(val[i, j]), (i, j)


@pytest.mark.parametrize("dim", mg.DIMS)
def test_integer_arms_rederived_with_numpy(gold, dim):
    m, q = gold[f"d{dim}/corpus"], gold[f"d{dim}/queries"]
    # u8: truncating affine map, integer dot -> f32 (scalar.rs:17-26, dot_product.rs:92-108)
    def u8codes(v):
        c = np.clip(v.astype(np.float32), np.float32(-1), np.float32(1))
        return ((c - np.float32(-1)) / np.float32(2) * np.float32(255)).astype(np.uint8)
    cm, cq = u8codes(m), u8codes(q)
    assert np.array_equal(cm, gold[f"d{dim}/st0/codes"]) and np.array_equal(cq, gold[f"d{dim}/st0/qcodes"])
    dots = cq.astype(np.int64) @ cm.astype(np.int64).T
    assert np.array_equal(bits(dots.astype(np.float32)), gold[f"d{dim}/st0/m3/value_bits"])
    # sub-byte: digit n = floor((x+1)/step) mod 2^r; plane 0 carries the MSB but is weighted 1 by the kernels
    for r in (1, 2, 3):
        step = np.float32(2.0) / np.float32(1 << r)
        def digits(v):
            n = np.floor((v.astype(np.float32) + np.float32(1)) / step)
            n = np.where(n < 0, 0, n).astype(np.int64) & ((1 << r) - 1)
            planes = [(n >> (r - 1 - p)) & 1 for p in range(r)]          # plane p = bit (r-1-p) of the digit
            return sum(planes[p] << p for p in range(r))                  # value the dot-product kernels see
        dm, dq = digits(m), digits(q)
        dots = dq @ dm.T
        assert np.array_equal(bits(dots.astype(np.float32)), gold[f"d{dim}/st{r}/m3/value_bits"]), r


def test_hnsw_golden_results_are_a_subset_of_good_neighbours(gold):
    """sanity of the stored search results against exact brute force (recall, not parity)"""
    vecs, queries = gold["hnsw/vectors"], gold["hnsw/queries"]
    exact, _ = orc.brute_topk_f32(vecs, queries, 5)
    got = gold["hnsw/st4_m0/result_ids"]
    hit = sum(len(set(exact[i]) & set(got[i])) for i in range(queries.shape[0]))
    assert hit >= 0.8 * exact.size


# ------------------------------------------------------------------ GPU: CUDA path through the C ABI

def _cdb():
    import cosdata_b200 as cdb
    return cdb


@pytest.mark.gpu
@pytest.mark.parametrize("dim", mg.DIMS)
def test_gpu_quantize_and_pair_distances_match_golden(gold, dim):
    cdb = _cdb()
    m, q = gold[f"d{dim}/corpus"], gold[f"d{dim}/queries"]
    sq = cdb.ScalarQuantization()
    codes, mags = sq.quantize_batch(m, cdb.StorageType.UnsignedByte, (-0.5, 0.75))
    assert np.array_equal(codes, gold[f"d{dim}/st0_range/codes"]) and np.array_equal(bits(mags), gold[f"d{dim}/st0_range/mag_bits"])
    for st in mg.STORAGES:
        codes, mags = sq.quantize_batch(m, st)
        qcodes, qmags = sq.quantize_batch(q, st)
        assert np.array_equal(codes, gold[f"d{dim}/st{st}/codes"]), st
        assert np.array_equal(bits(mags), gold[f"d{dim}/st{st}/mag_bits"]), st
        assert np.array_equal(qcodes, gold[f"d{dim}/st{st}/qcodes"]) and np.array_equal(bits(qmags), gold[f"d{dim}/st{st}/qmag_bits"])
        nq, n = q.shape[0], m.shape[0]
        xi, yi = np.repeat(np.arange(nq), n), np.tile(np.arange(n), nq)
        for metric in mg.METRICS:
            val, status = cdb.DistanceMetric(metric).calculate_pairs(st, dim, qcodes[xi], qmags[xi], codes[yi], mags[yi])
            want_status = gold[f"d{dim}/st{st}/m{metric}/status"].reshape(-1)
            want = gold[f"d{dim}/st{st}/m{metric}/value_bits"].reshape(-1)
            assert np.array_equal(status, want_status.astype(np.int32)), (st, metric)
            ok = want_status == 0
            assert np.array_equal(bits(val)[ok], want[ok]), (st, metric)


@pytest.mark.gpu
@pytest.mark.parametrize("dim", mg.DIMS)
def test_gpu_brute_force_topk_matches_golden(gold, dim):
    cdb = _cdb()
    m, q = gold[f"d{dim}/corpus"], gold[f"d{dim}/queries"]
    for tensor in (False, True):                                     # exact FFMA scan and wgmma prefilter + re-rank
        ix = cdb.DenseIndex(dim=dim, storage_type=cdb.StorageType.FullPrecisionFP, capacity=m.shape[0], tensor_prefilter=tensor)
        ix.append(m)
        ids, scores, counts, err = ix.batch_search(q, mg.K)
        assert np.array_equal(ids, gold[f"d{dim}/f32_topk_ids"]) and np.array_equal(bits(scores), gold[f"d{dim}/f32_topk_score_bits"])
        ix.close()
    for st in mg.STORAGES:
        for metric in mg.METRICS:
            key = f"d{dim}/st{st}/m{metric}/topk_ids"
            ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=m.shape[0])
            ix.append(m)
            if key not in gold:                                      # arm the reference does not have -> the search is an Err
                with pytest.raises(cdb.CosdataError):
                    ix.batch_search(q, mg.K, cdb.SearchMode.BRUTE_CODES)
            else:
                ids, scores, counts, err = ix.batch_search(q, mg.K, cdb.SearchMode.BRUTE_CODES)
                assert np.array_equal(ids, gold[key]), (st, metric)
                assert np.array_equal(bits(scores), gold[f"d{dim}/st{st}/m{metric}/topk_score_bits"]), (st, metric)
                assert np.array_equal(err, gold[f"d{dim}/st{st}/m{metric}/topk_err"]), (st, metric)
            ix.close()


@pytest.mark.gpu
@pytest.mark.parametrize("st,metric", [(4, 0), (0, 0), (2, 3)])
def test_gpu_hnsw_search_and_sequential_build_match_golden(gold, st, metric):
    cdb = _cdb()
    vecs, queries, root = gold["hnsw/vectors"], gold["hnsw/queries"], gold["hnsw/root_vector"]
    levels, nb, nb0, efc, shortlist, seed, ef, k = (int(x) for x in gold["hnsw/params"])
    tag = f"hnsw/st{st}_m{metric}"
    n, dim = vecs.shape
    node_row = [gold[f"{tag}/L{lv}/node_row"] for lv in range(levels + 1)]
    adj = [gold[f"{tag}/L{lv}/adj"] for lv in range(levels + 1)]
    child = [gold[f"{tag}/L{lv}/child"] for lv in range(levels + 1)]
    # search on the stored graph
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n + 1, keep_raw_f32=True)
    ix.append(np.concatenate([vecs, root[None]], axis=0))
    ix.set_graph(levels, nb, nb0, int(gold[f"{tag}/entry"][0]), n, node_row, adj, child)
    ev0, pp0 = ix.hnsw_counters()
    ids, scores, counts, err = ix.batch_search(queries, k, cdb.SearchMode.HNSW, ef_search=ef, shortlist_size=shortlist)
    ev1, pp1 = ix.hnsw_counters()
    assert np.array_equal(ids, gold[f"{tag}/result_ids"]) and np.array_equal(bits(scores), gold[f"{tag}/result_score_bits"])
    assert np.array_equal(counts, gold[f"{tag}/result_counts"]) and not err.any()
    assert [ev1 - ev0, pp1 - pp0] == gold[f"{tag}/evals_pops"].tolist()
    ix.close()
    # one-at-a-time GPU build reproduces the stored graph
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n + 1, keep_raw_f32=True)
    ix.append(vecs)
    ix.build_graph(levels, nb, nb0, efc, shortlist, 1, seed)
    g = ix.read_graph()
    assert g["entry"] == int(gold[f"{tag}/entry"][0])
    for lv in range(levels + 1):
        assert np.array_equal(g["node_row"][lv], node_row[lv]) and np.array_equal(g["adj"][lv], adj[lv]) and np.array_equal(g["child"][lv], child[lv]), lv
    ix.close()
