"""The s8 search's refilter against the final bound (tensor_scan.cu, s8_refilter_kernel): after the scan, each candidate
is tested again against the k-th largest of its query's final class maxima, and the re-rank scores the survivors only.
Results must stay bit-identical to the exact scan and the CPU oracle at every k of the resident kernel, at dimensions whose
s8 rows end in a partial word, on row counts that end inside a tile, and with lists that overflow their capacity."""
import numpy as np
import pytest

import cosdata_b200 as cdb
import oracle as orc

pytestmark = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def check(ix, x, q, k, oracle_rows=8, **kw):
    st0 = ix.stats()
    ids, scores, _, _ = ix.batch_search(q, k, **kw)
    assert ix.stats()["s8_searches"] == st0["s8_searches"] + 1, "the s8 form did not answer"
    ids_e, scores_e, _, _ = ix.batch_search(q, k, exact_only=True)
    assert np.array_equal(ids, ids_e) and np.array_equal(bits(scores), bits(scores_e))
    want_ids, want_scores = orc.brute_topk_f32(x, q[:oracle_rows], k)
    assert np.array_equal(ids[:oracle_rows], want_ids) and np.array_equal(bits(scores[:oracle_rows]), bits(want_scores))


@pytest.mark.parametrize("dim", [257, 1022])
def test_every_k_with_partial_words_and_tiles(dim, monkeypatch):
    monkeypatch.setenv("CDB_TS_S8", "1")
    n = 256 * 101 + 5
    x, q = orc.synth_matrix(9600 + dim, n, dim), orc.synth_matrix(9601, 640, dim)
    ix = cdb.DenseIndex(dim=dim, capacity=n)
    ix.append(x)
    for k in range(1, 13):
        check(ix, x, q, k)
    ix.close()


def test_overflowing_lists_keep_the_fallback(monkeypatch):
    monkeypatch.setenv("CDB_TS_S8", "1")
    rng = np.random.default_rng(21)
    n, dim = 100_000, 256
    x = orc.synth_matrix(9700, n, dim).copy()
    centre = rng.normal(size=dim).astype(np.float32)
    rows = rng.choice(n, 3000, replace=False)
    x[rows] = centre + 1e-4 * rng.normal(size=(3000, dim)).astype(np.float32)
    q = orc.synth_matrix(9701, 512, dim).copy()
    q[:3] = centre + 1e-4 * rng.normal(size=(3, dim)).astype(np.float32)
    ix = cdb.DenseIndex(dim=dim, capacity=n)
    ix.append(x)
    check(ix, x, q, 10, prefilter_k=1024)
    assert (ix.last_candidate_counts(len(q))[:3] > 1024).all()
    ix.close()
