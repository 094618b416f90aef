"""The restated sharded dense search plan (tests/sharded_plan.py) against the sources it restates, and the cases of
tests/test_gpu_sharded_edges.py against the plan: together they must make every final kernel write keys into the gather
buffer -- both prefilter forms, the u8 tensor path, HNSW and the exact scan in both merge branches and in selective
mode -- at every candidate-cap class and across a chunk boundary.  CPU only."""
from tests import sharded_plan as sp
from tests.test_gpu_dense_edges import scan_plan


def test_constants_equal_the_sources():
    got = sp.source_plan()
    assert got == {"CH": sp.CH, "SCAN_SEL_CAP": sp.SCAN_SEL_CAP, "PREFILTER_CAPS": sp.PREFILTER_CAPS, "U8_CAPS": sp.U8_CAPS,
                   "MERGE_SMEM_MAX": sp.MERGE_SMEM_MAX}


def test_the_restated_conditions_are_the_drivers_own():
    api, sg = sp._read("api.cu"), sp._read("shard_group.cu")
    assert "if (p->mode == CDB_MODE_HNSW) return hnsw_search_locked(" in api
    assert "const bool del_ok = ix->n_deleted == 0 || (p->flags & CDB_SEARCH_TENSOR_WITH_DELETED);" in api
    assert ("const bool tensor_ok = raw && ix->d_xh && !p->exact_only && del_ok && nq >= 4 && ix->size >= 16384 && p->k <= 64 &&"
            in api)
    assert ("const bool u8_ok = u8_rows && !p->exact_only && del_ok && (metric == CDB_METRIC_COSINE || metric == CDB_METRIC_DOT_PRODUCT) && "
            "max_digit * max_digit * d.dim <= 0x7F7FFFFFull && ix->size >= 16384 && p->k <= 64 &&") in api
    assert "if (const char *e = getenv(\"CDB_TS_S8\")) return atoi(e) != 0;" in api
    # each chunk's keys land at their queries' rows of the shard's slot
    assert "sc->cur_keys = sc->keys_out ? sc->keys_out + (size_t)off * p->k : nullptr;" in api
    assert "index_result_metric(g->shard[0], p->mode)" in sg


def test_chunk_path_examples():
    raw, codes = sp.RAW, sp.CODES
    assert sp.chunk_path(raw, sp.F32, sp.COSINE, 2051, 16384, 10, 128) == [("f16", 8192), ("scan", None)]
    assert sp.chunk_path(raw, sp.F32, sp.COSINE, 2051, 16383, 10, 128) == [("scan", None)] * 2
    assert sp.chunk_path(raw, sp.F32, sp.COSINE, 300, 20000, 65, 128) == [("scan", None)]
    assert sp.chunk_path(raw, sp.F32, sp.COSINE, 1024, 20000, 64, 128, ts_s8=1) == [("s8", 16384)]
    assert sp.chunk_path(raw, sp.F32, sp.COSINE, 40, 20000, 10, 64, exact_only=True) == [("scan", None)]
    assert sp.chunk_path(raw, sp.F32, sp.COSINE, 40, 20000, 10, 64, n_deleted=5) == [("scan", None)]
    assert sp.chunk_path(raw, sp.F32, sp.COSINE, 40, 20000, 10, 64, n_deleted=5, flags=sp.TENSOR_WITH_DELETED) == [("f16", 32768)]
    assert sp.chunk_path(codes, sp.U8, sp.EUCLIDEAN, 40, 20000, 10, 64) == [("scan", None)]
    assert sp.chunk_path(codes, sp.U8, sp.COSINE, 4097, 20000, 10, 64) == [("u8", 2048)] * 2 + [("u8", 16384)]
    assert sp.chunk_path(codes, sp.U8, sp.DOT, 40, 20000, 10, 32897) == [("scan", None)]          # s32 bound past a finite float
    assert sp.chunk_path(codes, sp.F16, sp.COSINE, 40, 20000, 10, 64) == [("scan", None)]
    assert sp.chunk_path(sp.HNSW, sp.F32, sp.COSINE, 2049, 100, 1024, 64) == [("hnsw", None)] * 2


def test_gpu_cases_reach_every_final_kernel_cap_class_and_fallback():
    kernels, caps, branches, fallbacks, spans = set(), set(), set(), set(), set()
    for c in sp.CASES:
        paths = sp.shard_paths(c)
        if c["crowded"]:
            assert c["crowded"] < c["nq"] <= sp.CH and c["prefilter_k"] < 300      # the crowded block overflows every list
            for s in paths:
                if s[0][0] != "scan":
                    fallbacks.add((s[0][0], sp.fallback_kind(c)))
        for r, s in enumerate(paths):
            if len(s) > 1:
                spans.add(s[0][0])
            st = None if c["mode"] == sp.RAW else c["st"]
            plan = scan_plan(st, c["metric"], c["dim"], c["shards"][r], c["nq"], c["k"], sp.H100_SMS)
            for (kern, cap), (_, _, branch) in zip(s, plan):
                kernels.add(kern)
                if cap is not None:
                    caps.add(("u8" if kern == "u8" else "prefilter", cap == c["prefilter_k"] or cap))
                if kern == "scan":
                    branches.add(branch)
        # a search mixes final kernels where its shards differ
        if len({s[0][0] for s in paths}) > 1:
            kernels.add("mixed")
    assert kernels == {"f16", "s8", "u8", "scan", "hnsw", "mixed"}
    assert caps == {("prefilter", x) for x in sp.PREFILTER_CAPS + (True,)} | {("u8", x) for x in sp.U8_CAPS + (True,)}
    assert branches == {"rank", "bitonic"}
    assert {("f16", "selective"), ("f16", "whole"), ("s8", "selective"), ("u8", "selective")} <= fallbacks
    assert spans == {"f16", "s8", "u8", "scan", "hnsw"}                          # every kernel across a chunk boundary
    assert any(c["mode"] == sp.HNSW and c["st"] == sp.F32 and c["k"] == 1024 and c["nq"] > sp.CH for c in sp.CASES)
    assert any(c["deleted"] and c["flags"] & sp.TENSOR_WITH_DELETED for c in sp.CASES)
    assert any(c["exact_only"] and min(c["shards"]) >= 16384 for c in sp.CASES)
    assert {c["ids"] for c in sp.CASES} == {"asc", "desc"}
    # world 64 at k = 400 is exactly the merge's shared memory
    assert 64 * 400 * 8 == sp.MERGE_SMEM_MAX < 64 * 401 * 8
