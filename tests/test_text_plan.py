"""The Python restatement of the sparse and TF-IDF search plans (tests/text_plan.py) against the sources it restates: the
constants are read from the .cu files, and the plan formulas' building blocks must still be the drivers' own.  Also pins
the plans that tests/test_gpu_text_limits.py names for its cases.  CPU only."""
import os
import re

from tests import text_plan as tp

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "cosdata_b200", "csrc")


def src(name):
    with open(os.path.join(CSRC, name)) as f:
        return re.sub(r"\s+", " ", f.read())


def test_constants_equal_the_sources():
    c = tp.source_constants()
    assert c["SP_MERGE_KEYS"] == tp.SP_MERGE_KEYS
    assert c["SP_MERGE_MAX_LISTS"] == tp.SP_MERGE_MAX_LISTS
    assert c["SP_MAX_CAND"] == tp.SP_MAX_CAND
    assert c["SP_QCHUNK"] == tp.SP_QCHUNK
    assert c["TF_QCHUNK"] == tp.TF_QCHUNK
    assert c["TF_BUCKETS"] == tp.TF_BUCKETS
    assert c["TILE_SHIFT"] == tp.TILE_SHIFT
    assert c["GROUP_GATHER_BUDGET"] == tp.GROUP_GATHER_BUDGET


def test_driver_formulas_are_the_restated_ones():
    sp, tf, sg = src("sparse.cu"), src("tfidf.cu"), src("shard_group.cu")
    g = "std::min<uint32_t>(SP_MERGE_MAX_LISTS, std::max<uint32_t>(2, SP_MERGE_KEYS / m))"
    assert sp.count(g) == 2                                        # search_locked and merge_lists
    assert "((size_t)n_tiles + n_lvl1) * m * 8 + ((size_t)n_tiles + n_lvl1) * 4" in sp
    assert "(size_t)n_tiles * m * 12" in sp                        # sparse_shard_select
    assert sp.count("std::min<size_t>({(size_t)nq, 65535, (512ull << 20) / per_q})") == 2
    assert "*per_q = (size_t)n_tiles * TF_BUCKETS * sizeof(uint2)" in tf
    assert "std::min<size_t>({(size_t)nq, 65535, (512ull << 20) / *per_q})" in tf
    assert "GROUP_GATHER_BUDGET / (g->world * per_q)" in sg
    assert "group_chunk(g, nq, (size_t)m * 8 + 4)" in sg and "group_chunk(g, nq, 512 * 8)" in sg


def test_merge_groups_and_levels():
    assert tp.merge_group(10) == 63 and tp.merge_group(50) == 63
    assert tp.merge_group(1024) == 25 and tp.merge_group(5000) == 5 and tp.merge_group(5120) == 5
    assert tp.tree_levels(1, 5120) == [] and tp.merge_lists_levels(1, 5120) == [1]
    assert tp.tree_levels(26, 1024) == [2, 1]                      # a last group of one list
    assert tp.tree_levels(5, 5120) == [1]
    assert tp.tree_levels(6, 5120) == [2, 1]
    assert tp.tree_levels(26, 5120) == [6, 2, 1] and tp.tree_levels(26, 5000) == [6, 2, 1]
    assert tp.merge_lists_levels(6, 5120) == [2, 1] and tp.merge_lists_levels(8, 5000) == [2, 1]
    assert tp.merge_lists_levels(11, 5120) == [3, 1]
    assert tp.merge_lists_levels(8, 1024) == [1]
    # the row counts of 26 tiles
    assert tp.n_tiles(819_201) == 26 and tp.n_tiles(851_968) == 26 and tp.n_tiles(851_969) == 27


def test_query_chunks():
    assert tp.chunks(500, tp.sparse_chunk(500, 26, 5120)) == [409, 91]
    assert tp.chunks(1500, tp.sparse_chunk(1500, 7, 5120)) == [1456, 44]
    assert tp.chunks(70_000, tp.sparse_chunk(70_000, 1, 10)) == [65535, 4465]
    assert tp.chunks(70_000, tp.tfidf_chunk(70_000, 1)) == [65535, 4465]
    assert tp.sparse_launches(500, 26, 5120) == 2 * 5 and tp.sparse_launches(70_000, 1, 10) == 2 * 2
    assert tp.tfidf_launches(70_000, 1) == 4 and tp.tfidf_launches(5, 0) == 0
    # a shard group of 8 at m = 5120: two group chunks, and an 11-tile shard splits the first into two of its own
    assert tp.chunks(900, tp.group_chunk(900, 8, 5120 * 8 + 4)) == [819, 81]
    assert tp.chunks(819, tp.shard_select_chunk(819, 11, 5120)) == [794, 25]
    assert tp.chunks(900, tp.group_chunk(900, 6, 5000 * 8 + 4)) == [900]
    assert tp.chunks(900, tp.shard_select_chunk(900, 11, 5000)) == [813, 87]
    # 11 tiles (2 chunks x (1 + 2 levels)), an empty shard, 3 one-tile shards (1 level): selection over 5 ranks, re-rank
    assert tp.sparse_group_launches(900, [11, 0, 1, 1, 1], 5000, True) == 2 * 3 + 3 * 2 + 1 + 6 + 1
