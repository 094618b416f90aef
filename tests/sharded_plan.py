"""Which final kernel writes each shard's packed keys in a sharded dense search, restated from search_chunk_locked
(csrc/api.cu): per 2048-query chunk the fp16 or s8 prefilter with its exact re-rank, the u8 tensor path, HNSW, or the exact
scan (whose merge also runs in selective mode for queries a tensor-core path hands back).  tests/test_sharded_plan.py
pins the constants to the sources and checks that the cases of tests/test_gpu_sharded_edges.py reach every kernel;
the GPU test asserts through each shard's stats() that it took the predicted paths."""
import os
import re

_CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "cosdata_b200", "csrc")

CH = 2048                          # queries per search chunk (search_device_locked)
SCAN_SEL_CAP = 64                  # queries the selective exact scan takes; more -> the whole chunk again
PREFILTER_CAPS = (32768, 16384, 8192)    # candidate slots per query of the prefilter for nq <= 256, <= 1024, above
U8_CAPS = (16384, 4096, 2048)            # the same for the u8 tensor path
MERGE_SMEM_MAX = 200 * 1024        # bytes of merge_gathered_kernel's world * k keys
H100_SMS = 132

# storage types (CDB_ST_*) and metrics (CDB_METRIC_*) by value
U8, SUB1, SUB2, SUB3, F16, F32, BF16 = 0, 1, 2, 3, 4, 5, 6
COSINE, EUCLIDEAN, HAMMING, DOT = 0, 1, 2, 3
RAW, CODES, HNSW = 0, 1, 2         # search modes
TENSOR_WITH_DELETED = 1


def _read(name):
    with open(os.path.join(_CSRC, name)) as f:
        return re.sub(r"\s+", " ", f.read())


def source_plan():
    """the constants above as the sources define them"""
    api, kh = _read("api.cu"), _read("kernels.h")
    m = re.search(r"const uint32_t CH = (\d+); for \(uint32_t off = 0; off < nq; off \+= CH\)", api)
    assert m, "search_device_locked's chunk loop not found"
    sel = re.search(r"constexpr uint32_t SCAN_SEL_CAP = (\d+);", kh)
    assert sel, "SCAN_SEL_CAP not found"
    caps = re.findall(r"const uint32_t cap = p->prefilter_k \? p->prefilter_k : \(nq <= 256 \? (\d+)u : \(nq <= 1024 \? (\d+)u : (\d+)u\)\);", api)
    assert len(caps) == 2, "the two candidate-cap lines of search_chunk_locked not found"
    sg = _read("shard_group.cu")
    mm = re.search(r"constexpr size_t MERGE_SMEM_MAX = (\d+) \* 1024;", sg)
    assert mm, "MERGE_SMEM_MAX not found"
    return {"CH": int(m.group(1)), "SCAN_SEL_CAP": int(sel.group(1)), "PREFILTER_CAPS": tuple(int(c) for c in caps[0]),
            "U8_CAPS": tuple(int(c) for c in caps[1]), "MERGE_SMEM_MAX": int(mm.group(1)) * 1024}


def cap_class(caps, nq, prefilter_k):
    return prefilter_k if prefilter_k else (caps[0] if nq <= 256 else (caps[1] if nq <= 1024 else caps[2]))


def chunk_path(mode, st, metric, nq, size, k, dim, exact_only=False, prefilter_k=0, n_deleted=0, flags=0, ts_s8=0,
               has_shadow=True, sms=H100_SMS):
    """-> [(kernel, candidate cap or None)] per chunk of one shard's search; kernel is one of "f16", "s8" (prefilter and
    exact re-rank), "u8" (u8 tensor path), "scan" (exact scan only), "hnsw".  ts_s8 is the CDB_TS_S8 value the search runs
    under (0 or 1; both GPU and plan cases set it), has_shadow whether the shard keeps the prefilter's fp16/s8 shadow (raw
    f32 rows and tensor_prefilter).  Shards are assumed to hold no degenerate rows."""
    out = []
    del_ok = n_deleted == 0 or bool(flags & TENSOR_WITH_DELETED)
    for off in range(0, nq, CH):
        m = min(CH, nq - off)
        if mode == HNSW:
            out.append(("hnsw", None))
            continue
        raw = mode == RAW
        tensor = (raw and has_shadow and not exact_only and del_ok and m >= 4 and size >= 16384 and k <= 64
                  and size >= k + n_deleted and (m + 127) // 128 <= sms)
        if tensor:
            out.append(("s8" if ts_s8 else "f16", cap_class(PREFILTER_CAPS, m, prefilter_k)))
            continue
        max_digit = 255 if st == U8 else ((1 << st) - 1 if st in (SUB1, SUB2, SUB3) else 0)
        u8 = (not raw and max_digit and not exact_only and del_ok and metric in (COSINE, DOT)
              and max_digit * max_digit * dim <= 0x7F7FFFFF and size >= 16384 and k <= 64 and (m + 127) // 128 <= sms)
        out.append(("u8", cap_class(U8_CAPS, m, prefilter_k)) if u8 else ("scan", None))
    return out


# ----------------------------------------------------------------------------- the GPU cases
# Every case: one loopback group; `shards` = rows per slot (slot order), `ids` "asc" (slot 0 holds the smallest ids) or
# "desc" (slot 0 the largest, so slot order and id order disagree); `crowded` = queries aimed at a block of duplicated
# rows on every shard, so many candidates tie that each such query overflows the candidate list of prefilter_k slots;
# `deleted` = rows deleted on the last shard.
def case(name, shards, mode=RAW, st=F32, metric=COSINE, dim=64, nq=5, k=10, exact_only=False, prefilter_k=0, deleted=0,
         flags=0, ts_s8=0, ids="asc", crowded=0):
    return dict(name=name, shards=list(shards), mode=mode, st=st, metric=metric, dim=dim, nq=nq, k=k, exact_only=exact_only,
                prefilter_k=prefilter_k, deleted=deleted, flags=flags, ts_s8=ts_s8, ids=ids, crowded=crowded)


BIG = 16384
CASES = [
    # raw cosine across a chunk boundary: 2048 queries on the fp16 prefilter, the last 3 on the exact scan; a third slot
    # too small for the prefilter scans both chunks
    case("raw-2051-f16", [BIG + 700, BIG, 5000], dim=128, nq=CH + 3, ids="desc"),
    case("raw-2051-s8", [BIG, BIG + 300], dim=128, nq=CH + 3, ts_s8=1),
    case("raw-300-s8", [BIG + 1, BIG + 2, 900], dim=96, nq=300, ts_s8=1, k=64),
    case("raw-200-f16", [BIG, BIG + 5], dim=64, nq=200, k=1, ids="desc"),
    # some queries hand back to the selective exact scan, then more than SCAN_SEL_CAP: the whole batch again
    case("raw-fallback-selective", [BIG + 400, BIG + 400], dim=64, nq=40, prefilter_k=256, crowded=5),
    case("raw-fallback-whole", [BIG + 400, BIG + 400], dim=64, nq=100, prefilter_k=256, crowded=70, ids="desc"),
    case("raw-fallback-selective-s8", [BIG + 400, BIG + 400], dim=64, nq=40, prefilter_k=256, crowded=3, ts_s8=1),
    # u8 tensor path across cap classes and a chunk boundary
    case("u8-2049", [BIG, BIG + 2000], mode=CODES, st=U8, metric=COSINE, dim=64, nq=CH + 1, ids="desc"),
    case("sub2-2049", [BIG + 17, BIG], mode=CODES, st=SUB2, metric=DOT, dim=128, nq=CH + 1),
    case("u8-600", [BIG, 3000, BIG], mode=CODES, st=U8, metric=DOT, dim=80, nq=600, k=33),
    case("u8-fallback-selective", [BIG + 400, BIG + 400], mode=CODES, st=U8, metric=COSINE, dim=64, nq=40, prefilter_k=256,
         crowded=4),
    # the exact scan only
    case("raw-exact-only", [BIG, BIG + 1000], dim=64, nq=20, k=64, exact_only=True, ids="desc"),
    case("raw-exact-k1024", [3000, 2000, 4000], dim=32, nq=5, k=1024),
    case("raw-exact-k1", [3000, 2000, 4000], dim=32, nq=7, k=1, ids="desc"),
    case("euclid-u8-k65", [3000, 2500], mode=CODES, st=U8, metric=EUCLIDEAN, dim=48, nq=9, k=65),
    case("hamming-sub3-k300", [2000, 2600, 1000], mode=CODES, st=SUB3, metric=HAMMING, dim=48, nq=5, k=300, ids="desc"),
    # deleted rows on the last shard: the prefilter with tensor_with_deleted, the exact scan without
    case("raw-deleted-tensor", [BIG, BIG + 100], dim=64, nq=24, deleted=300, flags=TENSOR_WITH_DELETED),
    case("raw-deleted-scan", [BIG, BIG + 100], dim=64, nq=24, deleted=300),
    # HNSW on F32 rows (the sharded-HNSW configuration's storage), k 1024, two chunks
    case("hnsw-f32-2050", [2500, 2300], mode=HNSW, dim=32, nq=CH + 2, k=1024, ids="desc"),
]


def shard_paths(c):
    """[shard][chunk] -> (kernel, cap) of one case"""
    return [chunk_path(c["mode"], c["st"], c["metric"], c["nq"], n, c["k"], c["dim"], c["exact_only"], c["prefilter_k"],
                       c["deleted"] if r == len(c["shards"]) - 1 else 0, c["flags"], c["ts_s8"])
            for r, n in enumerate(c["shards"])]


def fallback_kind(c):
    """how the crowded queries come back: None, "selective" (<= SCAN_SEL_CAP queries) or "whole" (the whole batch again)"""
    if not c["crowded"]:
        return None
    return "selective" if c["crowded"] <= SCAN_SEL_CAP else "whole"
