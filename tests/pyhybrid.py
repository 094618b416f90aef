"""Pure-Python restatement of the reference's reciprocal-rank fusion (hybrid_search, repo.rs:168-341, and
batch_hybrid_search, repo.rs:343-555), in numpy float32: one rounding per operation, evaluated left to right, NaN payloads
propagated as x86 SSE does.  A dict stands for the FxHashMap; its order does not matter because of the final sort.  Test
infrastructure only."""
import numpy as np

F32 = np.float32
EPS = F32(np.finfo(np.float32).eps)   # f32::EPSILON


def contribution(rank, k):
    """1.0 / (rank as f32 + k + f32::EPSILON)"""
    with np.errstate(all="ignore"):
        return F32(1.0) / ((F32(rank) + F32(k)) + EPS)


def replica_key(vid, stride):
    """get_raw_emb_by_internal_id (collection.rs:358-384): a replica id maps to id - id % max_replica_per_node"""
    vid = int(vid)
    return vid if stride <= 1 else vid - vid % int(stride)


def total_cmp_key(x):
    """f32::total_cmp as an unsigned key (the library's order_key for a higher-is-better metric)"""
    b = int(np.asarray(x, np.float32).view(np.uint32))
    return (~b & 0xFFFFFFFF) if b & 0x80000000 else b | 0x80000000


def fuse(first, second, k=60.0, form="batch", strides=(1, 1)):
    """first, second: ranked id lists -> [(key, score f32)] of every distinct key, total_cmp descending, ties to the smaller
    id.  form "batch": and_modify(+=).or_insert(score) on the second list; "single": or_insert(0.0).0 += score."""
    k = F32(k)
    scores = {}
    with np.errstate(all="ignore"):
        for rank, vid in enumerate(first):
            scores[replica_key(vid, strides[0])] = contribution(rank, k)
        for rank, vid in enumerate(second):
            key, c = replica_key(vid, strides[1]), contribution(rank, k)
            if form == "batch":
                scores[key] = scores[key] + c if key in scores else c
            else:
                scores[key] = scores.get(key, F32(0.0)) + c
    return sorted(((key, F32(s)) for key, s in scores.items()), key=lambda t: (-total_cmp_key(t[1]), t[0]))


def fuse_batch(first_ids, first_counts, second_ids, second_counts, k=60.0, strides=(1, 1), ld_out=None, form="batch"):
    """row-wise fuse -> (ids u32[B, ld_out], scores f32[B, ld_out], counts u32[B]) in the library's output layout"""
    first_ids, second_ids = np.atleast_2d(first_ids), np.atleast_2d(second_ids)
    nq = first_ids.shape[0]
    ld_out = first_ids.shape[1] + second_ids.shape[1] if ld_out is None else ld_out
    ids = np.full((nq, ld_out), 0xFFFFFFFF, np.uint32)
    scores = np.zeros((nq, ld_out), np.float32)
    counts = np.zeros(nq, np.uint32)
    for q in range(nq):
        na = min(int(first_counts[q]), first_ids.shape[1])
        nb = min(int(second_counts[q]), second_ids.shape[1])
        r = fuse(first_ids[q, :na].tolist(), second_ids[q, :nb].tolist(), k, form, strides)
        counts[q] = len(r)
        for j, (key, s) in enumerate(r):
            ids[q, j] = key
            scores[q, j] = s
    return ids, scores, counts


def association_case(lo=-64.0, hi=0.0, ranks=range(0, 64), seed=5):
    """a fusion constant k (and a rank) for which (rank + k) + eps and rank + (k + eps) round differently in f32, and so do
    their reciprocals: found by a seeded search over k in [lo, hi), -> (k f32, rank)"""
    rng = np.random.default_rng(seed)
    with np.errstate(all="ignore"):
        for _ in range(100000):
            k = F32(rng.uniform(lo, hi))
            for r in ranks:
                left, right = (F32(r) + k) + EPS, F32(r) + (k + EPS)
                if left != right and F32(1.0) / left != F32(1.0) / right:
                    return k, r
    raise AssertionError("no association case found")
