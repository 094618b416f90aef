"""Synthetic flat HNSW graphs with metadata replica nodes (test infrastructure).

Mirrors the node population the reference creates for a collection with a metadata schema (vector_store.rs:57-250, 485-712):
  * main component:   main root (id u32::MAX) + one base replica per vector (id = i*R, metadata = all-zero dims -> kind Base)
  * pseudo component: pseudo root (id u32::MAX-257, all-ones dims) + pseudo nodes (ids u32::MAX-256.., vector of the pseudo
                      root) + metadata replicas (id = i*R + j, j >= 1, weighted dims, vector of their base row)
Connectivity is random (parity tests only need GPU search == oracle search on the same arrays): every node gets a random level
(p = 1/4 per step), the roots exist on every level, each node links to random nodes of its own component and level."""
import numpy as np

import oracle as orc
from oracle import pyhnsw, pymeta

EMPTY = 0xFFFFFFFF
PSEUDO_ROOT_ID = 0xFFFFFFFF - 257


def schema_patterns(md_dims, n_patterns, rng):
    """dimension vectors of a schema-like collection: md_dims split into power-of-two fields (the set bits of md_dims, widest
    first; the reference sizes each field by nearest_power_of_two(cardinality + 1), metadata/schema.rs), each field absent
    (zeros) or holding a non-zero value id in binary (HIGH_WEIGHT = 1).  Rows are distinct and non-zero."""
    widths = [1 << b for b in reversed(range(md_dims.bit_length())) if (md_dims >> b) & 1]
    out, seen = [], set()
    while len(out) < n_patterns:
        row = []
        for w in widths:
            field = (rng.random(w) < 0.5).astype(np.int32) if rng.random() < 0.75 else np.zeros(w, np.int32)
            row.append(field)
        row = np.concatenate(row)
        if row.any() and row.tobytes() not in seen:
            seen.add(row.tobytes())
            out.append(row)
    return np.stack(out)


def build(n=300, dim=24, md_dims=6, levels=3, nb=8, nb0=16, replicas=4, n_pseudo=9, storage_type=4, metric=0, seed=1,
          patterns=None):
    """patterns: None (random 0/1 rows) or a function (md_dims, n_patterns, rng) -> int32[n_patterns, md_dims], such as
    schema_patterns"""
    rng = np.random.default_rng(seed)
    vecs = orc.synth_matrix(7000 + seed, n + 2, dim)                    # rows n = main root vector, n+1 = pseudo root vector
    codes, mags = orc.quantize_batch(storage_type, vecs)
    # metadata table: row 0 = base dims (zeros), row 1 = pseudo root (ones), then the patterns
    n_patterns = 10
    if patterns is None:
        patterns = (rng.random((n_patterns, md_dims)) < 0.5).astype(np.int32)
        patterns[patterns.sum(axis=1) == 0, 0] = 1
    else:
        patterns = np.asarray(patterns(md_dims, n_patterns, rng), np.int32)
    md_bits = np.concatenate([np.zeros((1, md_dims), np.int32), np.ones((1, md_dims), np.int32), patterns])
    md_mags = np.array([pymeta.metadata_mag(r) for r in md_bits], dtype=np.float32)
    # node population: (id, row, md row, component)
    nodes = [(0xFFFFFFFF, n, EMPTY, 0), (PSEUDO_ROOT_ID, n + 1, 1, 1)]
    for j in range(n_pseudo):
        nodes.append((PSEUDO_ROOT_ID + 1 + j, n + 1, 2 + j % n_patterns, 1))
    for i in range(n):
        nodes.append((i * replicas, i, 0 if i % 3 else EMPTY, 0))         # base replica: zero dims, or no metadata at all
        if i % 2 == 0:
            for j in range(1, 1 + int(rng.integers(1, replicas))):
                nodes.append((i * replicas + j, i, 2 + int(rng.integers(0, n_patterns)), 1))
    nodes = np.array(nodes, dtype=np.int64)
    top = np.zeros(len(nodes), dtype=np.int64)
    top[:2] = levels
    for t in range(2, len(nodes)):
        lv = 0
        while lv < levels and rng.random() < 0.25:
            lv += 1
        top[t] = lv
    node_row, node_id, node_md, adj, child, index_of = [], [], [], [], [], []
    for lv in range(levels + 1):
        members = np.flatnonzero(top >= lv)
        index_of.append({int(t): i for i, t in enumerate(members)})
        node_row.append(nodes[members, 1].astype(np.uint32))
        node_id.append(nodes[members, 0].astype(np.uint32))
        node_md.append(nodes[members, 2].astype(np.uint32))
        width = nb0 if lv == 0 else nb
        a = np.full((len(members), width), EMPTY, dtype=np.uint32)
        comp = nodes[members, 3]
        for i in range(len(members)):
            same = np.flatnonzero(comp == comp[i])
            same = same[same != i]
            if same.size == 0:
                continue
            pick = rng.choice(same, size=min(width, same.size), replace=False)
            slots = rng.permutation(width)[: pick.size]
            keep = rng.random(pick.size) < 0.8                               # leave some slots empty
            a[i, slots[keep]] = pick[keep]
        adj.append(a.reshape(-1))
        child.append(np.array([index_of[lv - 1][int(t)] for t in members], dtype=np.uint32) if lv else np.zeros(len(members), np.uint32))
    fg = pyhnsw.FlatGraph(metric, storage_type, dim, codes, mags, n, levels, nb, nb0, index_of[levels][0], node_row, adj, child)
    mg = pymeta.MdGraph(fg, md_bits, md_mags, node_id, node_md, index_of[levels][1])
    return vecs, mg


def make_queries(vecs, mg, nq, seed=2):
    """queries near stored vectors; per query: None (no filter) or 1-3 filter dim vectors (-1/0/1), some equal to node patterns"""
    rng = np.random.default_rng(seed)
    n = vecs.shape[0] - 2
    q = (vecs[rng.integers(0, n, nq)] + 0.05 * rng.normal(size=(nq, vecs.shape[1]))).astype(np.float32).clip(-0.999, 0.999)
    filters = []
    for i in range(nq):
        if i % 4 == 0:
            filters.append(None)
            continue
        fs = []
        for _ in range(1 + i % 3):
            if rng.random() < 0.7:
                fs.append(mg.md_bits[2 + int(rng.integers(0, mg.md_bits.shape[0] - 2))].astype(np.int8))
            else:
                fs.append(rng.integers(-1, 2, mg.md_dims).astype(np.int8))
        filters.append(fs)
    return q, filters


def replica_population(n=400, dim=24, md_dims=6, levels=4, n_patterns=7, seed=3, lo=-1.0, hi=1.0, patterns=None):
    """The node list the reference would index for a collection with a metadata schema, in its insertion order
    (vector_store.rs:629-712): pseudo replicas first (created with the collection), then per embedding its base replica
    (base dimensions, mag 0 -> main root) and, for embeddings with metadata fields, one replica per field combination.
    Dimension vectors are 0/1 (HIGH_WEIGHT = 1 binary encodings, metadata/mod.rs:19); pseudo replicas carry the same patterns
    the metadata replicas use, so perfect matches (cs == 1.0) exist.  patterns: None (the binary codes 1..n_patterns) or a
    function like schema_patterns.
    -> dict(vecs f32[n, dim], md_bits, md_mags, row, node_id, base_id, md_row, max_level, main_root_md, pseudo_root_md)"""
    from cosdata_b200.api import level_probs, max_insert_level, pseudo_level_probs
    rng = np.random.default_rng(seed)
    centres = rng.normal(size=(16, dim)).astype(np.float32)
    v = (centres[rng.integers(0, 16, n)] + 0.35 * rng.normal(size=(n, dim))).astype(np.float32)
    vecs = (v / (np.abs(v).max() * 1.01) * max(abs(lo), abs(hi))).astype(np.float32)
    if patterns is None:
        patterns = np.zeros((n_patterns, md_dims), np.int32)
        for p in range(n_patterns):                                     # distinct non-zero binary codes
            code = p + 1
            patterns[p] = [(code >> b) & 1 for b in range(md_dims)]
    else:
        patterns = np.asarray(patterns(md_dims, n_patterns, np.random.default_rng(seed + 1)), np.int32)
    md_bits = np.concatenate([np.zeros((1, md_dims), np.int32), np.ones((1, md_dims), np.int32), patterns])
    md_mags = np.array([pymeta.metadata_mag(r) for r in md_bits], dtype=np.float32)
    md_mags[0] = 0.0
    row, node_id, base_id, md_row, max_level = [], [], [], [], []
    plp = pseudo_level_probs(levels, n_patterns)
    for j in range(n_patterns):                                         # pseudo_metadata_replicas: ids follow the pseudo root's
        row.append(EMPTY); node_id.append(PSEUDO_ROOT_ID + 1 + j); base_id.append(PSEUDO_ROOT_ID); md_row.append(2 + j)
        max_level.append(max_insert_level(float(np.float32(rng.random())), plp))
    lp = level_probs(levels)
    replicas = 4
    for i in range(n):
        fields = [] if i % 3 == 0 else sorted(set(int(x) for x in rng.integers(0, n_patterns, 1 + i % 2)))
        # prop_metadata_replicas: replica 0 = base dimensions, then one per combination; ids base_id + j
        for j, m in enumerate([0] + [2 + f for f in fields]):
            row.append(i); node_id.append(i * replicas + j); base_id.append(i * replicas); md_row.append(m)
            max_level.append(max_insert_level(float(np.float32(rng.random())), lp))
    return dict(vecs=vecs, md_bits=md_bits, md_mags=md_mags, row=np.array(row, np.uint32), node_id=np.array(node_id, np.uint32),
                base_id=np.array(base_id, np.uint32), md_row=np.array(md_row, np.uint32), max_level=np.array(max_level, np.uint8),
                main_root_md=0, pseudo_root_md=1, n_pseudo=n_patterns)
