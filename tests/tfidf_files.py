"""The reference's TF-IDF index files in Python (TEST INFRASTRUCTURE ONLY): a writer that restates the in-memory
TFIDFIndexRoot with VersionedVec::push_sorted / delete and TFIDFIndexRoot::serialize (src/models/tf_idf_index.rs,
src/models/versioned_vec.rs, src/models/serializer/tf_idf/*.rs) -- serialized_at, is_serialized / is_dirty,
num_entries_serialized, the offset counter starting at 118 -- and a reader that restates TFIDFIndexRoot::deserialize.
Words are u64: doc_id << 32 | tf bits; bit 63 set is a tombstone (1 << 63 | version << 32 | index)."""
import os
import struct

import numpy as np

NONE = 0xFFFFFFFF
MAXW = (1 << 64) - 1
NODE_BYTES = 114
CHUNK = 4


def tf_bits(tf):
    return int(np.float32(tf).view(np.uint32))


def calculate_path(dim):
    """utils.rs calculate_path: the child indices from the root to the node of `dim`"""
    path, rem = [], dim
    while rem > 0:
        i = 0
        while 4 ** (i + 1) <= rem:
            i += 1
        path.append(i)
        rem -= 4 ** i
    return path


class VV:
    """VersionedVec<(u32, f32)>"""

    def __init__(self, version):
        self.version, self.list, self.next, self.serialized_at = version, [], None, None

    def push_sorted(self, version, doc, bits):
        if self.version == version:
            i = len(self.list)
            while i > 0 and (self.list[i - 1] >> 32) > doc:   # (storage >> 32) as u32: tombstones and u64::MAX compare high
                i -= 1
            self.list.insert(i, doc << 32 | bits)
            return
        if self.next is None:
            self.next = VV(version)
        self.next.push_sorted(version, doc, bits)

    def push(self, version, word):
        if self.version == version:
            self.list.append(word)
            return
        if self.next is None:
            self.next = VV(version)
        self.next.push(version, word)

    def _find_and_mark(self, doc):
        for i, w in enumerate(self.list):
            if (w >> 32) == doc:
                self.list[i] = MAXW
                return self.version, i
        return self.next._find_and_mark(doc) if self.next else None

    def _delete_internal(self, version, ins_version, idx):
        if self.version == version:
            if ins_version == self.version:
                del self.list[idx]
            else:
                self.list.append(1 << 63 | ins_version << 32 | idx)
            return
        if self.next is None:
            self.next = VV(version)
        self.next._delete_internal(version, ins_version, idx)

    def delete(self, version, doc):
        hit = self._find_and_mark(doc)
        if hit is not None:
            self._delete_internal(version, *hit)

    def __len__(self):
        return len(self.list) + (len(self.next) if self.next else 0)

    def records(self):
        r = self
        while r:
            yield r
            r = r.next

    def serialize(self, files):
        if self.next is not None:
            nxt_off, nxt_ver = self.next.serialize(files), self.next.version
        else:
            nxt_off, nxt_ver = NONE, NONE
        f = files.idat(self.version)
        if self.serialized_at is not None:
            f[self.serialized_at:self.serialized_at + 8] = struct.pack("<II", nxt_off, nxt_ver)
            return self.serialized_at
        off = len(f)
        f += struct.pack("<IIII", nxt_off, nxt_ver, self.version, len(self.list)) + struct.pack(f"<{len(self.list)}Q", *self.list)
        self.serialized_at = off
        return off


class Node:
    def __init__(self, dim, offset):
        self.dim, self.offset = dim, offset
        self.is_serialized, self.is_dirty = False, True
        self.map = {}            # quotient -> [sequence_idx, VV]
        self.map_len = 0
        self.num_entries_serialized = 0
        self.children = [None] * 16


class Files:
    """the bytes of index-tree.dim and of every <version>.idat"""

    def __init__(self):
        self.dim = bytearray()
        self.data = {}

    def idat(self, v):
        return self.data.setdefault(v, bytearray())

    def write(self, off, b):
        if len(self.dim) < off + len(b):
            self.dim += bytes(off + len(b) - len(self.dim))
        self.dim[off:off + len(b)] = b

    def u32(self, off):
        return struct.unpack_from("<I", self.dim, off)[0]

    def save(self, d):
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, "index-tree.dim"), "wb") as f:
            f.write(self.dim)
        for v, b in self.data.items():
            with open(os.path.join(d, f"{v}.idat"), "wb") as f:
                f.write(b)


class Root:
    """TFIDFIndexRoot in memory, with its files"""

    def __init__(self):
        self.root = Node(0, 4)
        self.counter = NODE_BYTES + 4
        self.n_docs = 0
        self.files = Files()

    def _node(self, dim, create):
        n = self.root
        for i in calculate_path(dim):
            if n.children[i] is None:
                if not create:
                    return None
                n.children[i] = Node(n.dim + 4 ** i, self.counter)
                self.counter += NODE_BYTES
            n = n.children[i]
        return n

    def insert(self, h, bits, doc, version):
        n = self._node(h & 0xFFFF, True)
        q = h >> 16
        if q in n.map:
            n.map[q][1].push_sorted(version, doc, bits)
        else:
            vv = VV(version)
            vv.push(version, doc << 32 | bits)
            n.map[q] = [n.map_len, vv]
            n.map_len += 1
        n.is_dirty = True

    def delete(self, h, doc, version):
        n = self._node(h & 0xFFFF, False)
        if n is None:
            return
        if (h >> 16) in n.map:
            n.map[h >> 16][1].delete(version, doc)
        n.is_dirty = True

    # ---- serialize
    def _data(self, n, cur):
        f = self.files
        lst = sorted(n.map.items(), key=lambda kv: kv[1][0])
        f.write(cur, struct.pack("<H", n.map_len))
        cur += 2
        total = (len(lst) + CHUNK - 1) // CHUNK
        for c in range(total):
            for i in range(c * CHUNK, (c + 1) * CHUNK):
                if n.num_entries_serialized > i:
                    lst[i][1][1].serialize(f)
                elif i < len(lst):
                    q, (_, vv) = lst[i]
                    off = vv.serialize(f)
                    f.write(cur, struct.pack("<HII", q, off, vv.version))
                else:
                    f.write(cur, b"\xff" * 10)
                cur += 10
            if n.num_entries_serialized > (c + 1) * CHUNK:
                cur = f.u32(cur)
            elif c == total - 1:
                f.write(cur, b"\xff" * 4)
            else:
                off = self.counter
                self.counter += 10 * CHUNK + 4
                f.write(cur, struct.pack("<I", off))
                cur = off
        n.num_entries_serialized = len(lst)

    def _children(self, n):
        at = n.offset + 10 * CHUNK + 10
        self.files.write(at, b"\xff" * 64)
        for i, c in enumerate(n.children):
            if c is not None:
                self.files.write(at + 4 * i, struct.pack("<I", self._node_ser(c)))

    def _node_ser(self, n):
        if not n.is_serialized:
            n.is_serialized = True
            self.files.write(n.offset, struct.pack("<I", n.dim))
            self._data(n, n.offset + 4)
        elif n.is_dirty:
            n.is_dirty = False
            self._data(n, n.offset + 4)
        self._children(n)
        return n.offset

    def serialize(self):
        self.files.write(0, struct.pack("<I", self.n_docs & 0xFFFFFFFF))
        self._node_ser(self.root)

    # ---- the in-memory state
    def terms(self):
        """{hash: (df, [(doc, tf bits, version)] live words in list order)}"""
        out = {}

        def walk(n):
            for q, (_, vv) in n.map.items():
                words = [(w >> 32, w & NONE, r.version) for r in vv.records() for w in r.list if w != MAXW and not w >> 63]
                out[q << 16 | n.dim] = (len(vv), words)
            for c in n.children:
                if c is not None:
                    walk(c)
        walk(self.root)
        return out


def deserialize(dim, idat):
    """TFIDFIndexRoot::deserialize over the bytes of index-tree.dim and {version: bytes of <version>.idat}
    -> (N, {hash: (df, [(doc, tf bits, version)])})"""
    n_docs = struct.unpack_from("<I", dim, 0)[0]
    out = {}

    def lst(off, ver):
        vd = {}
        while off != NONE:
            b = idat[ver]
            nxt, nver, v, ln = struct.unpack_from("<IIII", b, off)
            vd[v] = (list(struct.unpack_from(f"<{ln}Q", b, off + 16)), nver)
            off, ver = nxt, nver
        dels = [((w >> 32) & 0x7FFFFFFF, w & NONE) for l, _ in vd.values() for w in l if w >> 63]
        for tv, ti in dels:
            if tv in vd and ti < len(vd[tv][0]):
                vd[tv][0][ti] = MAXW
        return vd

    def node(off):
        d = struct.unpack_from("<I", dim, off)[0]
        map_len = struct.unpack_from("<H", dim, off + 4)[0]
        cur, slots = off + 6, {}
        for c in range((map_len + CHUNK - 1) // CHUNK):
            for i in range(c * CHUNK, (c + 1) * CHUNK):
                if i == map_len:
                    break
                slots[struct.unpack_from("<H", dim, cur)[0]] = struct.unpack_from("<II", dim, cur + 2)
                cur += 10
            nxt = struct.unpack_from("<I", dim, cur)[0]
            if nxt == NONE:
                break
            cur = nxt
        for q, (toff, tver) in slots.items():
            vd = lst(toff, tver)
            chain, cv = [], tver
            while cv in vd:
                chain.append(cv)
                if vd[cv][1] == NONE:
                    break
                cv = vd[cv][1]
            assert chain, "deserialize panics: no record of the slot's version"
            df = sum(len(vd[v][0]) for v in chain)
            words = [(w >> 32, w & NONE, v) for v in chain for w in vd[v][0] if w != MAXW and not w >> 63]
            out[q << 16 | d] = (df, words)
        for i in range(16):
            c = struct.unpack_from("<I", dim, off + 10 * CHUNK + 10 + 4 * i)[0]
            if c != NONE:
                node(c)
    node(4)
    return n_docs, out


def read_dir(d):
    """the bytes of a tf_idf_index directory -> (dim, {version: idat})"""
    dim = open(os.path.join(d, "index-tree.dim"), "rb").read()
    idat = {int(f[:-5]): open(os.path.join(d, f), "rb").read() for f in os.listdir(d) if f.endswith(".idat")}
    return dim, idat


class History:
    """a collection's TF-IDF index driven by documents: ids ascending, N as TFIDFIndex keeps it (+1 per document with text
    inserted, -1 per such document deleted; a document deleted twice, or without text, changes nothing here)"""

    def __init__(self):
        self.root = Root()
        self.docs = {}          # id -> (pairs, counted)
        self.deleted = set()

    def insert(self, doc, pairs, version, counted=True):
        self.docs[doc] = (list(pairs), counted)
        if not counted:
            return
        self.root.n_docs += 1
        for h, tf in pairs:
            self.root.insert(int(h), tf_bits(tf), doc, version)

    def delete(self, doc, version):
        pairs, counted = self.docs[doc]
        if doc in self.deleted or not counted:
            self.deleted.add(doc)
            return
        self.deleted.add(doc)
        self.root.n_docs -= 1
        for h, _ in pairs:
            self.root.delete(int(h), doc, version)

    def flush(self):
        self.root.serialize()

    def save(self, d):
        self.root.files.save(d)


def seeded_history(seed, n_versions=5, docs_per_version=40, vocab_size=12, flush_after=None, special=0.15, deletes=0.2, first_version=1):
    """a seeded history without the quirk -> (History, ops, vocab).  Each version appends documents (ascending ids, some
    without text) and deletes random earlier or same-version documents, some twice.  The files are written after every
    version in flush_after (None: all) and after the last; no operation touches a version once it is written.
    ops: ('append', rows [[(hash, tf)]], counted u8[m], version) / ('delete', ids u32[], version)"""
    from tests.tfidf_data import random_rows
    rng = np.random.default_rng(seed)
    vocab = rng.choice(1 << 31, vocab_size, replace=False).astype(np.uint32)
    hist, ops, n = History(), [], 0
    for v in range(first_version, first_version + n_versions):
        m = int(rng.integers(1, docs_per_version + 1))
        rows, counted = random_rows(rng, m, vocab, special=special)
        ops.append(("append", rows, counted, v))
        for r in range(m):
            hist.insert(n + r, rows[r], v, bool(counted[r]))
        n += m
        k = int(rng.binomial(n, deletes))
        if k:
            ids = rng.choice(n, k, replace=True).astype(np.uint32)
            ops.append(("delete", ids, v))
            for d in ids.tolist():
                hist.delete(d, v)
        if flush_after is None or v in flush_after or v == first_version + n_versions - 1:
            hist.flush()
    return hist, ops, vocab


def write_bulk(d, off, hashes, tfs, n1, deleted):
    """the files TFIDFIndexRoot::serialize writes, once, after documents [0, n1) were inserted at version 1, documents
    [n1, n) at version 2, and then `deleted` (ascending ids below n1) deleted at version 2 -- built with numpy for corpora of
    millions of documents.  Each term's version-1 record has u64::MAX at its deleted documents' words (find_and_mark_deleted),
    its version-2 record the version-2 documents, then a tombstone per deleted document."""
    n = len(off) - 1
    lens = np.diff(np.asarray(off, np.int64))
    doc = np.repeat(np.arange(n, dtype=np.uint64), lens)
    h = np.asarray(hashes, np.uint32)
    bits = np.asarray(tfs, np.float32).view(np.uint32).astype(np.uint64)
    order = np.lexsort((doc, h))
    h, doc, bits = h[order], doc[order], bits[order]
    dead = np.zeros(n, bool)
    dead[np.asarray(deleted, np.int64)] = True
    terms, start = np.unique(h, return_index=True)
    t_of = np.repeat(np.arange(terms.size), np.diff(np.append(start, h.size)))
    v1 = doc < n1
    word = doc << np.uint64(32) | bits
    # version-1 records: the version-1 pairs of each term in id order, dead words u64::MAX
    w1 = np.where(dead[doc[v1].astype(np.int64)], np.uint64(MAXW), word[v1])
    t1 = t_of[v1]
    len1 = np.bincount(t1, minlength=terms.size)
    idx1 = np.arange(t1.size) - np.repeat(np.cumsum(len1) - len1, len1)          # index inside its record
    # version-2 records: the version-2 pairs, then the tombstones of the dead version-1 words
    v2 = ~v1
    dk = dead[doc[v1].astype(np.int64)]
    tomb = np.uint64(1 << 63 | 1 << 32) | idx1[dk].astype(np.uint64)
    t2 = np.concatenate([t_of[v2], t1[dk]])
    w2 = np.concatenate([word[v2], tomb])
    o2 = np.argsort(t2, kind="stable")
    t2, w2 = t2[o2], w2[o2]
    len2 = np.bincount(t2, minlength=terms.size)

    def pack(tlen, tw, version, nxt_off, nxt_ver):
        has = tlen > 0
        sizes = np.where(has, 2 + tlen, 0)
        base = np.cumsum(sizes) - sizes                     # in u64 units
        buf = np.zeros(int(sizes.sum()), np.uint64)
        hb = base[has]
        buf[hb] = nxt_off[has].astype(np.uint64) | nxt_ver[has].astype(np.uint64) << np.uint64(32)
        buf[hb + 1] = np.uint64(version) | tlen[has].astype(np.uint64) << np.uint64(32)
        wpos = np.repeat(base + 2, tlen) + (np.arange(tw.size) - np.repeat(np.cumsum(tlen) - tlen, tlen))
        buf[wpos] = tw
        return buf, (base * 8).astype(np.uint64), has

    none = np.full(terms.size, NONE, np.uint64)
    buf2, boff2, has2 = pack(len2, w2, 2, none, none)
    buf1, boff1, has1 = pack(len1, w1, 1, np.where(has2, boff2, NONE), np.where(has2, 2, NONE))
    os.makedirs(d, exist_ok=True)
    for v, b in ((1, buf1), (2, buf2)):
        if b.size:
            b.tofile(os.path.join(d, f"{v}.idat"))
    # the tree: a node per dim on calculate_path, its slots in overflow chunks of 4
    dim = Files()
    counter = [NODE_BYTES + 4]
    nodes = {0: 4}

    def node(dm):
        if dm in nodes:
            return nodes[dm]
        path, cur = calculate_path(dm), 0
        for i in path:
            nd = cur + 4 ** i
            if nd not in nodes:
                nodes[nd] = counter[0]
                counter[0] += NODE_BYTES
                dim.write(nodes[cur] + 50 + 4 * i, struct.pack("<I", nodes[nd]))
            cur = nd
        return nodes[dm]

    def init(o, dm):
        dim.write(o, struct.pack("<IH", dm, 0) + b"\xff" * 44 + b"\xff" * 64)

    init(4, 0)
    slots = {}
    for t in range(terms.size):
        hh = int(terms[t])
        head = (int(boff1[t]), 1) if has1[t] else (int(boff2[t]), 2)
        slots.setdefault(hh & 0xFFFF, []).append((hh >> 16, *head))
    for dm in sorted(slots):
        before = set(nodes)
        o = node(dm)
        for nd in set(nodes) - before:
            init(nodes[nd], nd)
        sl = slots[dm]
        dim.write(o + 4, struct.pack("<H", len(sl)))
        cur = o + 6
        for c0 in range(0, len(sl), CHUNK):
            for q, so, sv in sl[c0:c0 + CHUNK]:
                dim.write(cur, struct.pack("<HII", q, so, sv))
                cur += 10
            if c0 + CHUNK < len(sl):
                nxt = counter[0]
                counter[0] += 10 * CHUNK + 4
                dim.write(cur + 10 * (CHUNK - len(sl[c0:c0 + CHUNK])), struct.pack("<I", nxt))
                cur = nxt
            else:
                dim.write(cur, b"\xff" * (10 * (CHUNK - len(sl[c0:c0 + CHUNK])) + 4))
    # child links, after every node's bytes exist
    for nd, o in nodes.items():
        if nd == 0:
            continue
        path, cur = calculate_path(nd), 0
        for i in path[:-1]:
            cur += 4 ** i
        dim.write(nodes[cur] + 50 + 4 * path[-1], struct.pack("<I", o))
    dim.write(0, struct.pack("<I", (n - int(dead.sum())) & NONE))
    with open(os.path.join(d, "index-tree.dim"), "wb") as f:
        f.write(dim.dim)


def reference_fixture_script():
    """the history tools/ref_fixtures/b200_fixtures.rs::dump_tfidf_fixtures drives through the reference (keep the two
    identical): three versions, each inserting documents, deleting some (in the same and in earlier versions) and then
    serializing -> History, with its files written the same way"""
    hashes = [q << 16 | dim for dim in (0, 1, 5, 21, 4096, 65535) for q in (0, 1, 2, 3, 4, 5, 0x7FFF, 0xFFFF)]

    def doc_pairs(doc):
        return [(h, -0.0 if (doc + j) % 7 == 0 else ((doc * 7 + j) % 13) * 0.25)
                for j, h in enumerate(hashes) if (doc + j) % 3 == 0]
    h = History()
    for v, d0, d1, deletes in ((1, 0, 8, (2,)), (2, 8, 14, (4, 9)), (3, 14, 18, (10, 15, 0))):
        for doc in range(d0, d1):
            h.insert(doc, doc_pairs(doc), v)
        for doc in deletes:
            h.delete(doc, v)
        h.flush()
    return h


def search_lists(n_docs, terms, queries, k):
    """search_bm25 in the caller's term order (the library's and the oracle's `query` order) straight over deserialized
    lists {hash: (df, [(doc, tf bits, version)])} under N = n_docs, for files no sequence of appends and deletes can
    reproduce (the quirk).  tests/test_tfidf_files.py pins it to the oracle on histories the oracle can replay.
    -> ids u32[B, kout], scores f32[B, kout], counts u32[B]"""
    from tests import pytfidf as pt
    kout = 512 if k == 0 or k > 512 else k
    ids = np.full((len(queries), kout), NONE, np.uint32)
    sc = np.zeros((len(queries), kout), np.float32)
    cnt = np.zeros(len(queries), np.uint32)
    with np.errstate(all="ignore"):
        for qi, q in enumerate(queries):
            acc = {}
            for h in q:
                if h not in terms:
                    continue
                idf = pt.idf(n_docs, terms[h][0])
                for doc, bits, _ in terms[h][1]:
                    p = np.float32(np.uint32(bits).view(np.float32)) * idf
                    acc[doc] = p if doc not in acc else np.float32(acc[doc] + p)
            best = {}
            for doc in sorted(acc):
                s = acc[doc]
                b = best.get(doc % 512)
                if s > (b[1] if b else -np.inf):
                    best[doc % 512] = (doc, s)

            def key(x):
                u = int(np.float32(x[1]).view(np.uint32))
                return (-(u ^ 0xFFFFFFFF if u >> 31 else u | 0x80000000), x[0])
            win = sorted(best.values(), key=key)[:kout]
            cnt[qi] = len(win)
            for j, (doc, s) in enumerate(win):
                ids[qi, j], sc[qi, j] = doc, s
    return ids, sc, cnt
