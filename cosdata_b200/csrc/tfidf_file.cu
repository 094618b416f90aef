// tfidf_file.cu -- reader of the reference's TF-IDF index files: TFIDFIndexRoot::deserialize (src/models/tf_idf_index.rs:369-401,
// src/models/serializer/tf_idf/*.rs) restated over read-only memory maps, with every malformed input refused
// (CDB_INVALID_PARAMS and a message) instead of a panic or an endless walk.  Host-only; cdb_tfidf_index_load_files
// (tfidf.cu) uploads the records this reader keeps.  Format and rules: DESIGN.md section 8d, "Loading the reference's files".
#include <algorithm>
#include <cstring>
#include <map>
#include <string>
#include <unordered_set>

#include "tfidf_file.h"

using cdb::set_error;
using cdb::reffiles::Mapped;

namespace {

constexpr uint32_t NONE = 0xFFFFFFFFu;
constexpr uint64_t NODE_BYTES = 114;    // u32 dim, u16 map_len, 4 x (u16 quotient, u32 offset, u32 version), u32 next, 16 x u32 children
constexpr uint64_t CHILDREN_AT = 50;
constexpr uint32_t CHUNK_SLOTS = 4;     // TF_IDF_INDEX_DATA_CHUNK_SIZE

inline uint16_t rd16(const uint8_t *p) { uint16_t v; memcpy(&v, p, 2); return v; }
inline uint32_t rd32(const uint8_t *p) { uint32_t v; memcpy(&v, p, 4); return v; }
inline uint64_t rd64(const uint8_t *p) { uint64_t v; memcpy(&v, p, 8); return v; }

struct Slot { uint32_t hash, offset, version; };

// one record as read by VersionedVec::deserialize
struct Rec { const uint8_t *words; uint32_t next_ver, version, len; uint32_t order; };

struct Reader {
    const std::string dir;
    cdb_tfidf_files &f;

    cdb_status fail(const std::string &msg) { set_error("tf-idf files: " + msg); return CDB_INVALID_PARAMS; }

    cdb_status idat(uint32_t version, const Mapped **out) {
        auto it = f.idat.find(version);
        if (it == f.idat.end()) {
            std::unique_ptr<Mapped> m(new Mapped());
            const std::string path = dir + "/" + std::to_string(version) + ".idat";
            if (m->open(path.c_str())) return fail("missing " + path);
            it = f.idat.emplace(version, std::move(m)).first;
        }
        *out = it->second.get();
        return CDB_OK;
    }

    // the tree (TFIDFIndexNode / AtomicArray / TFIDFIndexNodeData::deserialize): every term slot, with the replace rule
    cdb_status walk_tree(std::vector<Slot> &slots) {
        const Mapped &d = *f.dim;
        if (d.len < 4 + NODE_BYTES) return fail("index-tree.dim is truncated (no root node)");
        f.n_docs = rd32(d.p);
        struct Pos { uint64_t off; uint32_t dim; int last, run; };   // last child index on the path and how often it repeats
        std::vector<Pos> stack{{4, 0, 16, 0}};
        std::unordered_set<uint64_t> seen;
        while (!stack.empty()) {
            const Pos n = stack.back();
            stack.pop_back();
            if (!seen.insert(n.off).second) return fail("a node is reached twice (child offsets form a cycle)");
            if (n.off + NODE_BYTES > d.len) return fail("a node at offset " + std::to_string(n.off) + " is past the end of index-tree.dim");
            const uint8_t *p = d.p + n.off;
            if (rd32(p) != n.dim) return fail("node at offset " + std::to_string(n.off) + " has dim " + std::to_string(rd32(p)) +
                                               ", its tree position " + std::to_string(n.dim));
            // the node's data: map_len slots, four per chunk, chunks chained by offset; a later slot of a quotient wins
            const uint32_t map_len = rd16(p + 4);
            std::map<uint16_t, Slot> node;
            uint64_t cur = n.off + 6;
            for (uint32_t c = 0, i = 0; c < (map_len + CHUNK_SLOTS - 1) / CHUNK_SLOTS; ++c) {
                for (uint32_t j = 0; j < CHUNK_SLOTS && i < map_len; ++j, ++i) {
                    if (cur + 10 > d.len) return fail("a term slot is past the end of index-tree.dim");
                    const uint16_t q = rd16(d.p + cur);
                    node[q] = Slot{(uint32_t)q << 16 | n.dim, rd32(d.p + cur + 2), rd32(d.p + cur + 6)};
                    cur += 10;
                }
                if (cur + 4 > d.len) return fail("a chunk link is past the end of index-tree.dim");
                const uint32_t next = rd32(d.p + cur);
                if (next == NONE) break;
                cur = next;
            }
            for (const auto &kv : node) slots.push_back(kv.second);
            // children: child i has dim + 4^i; the reference creates a node only on calculate_path's path (child indices
            // non-increasing, each repeated at most 3 times), which also makes every dim unique
            for (int i = 0; i < 16; ++i) {
                const uint32_t off = rd32(p + CHILDREN_AT + 4 * i);
                if (off == NONE) continue;
                const uint64_t dim = (uint64_t)n.dim + (1ull << (2 * i));
                if (dim >= 65536) return fail("a child of the node of dim " + std::to_string(n.dim) + " would have a dim of 2^16 or more");
                if (i > n.last || (i == n.last && n.run >= 3)) return fail("a node off its dim's path (calculate_path) at offset " + std::to_string(off));
                stack.push_back({off, (uint32_t)dim, i, i == n.last ? n.run + 1 : 1});
            }
        }
        std::sort(slots.begin(), slots.end(), [](const Slot &a, const Slot &b) { return a.hash < b.hash; });
        return CDB_OK;
    }

    // one term's list (VersionedVec::deserialize): read the chain, key records by their version (a later one replaces),
    // collect every tombstone, apply them, then rebuild the chain from the slot's version
    cdb_status read_list(const Slot &s, uint32_t term, std::vector<Rec> &rd, std::vector<Rec> &chain, std::vector<uint64_t> &kills) {
        rd.clear();
        chain.clear();
        std::unordered_set<uint64_t> visited;   // (file version, offset) of every record read
        uint32_t off = s.offset, ver = s.version;
        while (off != NONE) {
            const Mapped *m = nullptr;
            cdb_status rc = idat(ver, &m);
            if (rc) return rc;
            if ((uint64_t)off + 16 > m->len) return fail("a list record at offset " + std::to_string(off) + " of " + std::to_string(ver) + ".idat is past its end");
            const uint8_t *p = m->p + off;
            const uint32_t len = rd32(p + 12);
            if ((uint64_t)off + 16 + 8ull * len > m->len) return fail("a list record of " + std::to_string(ver) + ".idat is truncated");
            if (!visited.insert((uint64_t)ver << 32 | off).second) return fail("a list's records form a cycle");
            rd.push_back(Rec{p + 16, rd32(p + 4), rd32(p + 8), len, (uint32_t)rd.size()});
            off = rd32(p);
            ver = rd32(p + 4);
        }
        // version_data: the last record read of each version
        std::stable_sort(rd.begin(), rd.end(), [](const Rec &a, const Rec &b) { return a.version < b.version; });
        size_t w = 0;
        for (size_t i = 0; i < rd.size(); ++i) {
            if (w && rd[w - 1].version == rd[i].version) rd[w - 1] = rd[i];
            else rd[w++] = rd[i];
        }
        rd.resize(w);
        auto find = [&](uint32_t v) -> const Rec * {
            auto it = std::lower_bound(rd.begin(), rd.end(), v, [](const Rec &r, uint32_t x) { return r.version < x; });
            return it != rd.end() && it->version == v ? &*it : nullptr;
        };
        // the chain from the slot's version
        for (const Rec *r = find(s.version); r; r = r->next_ver == NONE ? nullptr : find(r->next_ver)) {
            if (chain.size() == rd.size()) return fail("a list's versions form a cycle");
            chain.push_back(*r);
        }
        if (chain.empty()) return fail("term " + std::to_string(s.hash) + ": no record of its slot's version " + std::to_string(s.version));
        // tombstones of every record kept, applied to the records of the chain (a record outside it is dropped anyway)
        std::vector<uint64_t> base(chain.size());
        uint64_t b = f.n_words;
        for (size_t c = 0; c < chain.size(); ++c) { base[c] = b; b += chain[c].len; }
        const size_t k0 = kills.size();
        for (const Rec &r : rd)
            for (uint32_t i = 0; i < r.len; ++i) {
                const uint64_t x = rd64(r.words + 8ull * i);
                if (!(x >> 63)) continue;
                const uint32_t tv = (uint32_t)(x >> 32) & 0x7FFFFFFFu, ti = (uint32_t)x;
                for (size_t c = 0; c < chain.size(); ++c)
                    if (chain[c].version == tv) { if (ti < chain[c].len) kills.push_back(base[c] + ti); break; }
            }
        std::sort(kills.begin() + k0, kills.end());
        kills.erase(std::unique(kills.begin() + k0, kills.end()), kills.end());
        // the kept records, df, and the live words
        uint64_t df = 0;
        size_t k = k0;
        for (size_t c = 0; c < chain.size(); ++c) {
            const Rec &r = chain[c];
            f.recs.push_back(TfIdfFileRecord{r.words, base[c], r.len, term, r.version});
            f.max_version = std::max(f.max_version, r.version);
            df += r.len;
            for (uint32_t i = 0; i < r.len; ++i) {
                if (k < kills.size() && kills[k] == base[c] + i) { ++k; continue; }
                const uint64_t x = rd64(r.words + 8ull * i);
                if (x == ~0ull || (x >> 63)) continue;
                ++f.n_live;
                f.max_id_end = std::max<uint64_t>(f.max_id_end, (x >> 32) + 1);
            }
        }
        if (df > NONE) return fail("term " + std::to_string(s.hash) + " has 2^32 words or more");
        f.df.push_back((uint32_t)df);
        f.n_words = b;
        return CDB_OK;
    }

    cdb_status run() {
        f.dim.reset(new Mapped());
        const std::string path = dir + "/index-tree.dim";
        if (f.dim->open(path.c_str())) return fail("missing " + path);
        std::vector<Slot> slots;
        cdb_status rc = walk_tree(slots);
        if (rc) return rc;
        std::vector<Rec> rd, chain;
        f.rec_begin.push_back(0);
        for (size_t t = 0; t < slots.size(); ++t) {
            f.hashes.push_back(slots[t].hash);
            if ((rc = read_list(slots[t], (uint32_t)t, rd, chain, f.killed))) return rc;
            f.rec_begin.push_back(f.recs.size());
        }
        return CDB_OK;
    }
};

}  // namespace

extern "C" {

cdb_status cdb_tfidf_files_open(const char *dir, cdb_tfidf_files **out) {
    if (!dir || !out) { set_error("null argument"); return CDB_INVALID_PARAMS; }
    *out = nullptr;
    std::unique_ptr<cdb_tfidf_files> f(new cdb_tfidf_files());
    Reader r{dir, *f};
    const cdb_status rc = r.run();
    if (rc) return rc;
    *out = f.release();
    return CDB_OK;
}

cdb_status cdb_tfidf_files_close(cdb_tfidf_files *files) {
    delete files;
    return CDB_OK;
}

cdb_status cdb_tfidf_files_info(const cdb_tfidf_files *f, uint64_t *info) {
    if (!f || !info) { set_error("null argument"); return CDB_INVALID_PARAMS; }
    info[0] = f->n_docs;
    info[1] = f->hashes.size();
    info[2] = f->recs.size();
    info[3] = f->n_live;
    info[4] = f->max_id_end;
    info[5] = f->max_version;
    return CDB_OK;
}

cdb_status cdb_tfidf_files_read(const cdb_tfidf_files *f, uint32_t *hashes, uint32_t *df, uint64_t *offsets, uint32_t *doc_ids, float *tfs,
                                uint32_t *versions) {
    if (!f) { set_error("null argument"); return CDB_INVALID_PARAMS; }
    const size_t nt = f->hashes.size();
    if (hashes && nt) memcpy(hashes, f->hashes.data(), nt * 4);
    if (df && nt) memcpy(df, f->df.data(), nt * 4);
    uint64_t o = 0;
    size_t k = 0;
    if (offsets) offsets[0] = 0;
    for (size_t t = 0; t < nt; ++t) {
        for (uint64_t ri = f->rec_begin[t]; ri < f->rec_begin[t + 1]; ++ri) {
            const TfIdfFileRecord &r = f->recs[ri];
            for (uint32_t i = 0; i < r.len; ++i) {
                while (k < f->killed.size() && f->killed[k] < r.base + i) ++k;
                if (k < f->killed.size() && f->killed[k] == r.base + i) continue;
                const uint64_t x = rd64(r.words + 8ull * i);
                if (x == ~0ull || (x >> 63)) continue;
                if (doc_ids) doc_ids[o] = (uint32_t)(x >> 32);
                if (tfs) { const uint32_t bits = (uint32_t)x; memcpy(tfs + o, &bits, 4); }
                if (versions) versions[o] = r.version;
                ++o;
            }
        }
        if (offsets) offsets[t + 1] = o;
    }
    return CDB_OK;
}

}  // extern "C"
