// itoe_file.cu -- host-side reader for the reference's raw-embedding store (no device code here).
//
// Collection::internal_to_external_map is a TreeMap<InternalId, RawVectorEmbedding> (src/models/collection.rs:110) persisted
// as `itoe.dim` + one `itoe.<version>.data` per version (collection.rs:149-164).  finalize_ann_results reads the raw f32
// vectors for the exact re-rank from it (get_raw_emb_by_internal_id, collection.rs:368-384).  Format, all little endian:
//   itoe.dim    [0..4)   u32 offset of the root TreeMapNode                             (tree_map.rs:548-560, 563-570)
//   TreeMapNode          u16 node_idx | 8 x u32 child offset (u32::MAX = none) | u32 quotients offset
//                                                                                      (serializer/tree_map/node.rs:72-87)
//   QuotientsMap         u64 len | chunks of 4 x (u64 key, u32 item offset, u32 item version) + u32 next chunk offset
//                        (u32::MAX = last); unused slots are 0xFF                        (quotients_map.rs:182-267)
//   VersionedItem        in itoe.<version>.data: u32 next offset | u32 next version | u32 version | u32 value offset
//                        (u32::MAX = deleted); the newest state is the end of the `next` chain
//                                                                                      (versioned_item.rs:52-110, tree_map.rs:262-268)
//   RawVectorEmbedding   varint id len + id | varint doc-id len + bytes | varint dense_len + dense_len x f32 | metadata |
//                        sparse pairs | text                                            (raw_vector_embedding.rs:15-143)
//   varint               1-3 bytes, 7+7+8 bits                                          (serializer/mod.rs:25-57)
// A key lives in the node reached by calculate_path(key % 65536, 0) (models/utils.rs:3-24, tree_map.rs:512-518); the
// enumeration below walks every node instead, the point lookup follows that path.
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "kernels.h"

namespace cdb {
namespace {

struct MappedFile {
    const uint8_t *p = nullptr;
    size_t len = 0;
    bool open(const std::string &path) {
        int fd = ::open(path.c_str(), O_RDONLY);
        if (fd < 0) return false;
        struct stat st;
        if (fstat(fd, &st) != 0) { ::close(fd); return false; }
        len = (size_t)st.st_size;
        if (len) {
            void *m = mmap(nullptr, len, PROT_READ, MAP_PRIVATE, fd, 0);
            if (m == MAP_FAILED) { ::close(fd); len = 0; return false; }
            p = static_cast<const uint8_t *>(m);
        }
        ::close(fd);
        return true;
    }
    ~MappedFile() { if (p) munmap(const_cast<uint8_t *>(p), len); }
    bool has(uint64_t off, uint64_t n) const { return off <= len && n <= len - off; }
    uint16_t u16(uint64_t o) const { uint16_t v; memcpy(&v, p + o, 2); return v; }
    uint32_t u32(uint64_t o) const { uint32_t v; memcpy(&v, p + o, 4); return v; }
    uint64_t u64(uint64_t o) const { uint64_t v; memcpy(&v, p + o, 8); return v; }
};

// dense values (and, when the store reads sparse values, the (u32 dim, f32 value) pairs) inside itoe.<version>.data
struct Entry { uint64_t key; uint32_t version; uint64_t dense_off; uint32_t dense_len; uint64_t sparse_off = 0; uint32_t sparse_len = 0; };

struct ItoeStore {
    std::string dir;
    MappedFile dim;
    std::map<uint32_t, std::unique_ptr<MappedFile>> data;
    std::string err;
    bool sparse = false;   // parse past the metadata to the sparse pairs; enumerate embeddings that have them

    bool fail(const std::string &m) { if (err.empty()) err = m; return false; }

    const MappedFile *data_file(uint32_t version) {
        auto it = data.find(version);
        if (it != data.end()) return it->second.get();
        std::unique_ptr<MappedFile> f(new MappedFile());
        if (!f->open(dir + "/itoe." + std::to_string(version) + ".data")) { fail("cannot open itoe." + std::to_string(version) + ".data"); return nullptr; }
        return (data[version] = std::move(f)).get();
    }

    static bool read_len(const MappedFile &f, uint64_t &o, uint32_t &v) {   // serializer/mod.rs:42-57
        if (!f.has(o, 1)) return false;
        const uint32_t b0 = f.p[o++];
        if (!(b0 & 0x80)) { v = b0; return true; }
        if (!f.has(o, 1)) return false;
        const uint32_t b1 = f.p[o++];
        const uint32_t low14 = (b0 & 0x7F) | ((b1 & 0x7F) << 7);
        if (!(b1 & 0x80)) { v = low14; return true; }
        if (!f.has(o, 1)) return false;
        v = low14 | ((uint32_t)f.p[o++] << 14);
        return true;
    }

    // newest state of the VersionedItem chain starting at (offset, version): false = error, e.dense_len == 0 = no dense vector
    bool latest(uint32_t offset, uint32_t version, Entry &e) {
        uint32_t value_off = UINT32_MAX, value_version = version;
        for (int hops = 0;; ++hops) {
            if (hops > (1 << 20)) return fail("VersionedItem chain does not end");
            const MappedFile *f = data_file(version);
            if (!f) return false;
            if (!f->has(offset, 16)) return fail("VersionedItem outside itoe." + std::to_string(version) + ".data");
            const uint32_t next_off = f->u32(offset), next_ver = f->u32(offset + 4);
            value_off = f->u32(offset + 12);
            value_version = version;
            if (next_off == UINT32_MAX) break;
            offset = next_off; version = next_ver;
        }
        e.version = value_version; e.dense_off = 0; e.dense_len = 0;
        if (value_off == UINT32_MAX) return true;                       // deleted (tree_map.rs:237-244)
        const MappedFile *f = data_file(value_version);
        if (!f) return false;
        uint64_t o = value_off;
        uint32_t n;
        if (!read_len(*f, o, n) || !f->has(o, n)) return fail("truncated RawVectorEmbedding id");
        o += n;
        if (!read_len(*f, o, n) || !f->has(o, n)) return fail("truncated RawVectorEmbedding document id");
        o += n;
        if (!read_len(*f, o, n) || !f->has(o, (uint64_t)n * 4)) return fail("truncated RawVectorEmbedding dense values");
        e.dense_off = o; e.dense_len = n;
        if (!sparse) return true;
        o += (uint64_t)n * 4;
        uint32_t n_md;                                                   // raw_vector_embedding.rs:91-116
        if (!read_len(*f, o, n_md)) return fail("truncated RawVectorEmbedding metadata");
        for (uint32_t i = 0; i < n_md; ++i) {
            if (!read_len(*f, o, n) || !f->has(o, n)) return fail("truncated RawVectorEmbedding metadata field");
            o += n;
            if (!f->has(o, 1)) return fail("truncated RawVectorEmbedding metadata value");
            const uint8_t variant = f->p[o++];
            if (variant == 0) {
                if (!f->has(o, 4)) return fail("truncated RawVectorEmbedding metadata value");
                o += 4;
            } else if (variant == 1) {
                if (!read_len(*f, o, n) || !f->has(o, n)) return fail("truncated RawVectorEmbedding metadata value");
                o += n;
            } else {
                return fail("invalid FieldValue variant " + std::to_string(variant));
            }
        }
        if (!read_len(*f, o, n) || !f->has(o, (uint64_t)n * 8)) return fail("truncated RawVectorEmbedding sparse values");
        e.sparse_off = o; e.sparse_len = n;                             // raw_vector_embedding.rs:118-132
        return true;
    }

    bool quotients(uint32_t off, std::vector<Entry> *out, const uint64_t *want_key, Entry *found, bool *hit) {
        if (off == UINT32_MAX) return true;
        if (!dim.has(off, 8)) return fail("QuotientsMap outside itoe.dim");
        const uint64_t len = dim.u64(off);
        uint64_t o = (uint64_t)off + 8, chunks = 0;
        for (uint64_t i = 0; i < len;) {
            if (++chunks > dim.len / 68 + 1) return fail("QuotientsMap chunk chain does not end");   // a damaged next pointer
            if (!dim.has(o, 4 * 16 + 4)) return fail("QuotientsMap chunk outside itoe.dim");
            for (int s = 0; s < 4 && i < len; ++s, ++i) {
                const uint64_t key = dim.u64(o + s * 16);
                const uint32_t ioff = dim.u32(o + s * 16 + 8), iver = dim.u32(o + s * 16 + 12);
                if (want_key && key != *want_key) continue;
                Entry e; e.key = key;
                if (!latest(ioff, iver, e)) return false;
                if (want_key) { *found = e; *hit = true; return true; }
                if (sparse ? e.sparse_len : e.dense_len) out->push_back(e);
            }
            const uint32_t next = dim.u32(o + 64);
            if (next == UINT32_MAX) break;
            o = next;
        }
        return true;
    }

    std::vector<uint32_t> seen_nodes;
    bool walk(uint32_t node_off, std::vector<Entry> &out, int depth) {
        if (depth > 64) return fail("TreeMapNode nesting too deep");   // a path has at most 3 hops per power of 4: 24
        if (!dim.has(node_off, 38)) return fail("TreeMapNode outside itoe.dim");
        if (seen_nodes.size() > dim.len / 38 + 1) return fail("TreeMapNode links form a cycle");   // more visits than nodes fit in the file
        seen_nodes.push_back(node_off);
        if (!quotients(dim.u32((uint64_t)node_off + 34), &out, nullptr, nullptr, nullptr)) return false;
        for (int c = 0; c < 8; ++c) {
            const uint32_t child = dim.u32((uint64_t)node_off + 2 + c * 4);
            if (child != UINT32_MAX && !walk(child, out, depth + 1)) return false;
        }
        return true;
    }

    bool open(const char *d) {
        dir = d;
        if (!dim.open(dir + "/itoe.dim")) return fail("cannot open " + dir + "/itoe.dim");
        return true;
    }
    // every live key with dense values, ascending by key
    bool enumerate(std::vector<Entry> &out) {
        if (dim.len == 0) return true;                                   // never serialized
        if (!dim.has(0, 4)) return fail("itoe.dim shorter than its header");
        const uint32_t root = dim.u32(0);
        if (root == UINT32_MAX) return true;
        if (!walk(root, out, 0)) return false;
        std::sort(out.begin(), out.end(), [](const Entry &a, const Entry &b) { return a.key < b.key; });
        return true;
    }
    // TreeMap::get_latest (tree_map.rs:528-534): follow calculate_path(key % 65536, 0)
    bool lookup(uint64_t key, Entry &e, bool &hit) {
        hit = false;
        if (dim.len < 4 || dim.u32(0) == UINT32_MAX) return true;
        uint32_t node = dim.u32(0);
        uint32_t remaining = (uint32_t)(key % 65536);
        while (remaining > 0) {
            const uint32_t msb = 31 - (uint32_t)__builtin_clz(remaining), power = msb / 2;   // largest_power_of_4_below
            if (!dim.has(node, 38)) return fail("TreeMapNode outside itoe.dim");
            node = dim.u32((uint64_t)node + 2 + power * 4);
            if (node == UINT32_MAX) return true;
            remaining -= 1u << (power * 2);
        }
        if (!dim.has(node, 38)) return fail("TreeMapNode outside itoe.dim");
        return quotients(dim.u32((uint64_t)node + 34), nullptr, &key, &e, &hit);
    }
    void copy_dense(const Entry &e, float *dst) { memcpy(dst, data_file(e.version)->p + e.dense_off, (size_t)e.dense_len * 4); }
    void copy_sparse(const Entry &e, uint32_t *dims, float *vals) {
        const uint8_t *p = data_file(e.version)->p + e.sparse_off;
        for (uint32_t i = 0; i < e.sparse_len; ++i) { memcpy(dims + i, p + 8 * i, 4); memcpy(vals + i, p + 8 * i + 4, 4); }
    }
};

cdb_status store_error(const ItoeStore &s) {
    set_error("itoe store: " + s.err);
    return CDB_INVALID_PARAMS;
}

}  // namespace
}  // namespace cdb

using namespace cdb;

extern "C" {

cdb_status cdb_itoe_scan(const char *collection_dir, uint64_t *out_entries, uint32_t *out_dim, uint64_t *out_max_internal_id) {
    if (!collection_dir) { set_error("null path"); return CDB_INVALID_PARAMS; }
    ItoeStore s;
    std::vector<Entry> es;
    if (!s.open(collection_dir) || !s.enumerate(es)) return store_error(s);
    for (const Entry &e : es)
        if (e.dense_len != es[0].dense_len) { set_error("itoe store: dense vectors differ in length"); return CDB_STORAGE_MISMATCH; }
    if (out_entries) *out_entries = es.size();
    if (out_dim) *out_dim = es.empty() ? 0 : es[0].dense_len;
    if (out_max_internal_id) *out_max_internal_id = es.empty() ? 0 : es.back().key;
    return CDB_OK;
}

cdb_status cdb_itoe_load(const char *collection_dir, uint64_t first_entry, uint64_t max_entries, uint32_t *out_internal_ids,
                         float *out_vectors, uint64_t *out_read) {
    if (!collection_dir || !out_read) { set_error("null argument"); return CDB_INVALID_PARAMS; }
    ItoeStore s;
    std::vector<Entry> es;
    if (!s.open(collection_dir) || !s.enumerate(es)) return store_error(s);
    uint64_t got = 0;
    for (uint64_t i = first_entry; i < es.size() && got < max_entries; ++i, ++got) {
        if (es[i].dense_len != es[0].dense_len) { set_error("itoe store: dense vectors differ in length"); return CDB_STORAGE_MISMATCH; }
        if (out_internal_ids) out_internal_ids[got] = (uint32_t)es[i].key;
        if (out_vectors) s.copy_dense(es[i], out_vectors + got * es[0].dense_len);
    }
    *out_read = got;
    return CDB_OK;
}

cdb_status cdb_itoe_get(const char *collection_dir, uint32_t internal_id, float *out_vector, uint32_t capacity, uint32_t *out_len) {
    if (!collection_dir || !out_len) { set_error("null argument"); return CDB_INVALID_PARAMS; }
    ItoeStore s;
    Entry e;
    bool hit = false;
    if (!s.open(collection_dir) || !s.lookup(internal_id, e, hit)) return store_error(s);
    *out_len = hit ? e.dense_len : 0;
    if (hit && e.dense_len && out_vector) {
        if (capacity < e.dense_len) { set_error("itoe store: output buffer too small"); return CDB_INVALID_PARAMS; }
        s.copy_dense(e, out_vector);
    }
    return CDB_OK;
}

cdb_status cdb_index_append_itoe(cdb_index *index, const char *collection_dir, uint32_t *out_internal_ids, uint64_t max_ids,
                                 uint64_t *out_appended) {
    if (!index || !collection_dir) { set_error("null argument"); return CDB_INVALID_PARAMS; }
    cdb_index_desc desc;
    cdb_status rc = cdb_index_describe(index, &desc);
    if (rc) return rc;
    ItoeStore s;
    std::vector<Entry> es;
    if (!s.open(collection_dir) || !s.enumerate(es)) return store_error(s);
    const uint64_t CH = std::max<uint64_t>(1, (64ull << 20) / ((uint64_t)desc.dim * 4));
    std::vector<float> buf;
    buf.reserve(std::min<uint64_t>(CH, es.size()) * desc.dim);
    uint64_t done = 0;
    while (done < es.size()) {
        const uint64_t m = std::min<uint64_t>(CH, es.size() - done);
        buf.resize(m * desc.dim);
        for (uint64_t i = 0; i < m; ++i) {
            const Entry &e = es[done + i];
            if (e.dense_len != desc.dim) {
                set_error("itoe store: internal id " + std::to_string(e.key) + " has " + std::to_string(e.dense_len) + " dense values, index dim is " + std::to_string(desc.dim));
                return CDB_STORAGE_MISMATCH;
            }
            s.copy_dense(e, buf.data() + i * desc.dim);
            if (out_internal_ids && done + i < max_ids) out_internal_ids[done + i] = (uint32_t)e.key;
        }
        if ((rc = cdb_index_append_f32(index, buf.data(), m))) return rc;
        done += m;
    }
    if (out_appended) *out_appended = done;
    return CDB_OK;
}

// Cold start, second half: rows appended from prop.data (cdb_index_append_prop_file) carry only the quantized payload; the raw
// f32 embeddings the exact re-rank reads live in the itoe store, keyed by internal id.  row_ids[r] = the id whose embedding
// belongs to row r (what cdb_index_append_prop_file returned; for collections with a metadata schema the caller maps a
// replica id to its base id first, collection.rs:368-384).  CDB_INVALID_ID marks rows that have no embedding by design
// (the root vector, id u32::MAX, vector_store.rs:57-67): they stay zero and count as filled.
cdb_status cdb_index_fill_raw_from_itoe(cdb_index *index, const char *collection_dir, const uint32_t *row_ids, uint64_t n_rows,
                                        uint64_t *out_filled, uint64_t *out_missing) {
    if (!index || !collection_dir || (!row_ids && n_rows)) { set_error("null argument"); return CDB_INVALID_PARAMS; }
    cdb_index_desc desc;
    cdb_status rc = cdb_index_describe(index, &desc);
    if (rc) return rc;
    ItoeStore s;
    if (!s.open(collection_dir)) return store_error(s);
    const uint64_t CH = std::max<uint64_t>(1, (64ull << 20) / ((uint64_t)desc.dim * 4));
    std::vector<float> buf;
    uint64_t filled = 0, missing = 0;
    for (uint64_t r0 = 0; r0 < n_rows; r0 += CH) {
        const uint64_t m = std::min<uint64_t>(CH, n_rows - r0);
        buf.assign(m * desc.dim, 0.0f);
        for (uint64_t i = 0; i < m; ++i) {
            const uint32_t id = row_ids[r0 + i];
            if (id == CDB_INVALID_ID) { ++filled; continue; }
            Entry e;
            bool hit = false;
            if (!s.lookup(id, e, hit)) return store_error(s);
            if (!hit || e.dense_len == 0) { ++missing; continue; }
            if (e.dense_len != desc.dim) {
                set_error("itoe store: internal id " + std::to_string(id) + " has " + std::to_string(e.dense_len) + " dense values, index dim is " + std::to_string(desc.dim));
                return CDB_STORAGE_MISMATCH;
            }
            s.copy_dense(e, buf.data() + i * desc.dim);
            ++filled;
        }
        if ((rc = cdb_index_set_raw_f32(index, r0, buf.data(), m))) return rc;
    }
    if (out_filled) *out_filled = filled;
    if (out_missing) *out_missing = missing;
    if (missing) { set_error(std::to_string(missing) + " rows have no embedding in the itoe store (their raw rows are zero)"); return CDB_INVALID_PARAMS; }
    return CDB_OK;
}

// ---- the sparse pairs (InvertedIndex's rows): live embeddings with sparse values, ascending internal id
static bool sparse_entries(ItoeStore &s, const char *dir, std::vector<Entry> &es) {
    s.sparse = true;
    return s.open(dir) && s.enumerate(es);
}

cdb_status cdb_itoe_scan_sparse(const char *collection_dir, uint64_t *out_entries, uint64_t *out_pairs, uint64_t *out_max_internal_id) {
    if (!collection_dir) { set_error("null path"); return CDB_INVALID_PARAMS; }
    ItoeStore s;
    std::vector<Entry> es;
    if (!sparse_entries(s, collection_dir, es)) return store_error(s);
    uint64_t pairs = 0;
    for (const Entry &e : es) pairs += e.sparse_len;
    if (out_entries) *out_entries = es.size();
    if (out_pairs) *out_pairs = pairs;
    if (out_max_internal_id) *out_max_internal_id = es.empty() ? 0 : es.back().key;
    return CDB_OK;
}

cdb_status cdb_itoe_load_sparse(const char *collection_dir, uint64_t first_entry, uint64_t max_entries, uint64_t max_pairs,
                                uint32_t *out_internal_ids, uint64_t *out_row_offsets, uint32_t *out_dims, float *out_values,
                                uint64_t *out_read) {
    if (!collection_dir || !out_read || !out_row_offsets) { set_error("null argument"); return CDB_INVALID_PARAMS; }
    ItoeStore s;
    std::vector<Entry> es;
    if (!sparse_entries(s, collection_dir, es)) return store_error(s);
    uint64_t got = 0, pairs = 0;
    out_row_offsets[0] = 0;
    for (uint64_t i = first_entry; i < es.size() && got < max_entries; ++i, ++got) {
        if (pairs + es[i].sparse_len > max_pairs) { set_error("itoe store: more sparse pairs than max_pairs"); return CDB_INVALID_PARAMS; }
        if (!out_dims || !out_values) { set_error("null pair buffers"); return CDB_INVALID_PARAMS; }
        if (out_internal_ids) out_internal_ids[got] = (uint32_t)es[i].key;
        s.copy_sparse(es[i], out_dims + pairs, out_values + pairs);
        pairs += es[i].sparse_len;
        out_row_offsets[got + 1] = pairs;
    }
    *out_read = got;
    return CDB_OK;
}

cdb_status cdb_sparse_index_append_itoe(cdb_sparse_index *index, const char *collection_dir, uint32_t *out_internal_ids, uint64_t max_ids,
                                        uint64_t *out_appended) {
    if (!index || !collection_dir) { set_error("null argument"); return CDB_INVALID_PARAMS; }
    ItoeStore s;
    std::vector<Entry> es;
    if (!sparse_entries(s, collection_dir, es)) return store_error(s);
    uint64_t rows0 = 0, rows_left = 0, pairs_left = 0, pairs = 0;
    cdb_status rc = sparse_index_room(index, &rows0, &rows_left, &pairs_left);
    if (rc) return rc;
    for (const Entry &e : es) pairs += e.sparse_len;
    if (es.size() > rows_left || pairs > pairs_left) { set_error("itoe store: the embeddings exceed the index's capacity"); return CDB_INVALID_PARAMS; }
    const uint64_t CH = 16ull << 20;   // pairs per staged append
    std::vector<uint64_t> off;
    std::vector<uint32_t> dims;
    std::vector<float> vals;
    uint64_t done = 0;
    while (done < es.size()) {
        off.assign(1, 0);
        dims.clear();
        vals.clear();
        uint64_t m = 0;
        while (done + m < es.size() && (m == 0 || off.back() + es[done + m].sparse_len <= CH)) {
            const Entry &e = es[done + m];
            dims.resize(off.back() + e.sparse_len);
            vals.resize(off.back() + e.sparse_len);
            s.copy_sparse(e, dims.data() + off.back(), vals.data() + off.back());
            off.push_back(off.back() + e.sparse_len);
            if (out_internal_ids && done + m < max_ids) out_internal_ids[done + m] = (uint32_t)e.key;
            ++m;
        }
        if ((rc = cdb_sparse_index_append(index, off.data(), dims.data(), vals.data(), m))) {
            if (done) {                                   // the earlier chunks go too: all or nothing
                const std::string msg = cdb_last_error_string();
                sparse_index_truncate(index, rows0);
                set_error(msg);
            }
            return rc;
        }
        done += m;
    }
    if (out_appended) *out_appended = done;
    return CDB_OK;
}

}  // extern "C"
