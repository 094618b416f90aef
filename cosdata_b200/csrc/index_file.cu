// index_file.cu -- host-side reader that flattens the reference's on-disk HNSW index into the arrays of cdb_index_set_graph
// (SURVEY 8f-1 "graph export"; no device code here).
//
// Files of one dense index directory (src/models/types.rs:797-860, src/api_service.rs:64):
//   prop.data     Storage / Metadata records of the nodes (prop_file.cu)
//   nodes.ptr     "latest version links": 8 bytes per ProbNode slot = (u32 offset, u32 file id) of the newest serialized version
//                 (serializer/hnsw/latest_node.rs:17-44; flat image of the FilelessBufferManager, buffered_io.rs:497-522, 768-777)
//   <id>.index    node records (serializer/hnsw/node.rs:19-101), little endian:
//                   u8 level | u32 version | u32 prop offset | u32 prop length | u32 metadata offset (u32::MAX = none) | u32 length |
//                   u32 parent link | u32 child link | u16 n | n x (u32 neighbour id, u32 neighbour link, u8 tag, f32 similarity)
//                 every "link" is a byte offset into nodes.ptr (u32::MAX = null); an empty neighbour slot is 13 x 0xFF
//                 (serializer/hnsw/neighbors.rs:21-60); (tag, similarity) is the MetricResult add_neighbor kept for the slot
//                 (types.rs:425-431), kept as read (slot_tag / slot_score) for cdb_index_set_graph_slot_scores: the reader does
//                 not know the index's metric, so tags are not checked here.
// The two entry links (root_vec_ptr_offset / pseudo_root_vec_ptr_offset) live in LMDB next to the index parameters
// (types.rs:899-945) and are passed in by the caller.  With enable_context_history the link image is not one file: every
// flush writes each dirty 8192-byte region in full to "<region>-<version>.ptr" (cache_loader.rs:91-113,
// buffered_io.rs:779-797) and the loader takes, per region, the file of the highest version <= the current one
// (FilelessBufferManager::from_versioned, buffered_io.rs:524-570; file-name rule types.rs:820-842).  Both layouts are read:
// nodes.ptr when it exists, else the region files (cdb_hnsw_files_open_versioned picks the version).
//
// Flattening: breadth first from the entry links over neighbour, child and parent links; level-local indices in discovery order
// (the root is index 0 of every level it exists on).  node_row = ordinal of the node's Storage record in prop.data (the row
// cdb_index_append_prop_file gives it), node_id = replica id when the node has Metadata, else the Storage record's id
// (ProbNode::get_id).  Nodes that no link reaches are unreachable for the reference's search as well and are left out.
#include <dirent.h>

#include <algorithm>
#include <deque>
#include <map>
#include <memory>
#include <unordered_map>

#include "ref_files.h"

struct cdb_hnsw_files {
    uint32_t num_levels = 0, nbrs = 0, nbrs0 = 0, entry = 0, pseudo_entry = CDB_INVALID_ID, root_row = 0, md_dims = 0;
    bool has_md = false;
    std::vector<std::vector<uint32_t>> node_row, node_id, node_md, adj, child;
    std::vector<std::vector<float>> slot_score;     // per level, parallel to adj (empty slot: 0)
    std::vector<std::vector<uint8_t>> slot_tag;     // per level, parallel to adj (empty slot: 0xFF)
    std::vector<int32_t> md_bits;
    std::vector<float> md_mags;
};

namespace cdb {
namespace {
using namespace reffiles;

struct PropIndex {
    std::unordered_map<uint64_t, std::pair<uint32_t, uint32_t>> value;   // record offset -> (row ordinal, id)
    std::unordered_map<uint64_t, std::pair<uint32_t, uint32_t>> md;      // record offset -> (metadata table row, replica id)
    std::vector<int32_t> md_bits;
    std::vector<float> md_mags;
    uint32_t md_dims = 0;
};

cdb_status load_prop_index(const std::string &path, PropIndex &pi) {
    Mapped f;
    cdb_status rc = f.open(path.c_str());
    if (rc) return rc;
    Cur c{f.p, f.p + f.len};
    Record r;
    uint32_t rows = 0, mdrows = 0;
    while (c.p < c.end) {
        const uint64_t off = (uint64_t)(c.p - f.p);
        if (!parse_record(c, r)) { set_error("prop.data at byte " + std::to_string(off) + ": " + c.why); return CDB_INVALID_PARAMS; }
        if (r.is_metadata) {
            if (mdrows == 0) pi.md_dims = (uint32_t)r.mbits.size();
            else if (r.mbits.size() != pi.md_dims) { set_error("prop.data: Metadata records differ in length"); return CDB_STORAGE_MISMATCH; }
            pi.md[off] = {mdrows++, r.id};
            pi.md_bits.insert(pi.md_bits.end(), r.mbits.begin(), r.mbits.end());
            pi.md_mags.push_back(r.mag);
        } else pi.value[off] = {rows++, r.id};
    }
    return CDB_OK;
}

struct NodeRec {
    uint8_t level;
    uint32_t prop_off, md_off, parent, child;
    std::vector<uint32_t> nbr_link;   // CDB_INVALID_ID = empty slot
    std::vector<uint8_t> tag;         // MetricResult of each slot as stored
    std::vector<float> score;
};

struct Reader {
    std::string dir, err;
    struct { const uint8_t *p = nullptr; size_t len = 0; } links;
    Mapped links_file;                 // nodes.ptr, or
    std::vector<uint8_t> links_image;  // the image assembled from "<region>-<version>.ptr" files
    // "latest version links" of the index directory; latest_version bounds the versioned layout
    cdb_status open_links(uint32_t latest_version) {
        struct stat sb;
        const std::string flat = dir + "/nodes.ptr";
        if (::stat(flat.c_str(), &sb) == 0) {
            cdb_status rc = links_file.open(flat.c_str());
            if (rc) return rc;
            links.p = links_file.p; links.len = links_file.len;
            return CDB_OK;
        }
        const size_t REGION = 8192;    // buffer size of latest_version_links_bufman (types.rs:819-821)
        std::map<uint64_t, std::pair<uint32_t, std::string>> best;   // region -> (version, file)
        DIR *d = opendir(dir.c_str());
        if (!d) { set_error("cannot open index directory " + dir); return CDB_INVALID_PARAMS; }
        while (struct dirent *e = readdir(d)) {
            // "<region>-<version>.ptr": exactly one '.', exactly one '-', both parts decimal (types.rs:823-842)
            const std::string name = e->d_name;
            const size_t dot = name.find('.'), dash = name.find('-');
            if (dot == std::string::npos || name.find('.', dot + 1) != std::string::npos || name.substr(dot) != ".ptr") continue;
            if (dash == std::string::npos || dash == 0 || dash + 1 >= dot || name.find('-', dash + 1) != std::string::npos) continue;
            const std::string rs = name.substr(0, dash), vs = name.substr(dash + 1, dot - dash - 1);
            if (rs.find_first_not_of("0123456789") != std::string::npos || vs.find_first_not_of("0123456789") != std::string::npos) continue;
            if (rs.size() > 18 || vs.size() > 10) continue;
            const uint64_t region = std::stoull(rs), ver64 = std::stoull(vs);
            if (ver64 > 0xFFFFFFFFull || ver64 > latest_version) continue;
            auto it = best.find(region);
            if (it != best.end() && it->second.first > (uint32_t)ver64) continue;
            best[region] = {(uint32_t)ver64, dir + "/" + name};
        }
        closedir(d);
        if (best.empty()) { set_error("no nodes.ptr and no <region>-<version>.ptr files in " + dir); return CDB_INVALID_PARAMS; }
        for (auto &kv : best) {
            Mapped f;
            cdb_status rc = f.open(kv.second.second.c_str());
            if (rc) return rc;
            const size_t n = std::min(f.len, REGION), off = (size_t)kv.first * REGION;
            if (links_image.size() < off + n) links_image.resize(off + n, 0xFF);   // holes = null links
            if (n) memcpy(links_image.data() + off, f.p, n);
        }
        links.p = links_image.data(); links.len = links_image.size();
        return CDB_OK;
    }
    std::map<uint32_t, std::unique_ptr<Mapped>> files;

    bool fail(const std::string &m) { if (err.empty()) err = m; return false; }
    const Mapped *file(uint32_t id) {
        auto it = files.find(id);
        if (it != files.end()) return it->second.get();
        std::unique_ptr<Mapped> f(new Mapped());
        if (f->open((dir + "/" + std::to_string(id) + ".index").c_str())) { fail("cannot open " + std::to_string(id) + ".index"); return nullptr; }
        return (files[id] = std::move(f)).get();
    }
    static uint32_t u32(const uint8_t *p) { uint32_t v; memcpy(&v, p, 4); return v; }
    bool read(uint32_t link, NodeRec &n) {
        if ((uint64_t)link + 8 > links.len) return fail("link " + std::to_string(link) + " outside nodes.ptr");
        const uint32_t off = u32(links.p + link), fid = u32(links.p + link + 4);
        const Mapped *f = file(fid);
        if (!f) return false;
        if ((uint64_t)off + 31 > f->len) return fail("node record outside " + std::to_string(fid) + ".index");
        const uint8_t *p = f->p + off;
        n.level = p[0];
        n.prop_off = u32(p + 5); n.md_off = u32(p + 13); n.parent = u32(p + 21); n.child = u32(p + 25);
        uint16_t cnt; memcpy(&cnt, p + 29, 2);
        if ((uint64_t)off + 31 + (uint64_t)cnt * 13 > f->len) return fail("neighbour list outside " + std::to_string(fid) + ".index");
        n.nbr_link.resize(cnt); n.tag.resize(cnt); n.score.resize(cnt);
        for (uint32_t s = 0; s < cnt; ++s) {
            const uint8_t *e = p + 31 + s * 13;
            n.nbr_link[s] = u32(e + 4);   // 0xFFFFFFFF for an empty slot
            n.tag[s] = e[8];
            memcpy(&n.score[s], e + 9, 4);
        }
        return true;
    }
};

cdb_status flatten(const char *index_dir, uint32_t root_link, uint32_t pseudo_link, uint32_t latest_version, cdb_hnsw_files &out) {
    PropIndex pi;
    cdb_status rc = load_prop_index(std::string(index_dir) + "/prop.data", pi);
    if (rc) return rc;
    Reader rd;
    rd.dir = index_dir;
    if ((rc = rd.open_links(latest_version))) return rc;
    auto bad = [&](const std::string &m) { set_error("hnsw index files: " + (rd.err.empty() ? m : rd.err)); return CDB_INVALID_PARAMS; };

    std::unordered_map<uint32_t, std::pair<uint32_t, uint32_t>> where;   // link -> (level, local index)
    std::vector<std::vector<uint32_t>> order;                            // per level: links in discovery order
    std::vector<std::vector<NodeRec>> recs;
    std::deque<uint32_t> queue;
    auto visit = [&](uint32_t link, int want_level) -> bool {
        if (link == CDB_INVALID_ID || where.count(link)) return true;
        NodeRec n;
        if (!rd.read(link, n)) return false;
        if (want_level >= 0 && n.level != want_level) return rd.fail("a link crosses levels (node level " + std::to_string(n.level) + ", expected " + std::to_string(want_level) + ")");
        if (n.level > 31) return rd.fail("level out of range");
        if (order.size() <= n.level) { order.resize(n.level + 1); recs.resize(n.level + 1); }
        where[link] = {n.level, (uint32_t)order[n.level].size()};
        order[n.level].push_back(link);
        recs[n.level].push_back(std::move(n));
        queue.push_back(link);
        return true;
    };
    if (!visit(root_link, -1)) return bad("");
    if (pseudo_link != CDB_INVALID_ID && !visit(pseudo_link, -1)) return bad("");
    while (!queue.empty()) {
        const uint32_t link = queue.front();
        queue.pop_front();
        const auto w = where[link];
        const NodeRec n = recs[w.first][w.second];   // copy: recs may grow while visiting
        for (uint32_t nl : n.nbr_link) if (!visit(nl, n.level)) return bad("");
        if (n.level > 0 && !visit(n.child, n.level - 1)) return bad("");
        if (!visit(n.parent, n.level + 1)) return bad("");
    }
    const uint32_t L1 = (uint32_t)order.size();
    const auto rw = where[root_link];
    if (rw.first + 1 != L1) return bad("the root link is not on the top level");
    if (pseudo_link != CDB_INVALID_ID && where[pseudo_link].first + 1 != L1) return bad("the pseudo root link is not on the top level");
    out.num_levels = L1 - 1;
    out.entry = rw.second;
    out.pseudo_entry = pseudo_link == CDB_INVALID_ID ? CDB_INVALID_ID : where[pseudo_link].second;
    out.node_row.assign(L1, {}); out.node_id.assign(L1, {}); out.node_md.assign(L1, {}); out.adj.assign(L1, {}); out.child.assign(L1, {});
    out.slot_score.assign(L1, {}); out.slot_tag.assign(L1, {});
    out.nbrs = out.nbrs0 = 0;
    for (uint32_t L = 0; L < L1; ++L) {
        const uint32_t cnt = (uint32_t)order[L].size();
        if (cnt == 0) return bad("level " + std::to_string(L) + " has no reachable node");
        const uint32_t nb = (uint32_t)recs[L][0].nbr_link.size();
        if (nb < 1 || nb > 64) return bad("neighbour count must be in 1..64");
        if (L == 0) out.nbrs0 = nb;
        else if (out.nbrs == 0) out.nbrs = nb;
        else if (out.nbrs != nb) return bad("levels >= 1 differ in neighbour count");
        out.node_row[L].resize(cnt); out.node_id[L].resize(cnt); out.node_md[L].resize(cnt); out.child[L].assign(cnt, 0);
        out.adj[L].assign((size_t)cnt * nb, CDB_INVALID_ID);
        out.slot_score[L].assign((size_t)cnt * nb, 0.0f);
        out.slot_tag[L].assign((size_t)cnt * nb, 0xFF);
        for (uint32_t i = 0; i < cnt; ++i) {
            const NodeRec &n = recs[L][i];
            if (n.nbr_link.size() != nb) return bad("nodes of one level differ in neighbour count");
            const auto pv = pi.value.find(n.prop_off);
            if (pv == pi.value.end()) return bad("node refers to no Storage record of prop.data (offset " + std::to_string(n.prop_off) + ")");
            out.node_row[L][i] = pv->second.first;
            out.node_id[L][i] = pv->second.second;
            out.node_md[L][i] = CDB_INVALID_ID;
            if (n.md_off != CDB_INVALID_ID) {
                const auto pm = pi.md.find(n.md_off);
                if (pm == pi.md.end()) return bad("node refers to no Metadata record of prop.data (offset " + std::to_string(n.md_off) + ")");
                out.node_md[L][i] = pm->second.first;
                out.node_id[L][i] = pm->second.second;   // ProbNode::get_id(): the replica id
                out.has_md = true;
            }
            for (uint32_t s = 0; s < nb; ++s) {
                if (n.nbr_link[s] == CDB_INVALID_ID) continue;
                out.adj[L][(size_t)i * nb + s] = where[n.nbr_link[s]].second;
                out.slot_score[L][(size_t)i * nb + s] = n.score[s];
                out.slot_tag[L][(size_t)i * nb + s] = n.tag[s];
            }
            if (L > 0) {
                if (n.child == CDB_INVALID_ID) return bad("a node above level 0 has no child");
                out.child[L][i] = where[n.child].second;
            }
        }
    }
    if (out.nbrs == 0) out.nbrs = out.nbrs0;   // a graph with level 0 only
    out.root_row = out.node_row[L1 - 1][out.entry];
    out.md_dims = pi.md_dims;
    out.md_bits = std::move(pi.md_bits);
    out.md_mags = std::move(pi.md_mags);
    return CDB_OK;
}

}  // namespace
}  // namespace cdb

using namespace cdb;

extern "C" {

cdb_status cdb_hnsw_files_open_versioned(const char *index_dir, uint32_t root_link_offset, uint32_t pseudo_root_link_offset,
                                         uint32_t latest_version, cdb_hnsw_files **out) {
    if (!index_dir || !out) { set_error("null argument"); return CDB_INVALID_PARAMS; }
    std::unique_ptr<cdb_hnsw_files> h(new cdb_hnsw_files());
    const cdb_status rc = flatten(index_dir, root_link_offset, pseudo_root_link_offset, latest_version, *h);
    if (rc) return rc;
    *out = h.release();
    return CDB_OK;
}
cdb_status cdb_hnsw_files_open(const char *index_dir, uint32_t root_link_offset, uint32_t pseudo_root_link_offset, cdb_hnsw_files **out) {
    return cdb_hnsw_files_open_versioned(index_dir, root_link_offset, pseudo_root_link_offset, 0xFFFFFFFFu, out);
}

cdb_status cdb_hnsw_files_close(cdb_hnsw_files *h) {
    delete h;
    return CDB_OK;
}

cdb_status cdb_hnsw_files_info(const cdb_hnsw_files *h, uint32_t *info8, uint32_t *level_counts) {
    if (!h || !info8) { set_error("null argument"); return CDB_INVALID_PARAMS; }
    const uint32_t v[8] = {h->num_levels, h->nbrs, h->nbrs0, h->entry, h->pseudo_entry, h->root_row, h->md_dims, (uint32_t)h->md_mags.size()};
    memcpy(info8, v, sizeof(v));
    if (level_counts) for (uint32_t L = 0; L <= h->num_levels; ++L) level_counts[L] = (uint32_t)h->node_row[L].size();
    return CDB_OK;
}

cdb_status cdb_hnsw_files_level(const cdb_hnsw_files *h, uint32_t level, uint32_t *node_row, uint32_t *node_id, uint32_t *node_md,
                                uint32_t *adjacency, uint32_t *child) {
    if (!h || level > h->num_levels) { set_error("bad argument"); return CDB_INVALID_PARAMS; }
    const size_t cnt = h->node_row[level].size();
    if (node_row) memcpy(node_row, h->node_row[level].data(), cnt * 4);
    if (node_id) memcpy(node_id, h->node_id[level].data(), cnt * 4);
    if (node_md) memcpy(node_md, h->node_md[level].data(), cnt * 4);
    if (adjacency) memcpy(adjacency, h->adj[level].data(), h->adj[level].size() * 4);
    if (child) memcpy(child, h->child[level].data(), cnt * 4);
    return CDB_OK;
}

cdb_status cdb_hnsw_files_slot_scores(const cdb_hnsw_files *h, uint32_t level, float *out_scores, uint8_t *out_tags) {
    if (!h || level > h->num_levels) { set_error("bad argument"); return CDB_INVALID_PARAMS; }
    const size_t slots = h->adj[level].size();
    if (out_scores) memcpy(out_scores, h->slot_score[level].data(), slots * 4);
    if (out_tags) memcpy(out_tags, h->slot_tag[level].data(), slots);
    return CDB_OK;
}

cdb_status cdb_hnsw_files_metadata(const cdb_hnsw_files *h, int32_t *md_bits, float *md_mags) {
    if (!h) { set_error("null argument"); return CDB_INVALID_PARAMS; }
    if (md_bits) memcpy(md_bits, h->md_bits.data(), h->md_bits.size() * 4);
    if (md_mags) memcpy(md_mags, h->md_mags.data(), h->md_mags.size() * 4);
    return CDB_OK;
}

cdb_status cdb_index_set_graph_from_files(cdb_index *index, const cdb_hnsw_files *h) {
    if (!index || !h) { set_error("null argument"); return CDB_INVALID_PARAMS; }
    const uint32_t L1 = h->num_levels + 1;
    std::vector<uint32_t> counts(L1);
    std::vector<const uint32_t *> nr(L1), ad(L1), ch(L1), ni(L1), nm(L1);
    for (uint32_t L = 0; L < L1; ++L) {
        counts[L] = (uint32_t)h->node_row[L].size();
        nr[L] = h->node_row[L].data(); ad[L] = h->adj[L].data(); ch[L] = h->child[L].data();
        ni[L] = h->node_id[L].data(); nm[L] = h->node_md[L].data();
    }
    cdb_graph_desc gd{};
    gd.num_levels = h->num_levels;
    gd.neighbors_count = h->nbrs;
    gd.level0_neighbors_count = h->nbrs0;
    gd.entry = h->entry;
    gd.root_row = h->root_row;
    gd.level_counts = counts.data();
    gd.node_row = nr.data();
    gd.adjacency = ad.data();
    gd.child = ch.data();
    cdb_status rc = cdb_index_set_graph(index, &gd);
    if (rc) return rc;
    // node ids are always attached: the lossy fixed set of the traversal is keyed by the reference's InternalIds (not by row
    // ordinals), and results are reported under those ids like InternalSearchResult; the metadata table may be empty
    cdb_graph_metadata md{};
    md.md_dims = h->md_dims ? h->md_dims : 1u;
    md.n_md = (uint32_t)h->md_mags.size();
    md.md_bits = h->md_bits.data();
    md.md_mags = h->md_mags.data();
    md.node_id = ni.data();
    md.node_md = nm.data();
    md.pseudo_entry = h->pseudo_entry == CDB_INVALID_ID ? h->entry : h->pseudo_entry;
    return cdb_index_set_graph_metadata(index, &md);
}

}  // extern "C"
