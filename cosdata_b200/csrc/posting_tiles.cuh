// posting_tiles.cuh -- the row store and posting-list tiles the sparse (sparse.cu) and TF-IDF (tfidf.cu) indexes share
// (DESIGN.md section 8c, "Posting tiles").  Rows are kept as raw CSR on the device (a u32 key and an f32 value per pair, u64
// row offsets, and a host mirror of the offsets).  Posting lists are split into row tiles of 2^TILE_SHIFT rows; a tile holds
// its distinct keys (ascending), a segment start per key and one entry per pair of its rows, re-ordered by a CUB radix sort.
// An append rebuilds the last partial tile and builds the new ones, all or nothing.  Deleted rows are a tombstone bitmap.
//
// What an index puts into its entries is its codec C:
//   using Entry;                                       the posting entry
//   static constexpr int END_BIT, SEG_SHIFT;           sort keys are END_BIT bits wide; sort_key >> SEG_SHIFT is the pair's key
//   static constexpr const char *DUPLICATE_ERROR;      the error of two equal sort keys in a tile, or nullptr if they are allowed
//   __device__ SortPair encode(uint32_t key, float value, uint32_t row_in_tile) const;
//   __device__ Entry entry(uint64_t sort_key, uint32_t sort_val) const;
#pragma once
#include <algorithm>
#include <string>
#include <vector>

#include "common.cuh"

namespace cdb {

constexpr uint32_t TILE_SHIFT = 15;
constexpr uint32_t TILE_ROWS = 1u << TILE_SHIFT;

struct PostingTile {
    uint64_t entry_base;   // first entry of the tile
    uint64_t key_base;     // first distinct key in d_tkeys; its segment starts are d_tseg[key_base + tile ..]
    uint32_t n_keys;
    uint32_t pad;
};

struct SortPair {
    uint64_t key;
    uint32_t val;
};

// first i in [0, n) with a[i] >= x, else n
__device__ inline uint32_t lower_bound_u32(const uint32_t *a, uint32_t n, uint32_t x) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (a[mid] < x) lo = mid + 1; else hi = mid; }
    return lo;
}

// sort keys and values of the pairs of rows [r0, r0 + nr) (pairs from p0 on), one warp per row
template <class C>
__global__ void tile_keys_kernel(C codec, const uint64_t *__restrict__ row_off, uint64_t r0, uint32_t nr, uint64_t p0,
                                 const uint32_t *__restrict__ keys, const float *__restrict__ vals, uint64_t *__restrict__ sort_keys,
                                 uint32_t *__restrict__ sort_vals) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= nr) return;
    const uint64_t b = row_off[r0 + warp], e = row_off[r0 + warp + 1];
    for (uint64_t p = b + lane; p < e; p += 32) {
        const SortPair sp = codec.encode(keys[p], vals[p], warp);
        sort_keys[p - p0] = sp.key;
        sort_vals[p - p0] = sp.val;
    }
}

// entries from the sorted pairs, a flag on the first pair of every segment, and *dup = 1 on equal sort keys (dup may be null)
template <class C>
__global__ void tile_entries_kernel(C codec, const uint64_t *__restrict__ keys, const uint32_t *__restrict__ vals, uint32_t n,
                                    typename C::Entry *__restrict__ entries, uint32_t *__restrict__ flags, uint32_t *__restrict__ dup) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t k = keys[i];
    entries[i] = codec.entry(k, vals[i]);
    flags[i] = (i == 0 || (k >> C::SEG_SHIFT) != (keys[i - 1] >> C::SEG_SHIFT)) ? 1u : 0u;
    if (dup && i > 0 && k == keys[i - 1]) *dup = 1u;
}

// CUB temp storage and sort buffers of one append, sized for its largest tile or more
struct BuildBufs {
    void *tmp = nullptr;
    size_t tmp_bytes = 0;
    uint64_t *keys_in = nullptr, *keys_out = nullptr;
    uint32_t *vals_in = nullptr, *vals_out = nullptr, *flags = nullptr, *pos = nullptr, *dup = nullptr;
    cdb_status alloc(uint64_t n, int end_bit, cudaStream_t s);
    ~BuildBufs();
};

// an append between PostingStore::prepare_append and PostingTiles::commit_append
struct Append {
    uint64_t r_old = 0, p_old = 0, r_new = 0, np = 0, t0 = 0, t1 = 0;   // rows and pairs before, rows after, pairs added, tiles to build
    std::vector<uint64_t> off;                                          // end offsets of the new rows
    StreamGuard sg;
    BuildBufs b;
};

// the codec-independent part of the store
struct PostingStore {
    int device = 0;
    uint64_t capacity_rows = 0, capacity_pairs = 0;
    uint64_t n_rows = 0, n_pairs = 0, n_deleted = 0;
    std::vector<uint64_t> h_row_off{0};
    std::vector<PostingTile> h_tiles;
    std::vector<uint32_t> h_deleted;
    uint64_t *d_row_off = nullptr;
    uint32_t *d_keys = nullptr, *d_tkeys = nullptr, *d_tseg = nullptr, *d_deleted = nullptr;
    float *d_vals = nullptr;
    void *d_entries = nullptr;
    PostingTile *d_tiles = nullptr;

    PostingStore() = default;
    PostingStore(const PostingStore &) = delete;
    PostingStore &operator=(const PostingStore &) = delete;
    ~PostingStore();

    // capacity checks, then every device allocation (on `device`, made current)
    cdb_status init(int device, uint32_t id_base, uint64_t capacity_rows, uint64_t capacity_pairs, size_t entry_bytes);
    // the bitmap a search passes to its kernels: null while nothing is deleted
    const uint32_t *deleted() const { return n_deleted ? d_deleted : nullptr; }
    // Step one of an append of n rows (row_offsets checked with check_csr): every remaining check and allocation, scratch
    // for at least min_scratch pairs, a drain of the searches already queued (they read the tile the append rebuilds), then
    // the pairs and offsets copied in past the index's end, where nothing reads them yet.  `what` prefixes a copy error.
    cdb_status prepare_append(const uint64_t *row_offsets, const uint32_t *keys, const float *vals, uint64_t n, int end_bit,
                              uint64_t min_scratch, const char *what, Append &a);
    cdb_status deleted_rows(uint64_t first, uint64_t n, uint8_t *out, uint64_t *out_total) const;

    // Tombstones rows[0..n), each below n_rows.  apply(fresh), fresh the rows not deleted before, runs once queued searches
    // have drained and the new bitmap is on the device, before it becomes the index's; if apply fails the old bitmap goes back.
    template <class Fn>
    cdb_status mark_deleted(const uint32_t *rows, uint64_t n, Fn apply) {
        for (uint64_t i = 0; i < n; ++i) CDB_REQUIRE(rows[i] < n_rows, "row out of range");
        CDB_CUDA_TRY(cudaSetDevice(device));
        if (!n) return CDB_OK;
        std::vector<uint32_t> w = h_deleted, fresh;
        for (uint64_t i = 0; i < n; ++i) {
            uint32_t &x = w[rows[i] >> 5];
            const uint32_t bit = 1u << (rows[i] & 31);
            if (!(x & bit)) { x |= bit; fresh.push_back(rows[i]); }
        }
        // searches enqueued before this call finish first (they read the bitmap)
        CDB_CUDA_TRY(cudaDeviceSynchronize());
        CDB_CUDA_TRY(cudaMemcpy(d_deleted, w.data(), w.size() * 4, cudaMemcpyHostToDevice));
        const cdb_status rc = apply(fresh);
        if (rc) {
            cudaMemcpy(d_deleted, h_deleted.data(), w.size() * 4, cudaMemcpyHostToDevice);
            return rc;
        }
        h_deleted.swap(w);
        n_deleted += fresh.size();
        return CDB_OK;
    }

  protected:
    // tile t's record, its pair count and its first row
    PostingTile tile_at(uint64_t t, uint32_t *np, uint32_t *nr) const;
    cudaError_t sort_tile(BuildBufs &b, uint32_t np, int end_bit, cudaStream_t s) const;
    // tile t (sorted into b, its entries written, or np = 0) finished: segments, n_keys, the duplicate check, h_tiles
    cdb_status finish_tile(uint64_t t, PostingTile tile, uint32_t np, int seg_shift, const char *dup_error, BuildBufs &b, cudaStream_t s);
    cdb_status upload_tiles(uint64_t t0, uint64_t t1, cudaStream_t s);
    // the host state and the bitmap back to the first `rows` rows (tombstones of the dropped rows cleared)
    cdb_status drop_rows(uint64_t rows, cudaStream_t s);
};

template <class C>
struct PostingTiles : PostingStore {
    C codec;

    typename C::Entry *entries() const { return static_cast<typename C::Entry *>(d_entries); }
    cdb_status init(int device, uint32_t id_base, uint64_t capacity_rows, uint64_t capacity_pairs) {
        return PostingStore::init(device, id_base, capacity_rows, capacity_pairs, sizeof(typename C::Entry));
    }
    cdb_status prepare_append(const uint64_t *row_offsets, const uint32_t *keys, const float *vals, uint64_t n, uint64_t min_scratch,
                              const char *what, Append &a) {
        return PostingStore::prepare_append(row_offsets, keys, vals, n, C::END_BIT, min_scratch, what, a);
    }

    // tiles [t0, t1) of the current rows, host and device tables; CDB_INVALID_PARAMS on a duplicate the codec refuses
    cdb_status build_tiles(uint64_t t0, uint64_t t1, BuildBufs &b, cudaStream_t s) {
        h_tiles.resize(t0);
        cdb_status rc;
        for (uint64_t t = t0; t < t1; ++t) {
            uint32_t np, nr;
            const PostingTile tile = tile_at(t, &np, &nr);
            uint32_t *dup = C::DUPLICATE_ERROR ? b.dup : nullptr;
            if (np) {
                tile_keys_kernel<C><<<(nr * 32 + 255) / 256, 256, 0, s>>>(codec, d_row_off, t << TILE_SHIFT, nr, tile.entry_base, d_keys,
                                                                       d_vals, b.keys_in, b.vals_in);
                CDB_LAUNCH_CHECK();
                CDB_CUDA_TRY(sort_tile(b, np, C::END_BIT, s));
                if (dup) CDB_CUDA_TRY(cudaMemsetAsync(dup, 0, 4, s));
                tile_entries_kernel<C><<<(np + 255) / 256, 256, 0, s>>>(codec, b.keys_out, b.vals_out, np, entries() + tile.entry_base,
                                                                        b.flags, dup);
                CDB_LAUNCH_CHECK();
            }
            if ((rc = finish_tile(t, tile, np, C::SEG_SHIFT, C::DUPLICATE_ERROR, b, s))) return rc;
        }
        return upload_tiles(t0, t1, s);
    }

    // back to the first `rows` rows (rows <= n_rows): their pairs are still in place, the tile holding row `rows` is rebuilt
    // and tombstones of the dropped rows are cleared.  b must fit that tile.  Device work is ordered by the caller.
    cdb_status restore_rows(uint64_t rows, BuildBufs &b, cudaStream_t s) {
        cdb_status rc = drop_rows(rows, s);
        if (rc) return rc;
        return build_tiles(rows >> TILE_SHIFT, (rows + TILE_ROWS - 1) >> TILE_SHIFT, b, s);
    }

    // Step two of an append: the new rows become the index's, the last partial tile is rebuilt and the new ones built, then
    // finish() runs.  If either fails, the index goes back to its rows before the append and the first error stays.
    template <class Fn>
    cdb_status commit_append(Append &a, Fn finish) {
        h_row_off.insert(h_row_off.end(), a.off.begin(), a.off.end());
        n_rows = a.r_new;
        n_pairs += a.np;
        cdb_status rc = build_tiles(a.t0, a.t1, a.b, a.sg.s);
        if (!rc) rc = finish();
        if (rc) {
            const std::string msg = cdb_last_error_string();
            restore_rows(a.r_old, a.b, a.sg.s);
            set_error(msg);
        }
        return rc;
    }

    // A load into an empty store: rows [0, row_off.size() - 1) whose pairs the caller has written to d_keys / d_vals and whose
    // offsets (row_off, host) it has written to d_row_off.  The rows become the store's and every tile is built; if that
    // fails the store is empty again and the error stays.  b must fit the largest tile.
    cdb_status load_rows(std::vector<uint64_t> row_off, BuildBufs &b, cudaStream_t s) {
        h_row_off = std::move(row_off);
        n_rows = h_row_off.size() - 1;
        n_pairs = h_row_off.back();
        const cdb_status rc = build_tiles(0, (n_rows + TILE_ROWS - 1) >> TILE_SHIFT, b, s);
        if (rc) {
            const std::string msg = cdb_last_error_string();
            restore_rows(0, b, s);
            set_error(msg);
        }
        return rc;
    }
};

// the most pairs one row tile of the CSR offsets row_off holds
inline uint64_t max_tile_pairs(const std::vector<uint64_t> &row_off) {
    const uint64_t n = row_off.size() - 1;
    uint64_t m = 0;
    for (uint64_t r0 = 0; r0 < n; r0 += TILE_ROWS) m = std::max(m, row_off[std::min(n, r0 + TILE_ROWS)] - row_off[r0]);
    return m;
}

// the result of a search of an index without tiles: ids CDB_INVALID_ID, scores 0, counts 0
cdb_status fill_empty_results(uint32_t nq, uint32_t k, uint32_t *d_ids, float *d_scores, uint32_t *d_counts, cudaStream_t s);

}  // namespace cdb
