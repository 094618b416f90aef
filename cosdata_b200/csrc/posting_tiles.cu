// posting_tiles.cu -- the codec-independent half of the posting-tile store (posting_tiles.cuh): allocation, the sort, scan and
// segment scatter of a tile build, the append's checks and row copy, and the tombstone bitmap.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "posting_tiles.cuh"

namespace cdb {
namespace {

// distinct keys and segment starts of a tile's sorted pairs: pos = inclusive scan of the segment flags
__global__ void seg_scatter_kernel(const uint64_t *__restrict__ keys, const uint32_t *__restrict__ flags, const uint32_t *__restrict__ pos,
                                   uint32_t n, int seg_shift, uint32_t *__restrict__ tkeys, uint32_t *__restrict__ tseg) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (flags[i]) {
        tkeys[pos[i] - 1] = (uint32_t)(keys[i] >> seg_shift);
        tseg[pos[i] - 1] = i;
    }
    if (i == n - 1) tseg[pos[i]] = n;
}

}  // namespace

cdb_status BuildBufs::alloc(uint64_t n, int end_bit, cudaStream_t s) {
    if (!n) return CDB_OK;
    CDB_CUDA_TRY(cudaMalloc(&keys_in, n * 8));
    CDB_CUDA_TRY(cudaMalloc(&keys_out, n * 8));
    CDB_CUDA_TRY(cudaMalloc(&vals_in, n * 4));
    CDB_CUDA_TRY(cudaMalloc(&vals_out, n * 4));
    CDB_CUDA_TRY(cudaMalloc(&flags, n * 4));
    CDB_CUDA_TRY(cudaMalloc(&pos, n * 4));
    CDB_CUDA_TRY(cudaMalloc(&dup, 4));
    size_t t_sort = 0, t_scan = 0;
    CDB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, t_sort, keys_in, keys_out, vals_in, vals_out, (int)n, 0, end_bit, s));
    CDB_CUDA_TRY(cub::DeviceScan::InclusiveSum(nullptr, t_scan, flags, pos, (int)n, s));
    tmp_bytes = std::max(t_sort, t_scan);
    CDB_CUDA_TRY(cudaMalloc(&tmp, tmp_bytes));
    return CDB_OK;
}

BuildBufs::~BuildBufs() {
    for (void *p : {tmp, (void *)keys_in, (void *)keys_out, (void *)vals_in, (void *)vals_out, (void *)flags, (void *)pos, (void *)dup})
        if (p) cudaFree(p);
}

PostingStore::~PostingStore() {
    for (void *p : {(void *)d_row_off, (void *)d_keys, (void *)d_vals, d_entries, (void *)d_tkeys, (void *)d_tseg, (void *)d_deleted,
                    (void *)d_tiles})
        if (p) cudaFree(p);
}

cdb_status PostingStore::init(int dev, uint32_t id_base, uint64_t cap_rows, uint64_t cap_pairs, size_t entry_bytes) {
    CDB_REQUIRE(cap_rows >= 1 && (uint64_t)id_base + cap_rows <= 0xFFFFFFFFull,
                "capacity_rows must be >= 1 and id_base + capacity_rows <= 2^32 - 1");
    CDB_REQUIRE(cap_pairs < (1ull << 40), "capacity_pairs too large");
    CDB_CUDA_TRY(cudaSetDevice(dev));
    device = dev;
    capacity_rows = cap_rows;
    capacity_pairs = cap_pairs;
    const uint64_t max_tiles = (cap_rows + TILE_ROWS - 1) / TILE_ROWS;
    const size_t pairs = std::max<uint64_t>(1, cap_pairs);
    const size_t words = (cap_rows + 31) / 32;
    CDB_CUDA_TRY(cudaMalloc(&d_row_off, (cap_rows + 1) * 8));
    CDB_CUDA_TRY(cudaMalloc(&d_keys, pairs * 4));
    CDB_CUDA_TRY(cudaMalloc(&d_vals, pairs * 4));
    CDB_CUDA_TRY(cudaMalloc(&d_entries, pairs * entry_bytes));
    CDB_CUDA_TRY(cudaMalloc(&d_tkeys, pairs * 4));
    CDB_CUDA_TRY(cudaMalloc(&d_tseg, (pairs + max_tiles) * 4));   // a tile's segment starts end with one more
    CDB_CUDA_TRY(cudaMalloc(&d_deleted, words * 4));
    CDB_CUDA_TRY(cudaMalloc(&d_tiles, max_tiles * sizeof(PostingTile)));
    CDB_CUDA_TRY(cudaMemset(d_row_off, 0, 8));
    CDB_CUDA_TRY(cudaMemset(d_deleted, 0, words * 4));
    h_deleted.assign(words, 0u);
    return CDB_OK;
}

cdb_status PostingStore::prepare_append(const uint64_t *row_offsets, const uint32_t *keys, const float *vals, uint64_t n, int end_bit,
                                        uint64_t min_scratch, const char *what, Append &a) {
    const uint64_t np = row_offsets[n];
    CDB_REQUIRE(n_rows + n <= capacity_rows, "append exceeds capacity_rows");
    CDB_REQUIRE(n_pairs + np <= capacity_pairs, "append exceeds capacity_pairs");
    CDB_CUDA_TRY(cudaSetDevice(device));
    a.r_old = n_rows;
    a.p_old = n_pairs;
    a.r_new = n_rows + n;
    a.np = np;
    a.off.resize(n);
    for (uint64_t i = 0; i < n; ++i) a.off[i] = a.p_old + row_offsets[i + 1];
    auto row_off = [&](uint64_t r) { return r <= a.r_old ? h_row_off[r] : a.off[r - a.r_old - 1]; };
    a.t0 = a.r_old >> TILE_SHIFT;
    a.t1 = (a.r_new + TILE_ROWS - 1) >> TILE_SHIFT;
    uint64_t max_np = 0;
    for (uint64_t t = a.t0; t < a.t1; ++t)
        max_np = std::max(max_np, row_off(std::min<uint64_t>(a.r_new, (t + 1) << TILE_SHIFT)) - row_off(t << TILE_SHIFT));
    CDB_REQUIRE(max_np < (1ull << 31), "a row tile holds 2^31 pairs or more");
    CDB_CUDA_TRY(cudaStreamCreateWithFlags(&a.sg.s, cudaStreamNonBlocking));
    const cudaStream_t s = a.sg.s;
    cdb_status rc = a.b.alloc(std::max(max_np, min_scratch), end_bit, s);
    if (rc) return rc;
    // searches already enqueued on other streams (the *_search_batch_device forms) read the tile this append rebuilds
    CDB_CUDA_TRY(cudaDeviceSynchronize());
    cudaError_t e = cudaSuccess;
    if (np) {
        e = cudaMemcpyAsync(d_keys + a.p_old, keys, np * 4, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_vals + a.p_old, vals, np * 4, cudaMemcpyHostToDevice, s);
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_row_off + a.r_old + 1, a.off.data(), n * 8, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) { set_error(std::string(what) + ": " + cudaGetErrorString(e)); return CDB_CUDA_ERROR; }
    return CDB_OK;
}

cdb_status PostingStore::deleted_rows(uint64_t first, uint64_t n, uint8_t *out, uint64_t *out_total) const {
    CDB_REQUIRE(first + n <= capacity_rows, "first + n exceeds capacity_rows");
    for (uint64_t i = 0; i < n; ++i) out[i] = (h_deleted[(first + i) >> 5] >> ((first + i) & 31)) & 1u;
    if (out_total) *out_total = n_deleted;
    return CDB_OK;
}

PostingTile PostingStore::tile_at(uint64_t t, uint32_t *np, uint32_t *nr) const {
    const uint64_t r0 = t << TILE_SHIFT, r1 = std::min<uint64_t>(n_rows, r0 + TILE_ROWS);
    PostingTile tile;
    tile.entry_base = h_row_off[r0];   // a tile's entries are its rows' pairs, re-ordered
    tile.key_base = t ? h_tiles[t - 1].key_base + h_tiles[t - 1].n_keys : 0;
    tile.n_keys = 0;
    tile.pad = 0;
    *np = (uint32_t)(h_row_off[r1] - tile.entry_base);
    *nr = (uint32_t)(r1 - r0);
    return tile;
}

cudaError_t PostingStore::sort_tile(BuildBufs &b, uint32_t np, int end_bit, cudaStream_t s) const {
    size_t tb = b.tmp_bytes;
    return cub::DeviceRadixSort::SortPairs(b.tmp, tb, b.keys_in, b.keys_out, b.vals_in, b.vals_out, (int)np, 0, end_bit, s);
}

cdb_status PostingStore::finish_tile(uint64_t t, PostingTile tile, uint32_t np, int seg_shift, const char *dup_error, BuildBufs &b,
                                     cudaStream_t s) {
    uint32_t *tseg = d_tseg + tile.key_base + t;
    if (np == 0) {
        CDB_CUDA_TRY(cudaMemsetAsync(tseg, 0, 4, s));
    } else {
        size_t tb = b.tmp_bytes;
        CDB_CUDA_TRY(cub::DeviceScan::InclusiveSum(b.tmp, tb, b.flags, b.pos, (int)np, s));
        seg_scatter_kernel<<<(np + 255) / 256, 256, 0, s>>>(b.keys_out, b.flags, b.pos, np, seg_shift, d_tkeys + tile.key_base, tseg);
        CDB_LAUNCH_CHECK();
        uint32_t dup = 0;
        CDB_CUDA_TRY(cudaMemcpyAsync(&tile.n_keys, b.pos + np - 1, 4, cudaMemcpyDeviceToHost, s));
        if (dup_error) CDB_CUDA_TRY(cudaMemcpyAsync(&dup, b.dup, 4, cudaMemcpyDeviceToHost, s));
        CDB_CUDA_TRY(cudaStreamSynchronize(s));
        if (dup) { set_error(dup_error); return CDB_INVALID_PARAMS; }
    }
    h_tiles.push_back(tile);
    return CDB_OK;
}

cdb_status PostingStore::upload_tiles(uint64_t t0, uint64_t t1, cudaStream_t s) {
    if (t1 > t0)
        CDB_CUDA_TRY(cudaMemcpyAsync(d_tiles + t0, h_tiles.data() + t0, (t1 - t0) * sizeof(PostingTile), cudaMemcpyHostToDevice, s));
    CDB_CUDA_TRY(cudaStreamSynchronize(s));
    return CDB_OK;
}

cdb_status PostingStore::drop_rows(uint64_t rows, cudaStream_t s) {
    h_row_off.resize(rows + 1);
    n_rows = rows;
    n_pairs = h_row_off[rows];
    for (uint64_t w = rows >> 5; w < h_deleted.size(); ++w) {
        const uint32_t keep = w == (rows >> 5) ? (uint32_t)((1ull << (rows & 31)) - 1) : 0u;
        n_deleted -= __builtin_popcount(h_deleted[w] & ~keep);
        h_deleted[w] &= keep;
    }
    CDB_CUDA_TRY(cudaMemcpyAsync(d_deleted, h_deleted.data(), h_deleted.size() * 4, cudaMemcpyHostToDevice, s));
    return CDB_OK;
}

cdb_status fill_empty_results(uint32_t nq, uint32_t k, uint32_t *d_ids, float *d_scores, uint32_t *d_counts, cudaStream_t s) {
    CDB_CUDA_TRY(cudaMemsetAsync(d_ids, 0xFF, (size_t)nq * k * 4, s));
    CDB_CUDA_TRY(cudaMemsetAsync(d_scores, 0, (size_t)nq * k * 4, s));
    CDB_CUDA_TRY(cudaMemsetAsync(d_counts, 0, (size_t)nq * 4, s));
    return CDB_OK;
}

}  // namespace cdb
