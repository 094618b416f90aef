// api.cu -- the extern "C" boundary declared in include/cosdata_b200.h.
// Host-side orchestration only: device buffers, streams, launch order.  No torch,
// no CPU compute path -- without a CUDA device every entry point fails.
#include <condition_variable>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <shared_mutex>
#include <vector>

#include "kernels.h"
#include "hnsw_traverse.cuh"

namespace cdb {

static thread_local std::string t_last_error;
void set_error(const std::string &msg) { t_last_error = msg; }
std::atomic<uint64_t> g_launch_count{0};
std::atomic<uint32_t> g_hnsw_flags{CDB_HNSW_F_DEFAULT};

cudaError_t allow_max_dynamic_smem(const void *kernel) {
    static std::mutex mu;
    static std::vector<std::pair<int, const void *>> done;
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    std::lock_guard<std::mutex> g(mu);
    for (const auto &d : done)
        if (d.first == dev && d.second == kernel) return cudaSuccess;
    int optin = 0;
    if ((e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev)) != cudaSuccess) return e;
    cudaFuncAttributes fa;
    if ((e = cudaFuncGetAttributes(&fa, kernel)) != cudaSuccess) return e;
    if ((e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, optin - (int)fa.sharedSizeBytes)) != cudaSuccess) return e;
    done.emplace_back(dev, kernel);
    return cudaSuccess;
}

struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
    cdb_status ensure(size_t bytes) {
        if (bytes <= cap) return CDB_OK;
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
        size_t want = bytes + bytes / 4 + 256;
        CDB_CUDA_TRY(cudaMalloc(&p, want));
        cap = want;
        return CDB_OK;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <class T> T *as() const { return reinterpret_cast<T *>(p); }
};

// (metric, storage) arms of DistanceMetric::calculate: OK / StorageMismatch / unimplemented!()
static cdb_status arm_status(int metric, int st) {
    if (st < CDB_ST_U8 || st > CDB_ST_LAST) return CDB_INVALID_PARAMS;
    switch (metric) {
    case CDB_METRIC_COSINE: return CDB_OK;                                                        // cosine.rs:104-216
    case CDB_METRIC_DOT_PRODUCT: return st == CDB_ST_F32 ? CDB_STORAGE_MISMATCH : CDB_OK;          // dotproduct.rs:20-63
    case CDB_METRIC_EUCLIDEAN:                                                                      // euclidean.rs:17-39
        if (st == CDB_ST_U8 || st == CDB_ST_F16 || st == CDB_ST_BF16) return CDB_OK;
        return st == CDB_ST_F32 ? CDB_STORAGE_MISMATCH : CDB_UNSUPPORTED;
    case CDB_METRIC_HAMMING: return st == CDB_ST_F32 ? CDB_STORAGE_MISMATCH : CDB_OK;              // hamming.rs:21-57
    default: return CDB_INVALID_PARAMS;
    }
}

// host code layout: tight [n][code_bytes]; sub-byte planes at p*ceil(D/8)
static size_t host_code_bytes(int st, uint32_t dim) {
    switch (st) {
    case CDB_ST_U8: return dim;
    case CDB_ST_SUB1: case CDB_ST_SUB2: case CDB_ST_SUB3: return (size_t)st * plane_bytes(dim);
    case CDB_ST_F16: case CDB_ST_BF16: return (size_t)dim * 2;
    case CDB_ST_F32: return (size_t)dim * 4;
    default: return 0;
    }
}
static cdb_status copy_codes(void *dst, const void *src, int st, uint32_t dim, uint64_t n, bool to_device, cudaStream_t s) {
    if (!n) return CDB_OK;
    const uint32_t pitch = row_pitch_bytes(st, dim);
    const size_t hb = host_code_bytes(st, dim);
    const cudaMemcpyKind kind = to_device ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToHost;
    if (st >= CDB_ST_SUB1 && st <= CDB_ST_SUB3) {
        const uint32_t nb = plane_bytes(dim), pp = plane_pitch(dim);
        for (int p = 0; p < st; ++p) {
            if (to_device)
                CDB_CUDA_TRY(cudaMemcpy2DAsync((uint8_t *)dst + (size_t)p * pp, pitch, (const uint8_t *)src + (size_t)p * nb, hb, nb, n, kind, s));
            else
                CDB_CUDA_TRY(cudaMemcpy2DAsync((uint8_t *)dst + (size_t)p * nb, hb, (const uint8_t *)src + (size_t)p * pp, pitch, nb, n, kind, s));
        }
    } else {
        if (to_device) CDB_CUDA_TRY(cudaMemcpy2DAsync(dst, pitch, src, hb, hb, n, kind, s));
        else CDB_CUDA_TRY(cudaMemcpy2DAsync(dst, hb, src, pitch, hb, n, kind, s));
    }
    return CDB_OK;
}

// qsel != null: only after a fallback scan ran (n_sel > 0), otherwise the tensor-core path's flags stand
__global__ void err32_to_u8_kernel(const uint32_t *e, uint8_t *out, uint32_t n, const uint32_t *qsel = nullptr) {
    if (qsel && qsel[0] == 0) return;
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (uint8_t)e[i];
}

}  // namespace cdb

using namespace cdb;

// Per-call scratch of a search: every buffer a search writes, its own stream and events.  A handle keeps a small pool of
// these, so concurrent cdb_search_* calls on one handle (several host threads, several streams) do not serialise on a
// single arena -- the index data itself is read-only during a search (SURVEY 8b: the ABI is re-entrant per handle).
struct Scratch {
    DevBuf q_codes, q_mags, partial, err32, io_ids, io_scores, io_counts, io_err, io_q, misc;
    DevBuf qh, gthr, cand, cand_cnt, flags, progress, qsel;
    DevBuf hn_rows, hn_scores, hn_n, qraw, qraw_mags, hn_ids, hn_labels, flt_off, flt_dims, flt_has;
    cudaStream_t stream = nullptr;         // used by the host-buffer entry points
    cudaEvent_t ev[3] = {nullptr, nullptr, nullptr};
    bool ev_valid = false;
    cudaStream_t last_stream = nullptr;    // stream of the previous search on this set (stream-ordered hand-over of the buffers)
    // sharded searches (shard_group.cu): the final kernels also write the packed selection keys of every query here
    // ([nq][k], 0 = empty slot) -- straight into the collective's send buffer.  cur_keys = the current chunk's slice.
    uint64_t *keys_out = nullptr, *cur_keys = nullptr;
    bool busy = false;
    cdb_status init() {
        CDB_CUDA_TRY(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
        for (auto &e : ev) CDB_CUDA_TRY(cudaEventCreate(&e));
        cdb_status rc = flags.ensure(16);
        if (rc) return rc;
        CDB_CUDA_TRY(cudaMemset(flags.p, 0, 16));
        return CDB_OK;
    }
    void destroy() {
        if (stream) cudaStreamSynchronize(stream);
        for (DevBuf *b : {&q_codes, &q_mags, &partial, &err32, &io_ids, &io_scores, &io_counts, &io_err, &io_q, &misc, &qh, &gthr, &cand,
                          &cand_cnt, &flags, &progress, &qsel, &hn_rows, &hn_scores, &hn_n, &qraw, &qraw_mags, &hn_ids, &hn_labels,
                          &flt_off, &flt_dims, &flt_has})
            b->release();
        for (auto &e : ev) if (e) cudaEventDestroy(e);
        if (stream) cudaStreamDestroy(stream);
    }
};

struct cdb_index {
    cdb_index_desc desc{};
    int sm_count = 0;
    uint32_t row_pitch = 0;        // bytes per stored code row
    uint32_t raw_pitch_elems = 0;  // floats per raw row
    uint64_t size = 0;
    uint8_t *d_codes = nullptr;
    float *d_mags = nullptr;
    float *d_raw = nullptr;       // raw f32 rows (may alias d_codes)
    float *d_raw_mags = nullptr;  // |raw row| (may alias d_mags)
    bool raw_owned = false, raw_mags_owned = false;
    uint8_t *d_digits = nullptr;   // sub-byte storage unpacked to u8 digits for the u8 wgmma (tensor_scan_u8.cu)
    uint32_t digit_pitch = 0;
    void *d_xh = nullptr;          // fp16 L2-normalised rows for the wgmma prefilter (tensor_scan.cu)
    uint32_t xh_pitch = 0;         // halfs per shadow row
    uint64_t n_allzero_rows = 0;   // degenerate rows (tensor_scan.cu): all-zero rows score NaN against every query = last
    uint64_t n_odd_rows = 0;       // other degenerate rows (norm 0/inf/NaN/out of range): ride on every candidate list
    uint32_t *h_flags = nullptr;   // pinned host staging (16 words)
    std::atomic<uint64_t> stat_tensor_searches{0};
    cudaStream_t stream = nullptr; // ingest / build stream (exclusive operations)
    static constexpr int EV_RING = 64;
    cudaEvent_t ring0[EV_RING] = {}, ring1[EV_RING] = {};  // per-search (before scan, after scan)
    std::atomic<uint64_t> n_search{0};
    // searches hold the lock shared, operations that change the index (append, graph upload / build) exclusively
    std::shared_mutex rw;
    // scratch pool: sets are created on demand (at most POOL_MAX), a search leases one for its duration
    static constexpr size_t POOL_MAX = 4;
    std::vector<std::unique_ptr<Scratch>> pool;
    std::mutex pool_mu;
    std::condition_variable pool_cv;
    Scratch *last = nullptr;       // set of the most recently finished search (stats / timing queries)
    DevBuf stage, deg;             // ingest staging; degenerate-row bookkeeping (read-only during searches)
    // rows appended as codes into a keep_raw_f32 index have no raw f32 row yet (cold start from prop.data): searches that
    // re-rank with raw rows are refused until cdb_index_set_raw_f32 / cdb_index_fill_raw_from_itoe supplied them
    std::vector<bool> raw_have;
    uint64_t raw_missing = 0;
    // HNSW graph (cdb_index_set_graph)
    bool has_graph = false;
    GraphDev graph{};
    std::vector<void *> graph_allocs;
    // replica ids / metadata of the graph nodes (cdb_index_set_graph_metadata)
    bool has_md = false;
    std::vector<void *> md_allocs;
    const uint32_t *const *md_node_id = nullptr, *const *md_node_md = nullptr;
    const int32_t *md_bits = nullptr;
    const float *md_mags = nullptr;
    uint32_t md_dims = 0, md_pseudo_entry = 0;
    std::vector<uint32_t> g_cnt;
    std::vector<const uint32_t *> g_nr, g_ad, g_ch;  // host copies of the per-level device pointers
    std::vector<const uint32_t *> g_id, g_md;        // same for node_id / node_md when has_md
    DevBuf hn_counters, hn_prof;   // cumulative device counters (atomics: shared by concurrent searches)
    bool hn_prof_on = false;
};

// a leased scratch set; returned to the pool (and remembered as "last") on destruction
struct Lease {
    cdb_index *ix = nullptr;
    Scratch *sc = nullptr;
    ~Lease() {
        if (!sc) return;
        std::lock_guard<std::mutex> g(ix->pool_mu);
        sc->busy = false;
        ix->last = sc;
        ix->pool_cv.notify_one();
    }
};
static cdb_status lease_scratch(cdb_index *ix, Lease &l) {
    std::unique_lock<std::mutex> g(ix->pool_mu);
    for (;;) {
        for (auto &u : ix->pool)
            if (!u->busy) { u->busy = true; l.ix = ix; l.sc = u.get(); return CDB_OK; }
        if (ix->pool.size() < cdb_index::POOL_MAX) {
            std::unique_ptr<Scratch> u(new Scratch());
            cdb_status rc = u->init();
            if (rc) { u->destroy(); return rc; }
            u->busy = true;
            l.ix = ix; l.sc = u.get();
            ix->pool.push_back(std::move(u));
            return CDB_OK;
        }
        ix->pool_cv.wait(g);
    }
}

#define CDB_REQUIRE(cond, msg)                              \
    do {                                                    \
        if (!(cond)) { set_error(msg); return CDB_INVALID_PARAMS; } \
    } while (0)

extern "C" {

int32_t cdb_abi_version(void) { return CDB_ABI_VERSION; }
const char *cdb_last_error_string(void) { return t_last_error.c_str(); }
uint64_t cdb_kernel_launch_count(void) { return g_launch_count.load(); }

cdb_status cdb_device_count(int32_t *out) {
    CDB_REQUIRE(out, "null out");
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) { *out = 0; set_error(std::string("cudaGetDeviceCount: ") + cudaGetErrorString(e)); return CDB_CUDA_ERROR; }
    *out = n;
    return CDB_OK;
}

cdb_status cdb_synth_fill_host(uint64_t seed, uint64_t first_idx, uint64_t n, float *out) {
    CDB_REQUIRE(out || !n, "null out");
    for (uint64_t i = 0; i < n; ++i) out[i] = synth_value(seed, first_idx + i);
    return CDB_OK;
}

size_t cdb_code_bytes(int32_t st, uint32_t dim) { return host_code_bytes(st, dim); }

cdb_status cdb_quantize_batch(int32_t device, int32_t st, float lo, float hi, const float *vecs, uint64_t n, uint32_t dim,
                              void *out_codes, float *out_mags) {
    CDB_REQUIRE(st >= CDB_ST_U8 && st <= CDB_ST_LAST, "bad storage type");
    CDB_REQUIRE(dim > 0 && (vecs || !n) && (out_codes || !n) && (out_mags || !n), "bad arguments");
    CDB_CUDA_TRY(cudaSetDevice(device));
    const uint32_t pitch = row_pitch_bytes(st, dim);
    const uint64_t chunk = std::max<uint64_t>(1, (64ull << 20) / ((size_t)dim * 4));
    DevBuf in, codes, mags;
    cdb_status rc = CDB_OK;
    for (uint64_t off = 0; off < n && rc == CDB_OK; off += chunk) {
        uint64_t m = std::min(chunk, n - off);
        if ((rc = in.ensure(m * dim * 4)) || (rc = codes.ensure(m * pitch)) || (rc = mags.ensure(m * 4))) break;
        cudaMemcpyAsync(in.p, vecs + off * dim, m * dim * 4, cudaMemcpyHostToDevice, 0);
        cudaMemsetAsync(codes.p, 0, m * pitch, 0);
        rc = quantize_rows_device(in.as<float>(), m, dim, st, lo, hi, codes.as<uint8_t>(), pitch, mags.as<float>(), nullptr, 0, 0);
        if (rc) break;
        rc = copy_codes((uint8_t *)out_codes + off * host_code_bytes(st, dim), codes.p, st, dim, m, false, 0);
        if (rc) break;
        cudaMemcpyAsync(out_mags + off, mags.p, m * 4, cudaMemcpyDeviceToHost, 0);
        cudaError_t e = cudaStreamSynchronize(0);
        if (e != cudaSuccess) { set_error(cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; }
    }
    in.release(); codes.release(); mags.release();
    return rc;
}

static cdb_status finish_sampling(const unsigned long long *d_counts, uint64_t n_values, float clamp, const uint64_t *prior,
                                  uint64_t prior_values, uint64_t *out_counts, float *out_range, cudaStream_t s) {
    uint64_t c[CDB_SAMPLE_COUNTERS];
    CDB_CUDA_TRY(cudaMemcpyAsync(c, d_counts, sizeof(c), cudaMemcpyDeviceToHost, s));
    CDB_CUDA_TRY(cudaStreamSynchronize(s));
    for (int i = 0; i < CDB_SAMPLE_COUNTERS; ++i) {
        if (prior) c[i] += prior[i];
        if (out_counts) out_counts[i] = c[i];
    }
    if (out_range) values_range_from_counts(c, n_values + (prior ? prior_values : 0), clamp, out_range);
    return CDB_OK;
}

cdb_status cdb_sample_values_range_device(int32_t device, const float *d_vecs, uint64_t n, uint32_t dim, float clamp,
                                          const uint64_t *prior, uint64_t prior_values, uint64_t *out_counts,
                                          float *out_range, void *stream) {
    CDB_REQUIRE((d_vecs || !n) && (out_counts || out_range), "bad arguments");
    CDB_CUDA_TRY(cudaSetDevice(device));
    int sms = 0;
    CDB_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    cudaStream_t s = (cudaStream_t)stream;
    DevBuf counts;
    cdb_status rc = counts.ensure(CDB_SAMPLE_COUNTERS * 8);
    if (rc) return rc;
    cudaMemsetAsync(counts.p, 0, CDB_SAMPLE_COUNTERS * 8, s);
    rc = sample_counts_device(d_vecs, n * dim, counts.as<unsigned long long>(), sms, s);
    if (!rc) rc = finish_sampling(counts.as<unsigned long long>(), n * dim, clamp, prior, prior_values, out_counts, out_range, s);
    counts.release();
    return rc;
}

cdb_status cdb_sample_values_range(int32_t device, const float *vecs, uint64_t n, uint32_t dim, float clamp,
                                   const uint64_t *prior, uint64_t prior_values, uint64_t *out_counts, float *out_range) {
    CDB_REQUIRE((vecs || !n) && (out_counts || out_range), "bad arguments");
    CDB_CUDA_TRY(cudaSetDevice(device));
    int sms = 0;
    CDB_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    const uint64_t total = n * dim;
    const uint64_t chunk = 16ull << 20;   // values per staging copy (64 MB)
    DevBuf in, counts;
    cdb_status rc = counts.ensure(CDB_SAMPLE_COUNTERS * 8);
    if (!rc) rc = in.ensure(std::min(std::max<uint64_t>(total, 1), chunk) * 4);
    if (!rc) {
        cudaMemsetAsync(counts.p, 0, CDB_SAMPLE_COUNTERS * 8, 0);
        for (uint64_t off = 0; off < total && !rc; off += chunk) {
            const uint64_t m = std::min(chunk, total - off);
            cudaMemcpyAsync(in.p, vecs + off, m * 4, cudaMemcpyHostToDevice, 0);
            rc = sample_counts_device(in.as<float>(), m, counts.as<unsigned long long>(), sms, 0);
        }
    }
    if (!rc) rc = finish_sampling(counts.as<unsigned long long>(), total, clamp, prior, prior_values, out_counts, out_range, 0);
    in.release(); counts.release();
    return rc;
}

cdb_status cdb_distance_pairs(int32_t device, int32_t metric, int32_t st, uint32_t dim, const void *x_codes,
                              const float *x_mags, const void *y_codes, const float *y_mags, uint64_t n, float *out,
                              int32_t *out_status) {
    CDB_REQUIRE(st >= CDB_ST_U8 && st <= CDB_ST_LAST && metric >= 0 && metric <= 3 && dim > 0, "bad metric/storage/dim");
    if (!n) return CDB_OK;
    CDB_REQUIRE(x_codes && y_codes && x_mags && y_mags && out && out_status, "null buffer");
    CDB_CUDA_TRY(cudaSetDevice(device));
    const uint32_t pitch = row_pitch_bytes(st, dim);
    DevBuf x, y, xm, ym, o, os;
    cdb_status rc;
    if ((rc = x.ensure(n * pitch)) || (rc = y.ensure(n * pitch)) || (rc = xm.ensure(n * 4)) || (rc = ym.ensure(n * 4)) ||
        (rc = o.ensure(n * 4)) || (rc = os.ensure(n * 4)))
        goto done;
    cudaMemsetAsync(x.p, 0, n * pitch, 0);
    cudaMemsetAsync(y.p, 0, n * pitch, 0);
    if ((rc = copy_codes(x.p, x_codes, st, dim, n, true, 0)) || (rc = copy_codes(y.p, y_codes, st, dim, n, true, 0))) goto done;
    cudaMemcpyAsync(xm.p, x_mags, n * 4, cudaMemcpyHostToDevice, 0);
    cudaMemcpyAsync(ym.p, y_mags, n * 4, cudaMemcpyHostToDevice, 0);
    rc = distance_pairs_device(metric, st, dim, x.as<uint8_t>(), xm.as<float>(), y.as<uint8_t>(), ym.as<float>(), pitch, n,
                               o.as<float>(), os.as<int32_t>(), 0);
    if (rc) goto done;
    cudaMemcpyAsync(out, o.p, n * 4, cudaMemcpyDeviceToHost, 0);
    cudaMemcpyAsync(out_status, os.p, n * 4, cudaMemcpyDeviceToHost, 0);
    {
        cudaError_t e = cudaStreamSynchronize(0);
        if (e != cudaSuccess) { set_error(cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; }
    }
done:
    x.release(); y.release(); xm.release(); ym.release(); o.release(); os.release();
    return rc;
}

cdb_status cdb_distance_pairs_md(int32_t device, int32_t metric, int32_t st, uint32_t dim, uint32_t M, const cdb_vector_data_batch *x,
                                 const cdb_vector_data_batch *y, uint64_t n, float *out, int32_t *out_status) {
    CDB_REQUIRE(st >= CDB_ST_U8 && st <= CDB_ST_LAST && metric >= 0 && metric <= 3 && dim > 0, "bad metric/storage/dim");
    CDB_REQUIRE(x && y, "null argument");
    if (!n) return CDB_OK;
    CDB_REQUIRE(x->codes && y->codes && x->mags && y->mags && out && out_status, "null buffer");
    CDB_REQUIRE((!x->md_bits || (x->md_mags && M)) && (!y->md_bits || (y->md_mags && M)), "metadata needs md_mags and md_dims");
    CDB_CUDA_TRY(cudaSetDevice(device));
    const uint32_t pitch = row_pitch_bytes(st, dim);
    std::vector<DevBuf> bufs(16);
    size_t nb = 0;
    cdb_status rc = CDB_OK;
    auto up = [&](const void *src, size_t bytes) -> const void * {
        if (!src || rc) return nullptr;
        DevBuf &b = bufs[nb++];
        if ((rc = b.ensure(bytes))) return nullptr;
        cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, 0);
        return b.p;
    };
    auto side = [&](const cdb_vector_data_batch *v) -> MdBatchDev {
        MdBatchDev d{};
        DevBuf &c = bufs[nb++];
        if (!rc && !(rc = c.ensure(n * pitch))) {
            cudaMemsetAsync(c.p, 0, n * pitch, 0);
            rc = copy_codes(c.p, v->codes, st, dim, n, true, 0);
        }
        d.codes = c.as<uint8_t>();
        d.mags = (const float *)up(v->mags, n * 4);
        d.ids = (const uint32_t *)up(v->ids, n * 4);
        d.has_id = (const uint8_t *)up(v->ids ? v->has_id : nullptr, n);
        d.md_bits = (const int32_t *)up(v->md_bits, n * (size_t)M * 4);
        d.md_mags = (const float *)up(v->md_bits ? v->md_mags : nullptr, n * 4);
        d.has_md = (const uint8_t *)up(v->md_bits ? v->has_md : nullptr, n);
        return d;
    };
    const MdBatchDev dx = side(x), dy = side(y);
    DevBuf &o = bufs[nb++], &os = bufs[nb++];
    if (!rc && !(rc = o.ensure(n * 4)) && !(rc = os.ensure(n * 4)))
        rc = distance_pairs_md_device(metric, st, dim, M, dx, dy, pitch, n, o.as<float>(), os.as<int32_t>(), 0);
    if (!rc) {
        cudaMemcpyAsync(out, o.p, n * 4, cudaMemcpyDeviceToHost, 0);
        cudaMemcpyAsync(out_status, os.p, n * 4, cudaMemcpyDeviceToHost, 0);
        cudaError_t e = cudaStreamSynchronize(0);
        if (e != cudaSuccess) { set_error(cudaGetErrorString(e)); rc = CDB_CUDA_ERROR; }
    }
    for (DevBuf &b : bufs) b.release();
    return rc;
}

// ------------------------------------------------------------------ index lifecycle

cdb_status cdb_index_create(const cdb_index_desc *d, cdb_index **out) {
    CDB_REQUIRE(d && out, "null argument");
    CDB_REQUIRE(d->dim > 0 && d->storage_type >= CDB_ST_U8 && d->storage_type <= CDB_ST_LAST, "bad dim/storage type");
    CDB_REQUIRE(d->metric >= CDB_METRIC_COSINE && d->metric <= CDB_METRIC_DOT_PRODUCT, "bad metric");
    CDB_REQUIRE(d->capacity > 0 && d->capacity < 0xFFFFFFFFull, "capacity must be in 1..2^32-2");
    CDB_CUDA_TRY(cudaSetDevice(d->device));
    int sms = 0;
    CDB_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, d->device));
    cdb_index *ix = new cdb_index();
    ix->desc = *d;
    ix->sm_count = sms;
    ix->row_pitch = row_pitch_bytes(d->storage_type, d->dim);
    ix->raw_pitch_elems = round_up(d->dim * 4, 16) / 4;
    auto fail = [&](cudaError_t e, const char *what) {
        set_error(std::string(what) + ": " + cudaGetErrorString(e));
        cdb_index_destroy(ix);
        return CDB_CUDA_ERROR;
    };
    cudaError_t e;
    if ((e = cudaStreamCreateWithFlags(&ix->stream, cudaStreamNonBlocking)) != cudaSuccess) return fail(e, "stream");
    for (int i = 0; i < cdb_index::EV_RING; ++i)
        if ((e = cudaEventCreate(&ix->ring0[i])) != cudaSuccess || (e = cudaEventCreate(&ix->ring1[i])) != cudaSuccess) return fail(e, "event");
    if ((e = cudaMalloc(&ix->d_codes, (size_t)d->capacity * ix->row_pitch)) != cudaSuccess) return fail(e, "cudaMalloc(codes)");
    if ((e = cudaMemsetAsync(ix->d_codes, 0, (size_t)d->capacity * ix->row_pitch, ix->stream)) != cudaSuccess) return fail(e, "memset");
    if ((e = cudaMalloc(&ix->d_mags, (size_t)d->capacity * 4)) != cudaSuccess) return fail(e, "cudaMalloc(mags)");
    if (d->storage_type == CDB_ST_F32) {
        ix->d_raw = reinterpret_cast<float *>(ix->d_codes);
        ix->d_raw_mags = ix->d_mags;
    } else if (d->keep_raw_f32) {
        if ((e = cudaMalloc(&ix->d_raw, (size_t)d->capacity * ix->raw_pitch_elems * 4)) != cudaSuccess) return fail(e, "cudaMalloc(raw)");
        ix->raw_owned = true;
        if ((e = cudaMemsetAsync(ix->d_raw, 0, (size_t)d->capacity * ix->raw_pitch_elems * 4, ix->stream)) != cudaSuccess) return fail(e, "memset");
        if (d->storage_type == CDB_ST_U8) {
            if ((e = cudaMalloc(&ix->d_raw_mags, (size_t)d->capacity * 4)) != cudaSuccess) return fail(e, "cudaMalloc(raw mags)");
            ix->raw_mags_owned = true;
        } else {
            ix->d_raw_mags = ix->d_mags;  // same formula: sequential fold of the original values
        }
    }
    if (d->tensor_prefilter && ix->d_raw) {
        ix->xh_pitch = round_up(d->dim * 2, 16) / 2;
        if ((e = cudaMalloc(&ix->d_xh, (size_t)d->capacity * ix->xh_pitch * 2)) != cudaSuccess) return fail(e, "cudaMalloc(fp16 shadow)");
        if ((e = cudaMemsetAsync(ix->d_xh, 0, (size_t)d->capacity * ix->xh_pitch * 2, ix->stream)) != cudaSuccess) return fail(e, "memset");
    }
    if (d->tensor_prefilter && d->storage_type >= CDB_ST_SUB1 && d->storage_type <= CDB_ST_SUB3) {
        ix->digit_pitch = round_up(d->dim, 16);
        if ((e = cudaMalloc(&ix->d_digits, (size_t)d->capacity * ix->digit_pitch)) != cudaSuccess) return fail(e, "cudaMalloc(digits)");
        if ((e = cudaMemsetAsync(ix->d_digits, 0, (size_t)d->capacity * ix->digit_pitch, ix->stream)) != cudaSuccess) return fail(e, "memset");
    }
    if ((e = cudaMallocHost(&ix->h_flags, 64)) != cudaSuccess) return fail(e, "cudaMallocHost");
    if (ix->deg.ensure(TS_DEG_WORDS * 4) != CDB_OK) return fail(cudaErrorMemoryAllocation, "deg");
    if ((e = cudaMemsetAsync(ix->deg.p, 0, TS_DEG_WORDS * 4, ix->stream)) != cudaSuccess) return fail(e, "memset");
    if ((e = cudaStreamSynchronize(ix->stream)) != cudaSuccess) return fail(e, "sync");
    *out = ix;
    return CDB_OK;
}

cdb_status cdb_index_destroy(cdb_index *ix) {
    if (!ix) return CDB_OK;
    cudaSetDevice(ix->desc.device);
    if (ix->stream) cudaStreamSynchronize(ix->stream);
    if (ix->d_codes) cudaFree(ix->d_codes);
    if (ix->d_mags) cudaFree(ix->d_mags);
    if (ix->raw_owned && ix->d_raw) cudaFree(ix->d_raw);
    if (ix->raw_mags_owned && ix->d_raw_mags) cudaFree(ix->d_raw_mags);
    if (ix->d_xh) cudaFree(ix->d_xh);
    if (ix->d_digits) cudaFree(ix->d_digits);
    for (void *g : ix->graph_allocs) cudaFree(g);
    for (void *g : ix->md_allocs) cudaFree(g);
    if (ix->h_flags) cudaFreeHost(ix->h_flags);
    for (auto &u : ix->pool) u->destroy();
    ix->pool.clear();
    for (DevBuf *b : {&ix->stage, &ix->deg, &ix->hn_counters, &ix->hn_prof}) b->release();
    for (int i = 0; i < cdb_index::EV_RING; ++i) {
        if (ix->ring0[i]) cudaEventDestroy(ix->ring0[i]);
        if (ix->ring1[i]) cudaEventDestroy(ix->ring1[i]);
    }
    if (ix->stream) cudaStreamDestroy(ix->stream);
    delete ix;
    return CDB_OK;
}

cdb_status cdb_index_describe(const cdb_index *ix, cdb_index_desc *out) {
    CDB_REQUIRE(ix && out, "null argument");
    *out = ix->desc;
    return CDB_OK;
}

uint64_t cdb_index_size(const cdb_index *ix) { return ix ? ix->size : 0; }

static cdb_status index_after_append(cdb_index *ix, uint64_t first, uint64_t n) {
    cdb_status rc;
    if (ix->raw_mags_owned &&
        (rc = raw_mags_device(ix->d_raw + first * ix->raw_pitch_elems, ix->raw_pitch_elems, n, ix->desc.dim,
                              ix->d_raw_mags + first, ix->stream)))
        return rc;
    if (ix->d_digits &&
        (rc = unpack_digits_device(ix->d_codes + first * ix->row_pitch, ix->row_pitch, n, ix->desc.dim, ix->desc.storage_type,
                                   ix->d_digits + first * ix->digit_pitch, ix->digit_pitch, ix->stream)))
        return rc;
    if (ix->d_xh) {
        if ((rc = normalize_f16_device(ix->d_raw + first * ix->raw_pitch_elems, ix->raw_pitch_elems, ix->d_raw_mags + first, n,
                                       ix->desc.dim, (uint8_t *)ix->d_xh + first * ix->xh_pitch * 2, ix->xh_pitch, ix->stream)))
            return rc;
        // deg[0], deg[1] accumulate the all-zero / other degenerate rows, deg[2..] lists the first of the latter
        if ((rc = classify_rows_device(ix->d_raw + first * ix->raw_pitch_elems, ix->raw_pitch_elems, ix->d_raw_mags + first, n,
                                       ix->desc.dim, (uint32_t)first, ix->deg.as<uint32_t>(), ix->stream)))
            return rc;
        CDB_CUDA_TRY(cudaMemcpyAsync(ix->h_flags + 4, ix->deg.p, 8, cudaMemcpyDeviceToHost, ix->stream));
        CDB_CUDA_TRY(cudaStreamSynchronize(ix->stream));
        ix->n_allzero_rows = ix->h_flags[4];
        ix->n_odd_rows = ix->h_flags[5];
    }
    return CDB_OK;
}

static cdb_status append_f32_locked(cdb_index *ix, const float *vecs, uint64_t n);
cdb_status cdb_index_append_f32(cdb_index *ix, const float *vecs, uint64_t n) {
    CDB_REQUIRE(ix && (vecs || !n), "null argument");
    std::unique_lock<std::shared_mutex> lock(ix->rw);
    return append_f32_locked(ix, vecs, n);
}
static cdb_status append_f32_locked(cdb_index *ix, const float *vecs, uint64_t n) {
    CDB_REQUIRE(ix->size + n <= ix->desc.capacity, "append exceeds capacity");
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    const uint32_t dim = ix->desc.dim;
    const uint64_t chunk = std::max<uint64_t>(1, (256ull << 20) / ((size_t)dim * 4));
    for (uint64_t off = 0; off < n; off += chunk) {
        uint64_t m = std::min(chunk, n - off);
        cdb_status rc = ix->stage.ensure(m * dim * 4);
        if (rc) return rc;
        CDB_CUDA_TRY(cudaMemcpyAsync(ix->stage.p, vecs + off * dim, m * dim * 4, cudaMemcpyHostToDevice, ix->stream));
        uint64_t first = ix->size;
        float *raw = ix->raw_owned ? ix->d_raw + first * ix->raw_pitch_elems : nullptr;
        rc = quantize_rows_device(ix->stage.as<float>(), m, dim, ix->desc.storage_type, ix->desc.range_lo, ix->desc.range_hi,
                                  ix->d_codes + first * ix->row_pitch, ix->row_pitch, ix->d_mags + first, raw,
                                  ix->raw_pitch_elems, ix->stream);
        if (rc) return rc;
        if ((rc = index_after_append(ix, first, m))) return rc;
        CDB_CUDA_TRY(cudaStreamSynchronize(ix->stream));
        ix->size += m;
    }
    return CDB_OK;
}

cdb_status cdb_index_append_f32_device(cdb_index *ix, const float *d_vecs, uint64_t n) {
    CDB_REQUIRE(ix && (d_vecs || !n), "null argument");
    std::unique_lock<std::shared_mutex> lock(ix->rw);
    CDB_REQUIRE(ix->size + n <= ix->desc.capacity, "append exceeds capacity");
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    if (!n) return CDB_OK;
    const uint64_t first = ix->size;
    float *raw = ix->raw_owned ? ix->d_raw + first * ix->raw_pitch_elems : nullptr;
    cdb_status rc = quantize_rows_device(d_vecs, n, ix->desc.dim, ix->desc.storage_type, ix->desc.range_lo, ix->desc.range_hi,
                                         ix->d_codes + first * ix->row_pitch, ix->row_pitch, ix->d_mags + first, raw,
                                         ix->raw_pitch_elems, ix->stream);
    if (rc) return rc;
    if ((rc = index_after_append(ix, first, n))) return rc;
    CDB_CUDA_TRY(cudaStreamSynchronize(ix->stream));
    ix->size += n;
    return CDB_OK;
}

cdb_status cdb_index_append_codes(cdb_index *ix, const void *codes, const float *mags, uint64_t n) {
    CDB_REQUIRE(ix && ((codes && mags) || !n), "null argument");
    std::unique_lock<std::shared_mutex> lock(ix->rw);
    CDB_REQUIRE(ix->size + n <= ix->desc.capacity, "append exceeds capacity");
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    cdb_status rc = copy_codes(ix->d_codes + ix->size * ix->row_pitch, codes, ix->desc.storage_type, ix->desc.dim, n, true, ix->stream);
    if (rc) return rc;
    CDB_CUDA_TRY(cudaMemcpyAsync(ix->d_mags + ix->size, mags, n * 4, cudaMemcpyHostToDevice, ix->stream));
    if (ix->raw_owned) {
        // keep_raw_f32 index: the raw rows arrive later (cdb_index_set_raw_f32 / cdb_index_fill_raw_from_itoe); until then the
        // rows stay zero and are counted as missing.  Digits are derived from the codes and can be built now.
        if (ix->d_digits && (rc = unpack_digits_device(ix->d_codes + ix->size * ix->row_pitch, ix->row_pitch, n, ix->desc.dim,
                                                       ix->desc.storage_type, ix->d_digits + ix->size * ix->digit_pitch, ix->digit_pitch, ix->stream)))
            return rc;
        if (ix->raw_have.size() < ix->size) ix->raw_have.resize(ix->size, true);
        ix->raw_have.resize(ix->size + n, false);
        ix->raw_missing += n;
    } else if ((rc = index_after_append(ix, ix->size, n))) {
        return rc;
    }
    CDB_CUDA_TRY(cudaStreamSynchronize(ix->stream));
    ix->size += n;
    return CDB_OK;
}

cdb_status cdb_index_set_raw_f32(cdb_index *ix, uint64_t first_row, const float *vecs, uint64_t n) {
    CDB_REQUIRE(ix && (vecs || !n), "null argument");
    std::unique_lock<std::shared_mutex> lock(ix->rw);
    CDB_REQUIRE(ix->raw_owned, "the index keeps no separate raw f32 rows (F32 storage or keep_raw_f32 = 0)");
    CDB_REQUIRE(first_row + n <= ix->size, "row range out of bounds");
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    const uint32_t dim = ix->desc.dim;
    const uint64_t chunk = std::max<uint64_t>(1, (256ull << 20) / ((size_t)dim * 4));
    for (uint64_t off = 0; off < n; off += chunk) {
        const uint64_t m = std::min(chunk, n - off), first = first_row + off;
        CDB_CUDA_TRY(cudaMemcpy2DAsync(ix->d_raw + first * ix->raw_pitch_elems, (size_t)ix->raw_pitch_elems * 4, vecs + off * dim,
                                       (size_t)dim * 4, (size_t)dim * 4, m, cudaMemcpyHostToDevice, ix->stream));
        cdb_status rc;
        if (ix->raw_mags_owned &&
            (rc = raw_mags_device(ix->d_raw + first * ix->raw_pitch_elems, ix->raw_pitch_elems, m, dim, ix->d_raw_mags + first, ix->stream)))
            return rc;
        if (ix->d_xh) {
            if ((rc = normalize_f16_device(ix->d_raw + first * ix->raw_pitch_elems, ix->raw_pitch_elems, ix->d_raw_mags + first, m, dim,
                                           (uint8_t *)ix->d_xh + first * ix->xh_pitch * 2, ix->xh_pitch, ix->stream)) ||
                (rc = classify_rows_device(ix->d_raw + first * ix->raw_pitch_elems, ix->raw_pitch_elems, ix->d_raw_mags + first, m, dim,
                                           (uint32_t)first, ix->deg.as<uint32_t>(), ix->stream)))
                return rc;
            CDB_CUDA_TRY(cudaMemcpyAsync(ix->h_flags + 4, ix->deg.p, 8, cudaMemcpyDeviceToHost, ix->stream));
        }
        CDB_CUDA_TRY(cudaStreamSynchronize(ix->stream));
        if (ix->d_xh) { ix->n_allzero_rows = ix->h_flags[4]; ix->n_odd_rows = ix->h_flags[5]; }
    }
    if (ix->raw_have.size() < ix->size) ix->raw_have.resize(ix->size, true);
    for (uint64_t r = first_row; r < first_row + n; ++r)
        if (!ix->raw_have[r]) { ix->raw_have[r] = true; --ix->raw_missing; }
    return CDB_OK;
}

uint64_t cdb_index_raw_missing(const cdb_index *ix) { return ix ? ix->raw_missing : 0; }

cdb_status cdb_index_append_synthetic(cdb_index *ix, uint64_t seed, uint64_t first_row, uint64_t n) {
    CDB_REQUIRE(ix, "null index");
    std::unique_lock<std::shared_mutex> lock(ix->rw);
    CDB_REQUIRE(ix->size + n <= ix->desc.capacity, "append exceeds capacity");
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    uint64_t first = ix->size;
    float *raw = ix->raw_owned ? ix->d_raw + first * ix->raw_pitch_elems : nullptr;
    cdb_status rc = quantize_rows_synth(seed, first_row, n, ix->desc.dim, ix->desc.storage_type, ix->desc.range_lo,
                                        ix->desc.range_hi, ix->d_codes + first * ix->row_pitch, ix->row_pitch,
                                        ix->d_mags + first, raw, ix->raw_pitch_elems, ix->stream);
    if (rc) return rc;
    if ((rc = index_after_append(ix, first, n))) return rc;
    CDB_CUDA_TRY(cudaStreamSynchronize(ix->stream));
    ix->size += n;
    return CDB_OK;
}

cdb_status cdb_index_read_codes(const cdb_index *ix, uint64_t first, uint64_t n, void *out_codes, float *out_mags) {
    CDB_REQUIRE(ix && first + n <= ix->size, "range out of bounds");
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    if (out_codes) {
        cdb_status rc = copy_codes(out_codes, ix->d_codes + first * ix->row_pitch, ix->desc.storage_type, ix->desc.dim, n, false, ix->stream);
        if (rc) return rc;
    }
    if (out_mags) CDB_CUDA_TRY(cudaMemcpyAsync(out_mags, ix->d_mags + first, n * 4, cudaMemcpyDeviceToHost, ix->stream));
    CDB_CUDA_TRY(cudaStreamSynchronize(ix->stream));
    return CDB_OK;
}

// ------------------------------------------------------------------ S1 search

// prepared (quantized) queries live in sc->q_codes / sc->q_mags.
// qsel == null: unconditional scan of the whole batch.  Otherwise the device decides (ScanArgs): a selective scan of the
// <= SCAN_SEL_CAP queries the tensor-core path could not answer, or -- if there are more -- the whole batch again.
static cdb_status exact_scan_locked(cdb_index *ix, Scratch *sc, bool raw, int st, int metric, uint32_t pitch, uint32_t nq, uint32_t k,
                                    uint32_t *d_ids, float *d_scores, uint32_t *d_counts, uint8_t *d_err, cudaStream_t s,
                                    const uint32_t *qsel = nullptr) {
    const cdb_index_desc &d = ix->desc;
    cdb_status rc;
    ScanArgs a{};
    a.rows = raw ? reinterpret_cast<const uint8_t *>(ix->d_raw) : ix->d_codes;
    a.row_pitch = pitch;
    a.mags = raw ? ix->d_raw_mags : ix->d_mags;
    a.n = ix->size;
    a.dim = d.dim;
    a.st = st;
    a.metric = metric;
    a.raw_mode = raw ? 1 : 0;
    a.q = sc->q_codes.as<uint8_t>();
    a.qmags = sc->q_mags.as<float>();
    a.nq = nq;
    a.k = k;
    a.id_base = d.id_base;
    a.nsplit = scan_plan_nsplit(a, ix->sm_count);
    a.qsel = qsel;
    a.sel_cap = SCAN_SEL_CAP;
    a.sel_grid = scan_sel_grid(ix->sm_count, k);
    const size_t part_full = (size_t)nq * a.nsplit * k * 8, part_sel = qsel ? (size_t)SCAN_SEL_CAP * a.sel_grid * k * 8 : 0;
    if ((rc = sc->partial.ensure(std::max(part_full, part_sel))) || (rc = sc->err32.ensure((size_t)nq * 4))) return rc;
    a.partial = sc->partial.as<uint64_t>();
    a.err32 = sc->err32.as<uint32_t>();
    if (!qsel) CDB_CUDA_TRY(cudaMemsetAsync(a.err32, 0, (size_t)nq * 4, s));   // the tensor-core path prepared it otherwise
    if (qsel) {
        a.sel_mode = 1;
        if ((rc = scan_topk_device(a, s))) return rc;
        if ((rc = merge_partials_device(metric, a.partial, nq, a.nsplit, k, d_ids, d_scores, d_counts, s, qsel, a.sel_cap, 1,
                                        a.sel_grid, scan_sel_qb(a), sc->cur_keys)))
            return rc;
        a.sel_mode = 0;
    }
    if ((rc = scan_topk_device(a, s))) return rc;
    if ((rc = merge_partials_device(metric, a.partial, nq, a.nsplit, k, d_ids, d_scores, d_counts, s, qsel, a.sel_cap, 0, 0, 0,
                                    sc->cur_keys)))
        return rc;
    if (d_err) {
        err32_to_u8_kernel<<<(nq + 255) / 256, 256, 0, s>>>(a.err32, d_err, nq, qsel);
        CDB_LAUNCH_CHECK();
    }
    return CDB_OK;
}

// search_internal (hnsw/mod.rs:390-440): quantized ann_search on the uploaded graph, then
// remove_duplicates_and_filter and the exact f32 re-rank of finalize_ann_results.
static cdb_status hnsw_search_locked(cdb_index *ix, Scratch *sc, const float *d_queries, uint32_t nq, const cdb_search_params *p,
                                     uint32_t *d_ids, float *d_scores, uint32_t *d_counts, uint8_t *d_err, cudaStream_t s,
                                     const uint32_t *d_foff = nullptr, const int8_t *d_fdims = nullptr, const uint8_t *d_fhas = nullptr) {
    const cdb_index_desc &d = ix->desc;
    CDB_REQUIRE(ix->has_graph, "CDB_MODE_HNSW needs cdb_index_set_graph");
    CDB_REQUIRE(ix->has_md || !d_fhas, "metadata filters need cdb_index_set_graph_metadata");
    CDB_REQUIRE(ix->d_raw, "HNSW search re-ranks with raw f32 rows (F32 storage or keep_raw_f32)");
    CDB_REQUIRE(ix->raw_missing == 0, "rows appended as codes still lack their raw f32 rows (cdb_index_set_raw_f32 / cdb_index_fill_raw_from_itoe)");
    CDB_REQUIRE(p->shortlist_size >= 1 && p->shortlist_size <= 64, "shortlist_size must be in 1..64");
    CDB_REQUIRE(p->ef_search >= 1 && p->ef_search <= 4096, "ef_search must be in 1..4096");
    cdb_status rc;
    if ((rc = arm_status(d.metric, d.storage_type)) != CDB_OK) {
        set_error("metric/storage arm is an Err in the reference (StorageMismatch / unimplemented)");
        return rc;
    }
    const uint32_t out_cap = (ix->graph.num_levels + 1) * 100;
    const uint32_t k5 = 5 * p->k;
    const uint32_t rpitch = ix->raw_pitch_elems * 4;
    if ((rc = sc->q_codes.ensure((size_t)nq * ix->row_pitch)) || (rc = sc->q_mags.ensure((size_t)nq * 4)) ||
        (rc = sc->qraw.ensure((size_t)nq * rpitch)) || (rc = sc->qraw_mags.ensure((size_t)nq * 4)) ||
        (rc = sc->hn_rows.ensure((size_t)nq * out_cap * 4)) || (rc = sc->hn_scores.ensure((size_t)nq * out_cap * 4)) ||
        (rc = sc->hn_n.ensure((size_t)nq * 4)) || (rc = sc->err32.ensure((size_t)nq * 4)) ||
        (rc = sc->cand.ensure((size_t)nq * k5 * 4)) || (rc = sc->cand_cnt.ensure((size_t)nq * 4)))
        return rc;
    if (ix->has_md && ((rc = sc->hn_ids.ensure((size_t)nq * out_cap * 4)) || (rc = sc->hn_labels.ensure((size_t)nq * k5 * 4)))) return rc;
    if (!ix->hn_counters.p) {
        if ((rc = ix->hn_counters.ensure(16))) return rc;
        CDB_CUDA_TRY(cudaMemsetAsync(ix->hn_counters.p, 0, 16, s));
    }
    CDB_CUDA_TRY(cudaMemsetAsync(sc->q_codes.p, 0, (size_t)nq * ix->row_pitch, s));
    CDB_CUDA_TRY(cudaMemsetAsync(sc->qraw.p, 0, (size_t)nq * rpitch, s));
    CDB_CUDA_TRY(cudaMemsetAsync(sc->err32.p, 0, (size_t)nq * 4, s));
    // the query is quantized like a stored vector (hnsw/mod.rs:399-403); the re-rank uses the raw query
    if ((rc = quantize_rows_device(d_queries, nq, d.dim, d.storage_type, d.range_lo, d.range_hi, sc->q_codes.as<uint8_t>(),
                                   ix->row_pitch, sc->q_mags.as<float>(), nullptr, 0, s)) ||
        (rc = quantize_rows_device(d_queries, nq, d.dim, CDB_ST_F32, 0.f, 0.f, sc->qraw.as<uint8_t>(), rpitch,
                                   sc->qraw_mags.as<float>(), nullptr, 0, s)))
        return rc;
    HnswArgs a{};
    a.g = ix->graph;
    a.rows = ix->d_codes;
    a.row_pitch = ix->row_pitch;
    a.mags = ix->d_mags;
    a.dim = d.dim;
    a.st = d.storage_type;
    a.metric = d.metric;
    a.q = sc->q_codes.as<uint8_t>();
    a.qmags = sc->q_mags.as<float>();
    a.nq = nq;
    a.ef = p->ef_search;
    a.shortlist = p->shortlist_size;
    a.out_cap = out_cap;
    a.out_rows = sc->hn_rows.as<uint32_t>();
    a.out_scores = sc->hn_scores.as<float>();
    a.out_n = sc->hn_n.as<uint32_t>();
    a.err32 = sc->err32.as<uint32_t>();
    a.counters = ix->hn_counters.as<unsigned long long>();
    const int slot = (int)(ix->n_search.fetch_add(1) % cdb_index::EV_RING);
    CDB_CUDA_TRY(cudaEventRecord(sc->ev[0], s));
    CDB_CUDA_TRY(cudaEventRecord(ix->ring0[slot], s));
    if (ix->has_md) {
        // graph with replica nodes: metadata-aware traversal (hnsw_md.cu); results carry replica ids, the re-rank scores
        // the base vector of each replica (collection.rs:368-384)
        HnswMdArgs ma{};
        ma.a = a;
        ma.node_id = ix->md_node_id;
        ma.node_md = ix->md_node_md;
        ma.md_bits = ix->md_bits;
        ma.md_mags = ix->md_mags;
        ma.M = ix->md_dims;
        ma.pseudo_entry = ix->md_pseudo_entry;
        ma.filter_offsets = d_foff;
        ma.filter_dims = d_fdims;
        ma.has_filter = d_fhas;
        ma.out_ids = sc->hn_ids.as<uint32_t>();
        if ((rc = hnsw_search_md_device(ma, s))) return rc;
        CDB_CUDA_TRY(cudaEventRecord(ix->ring1[slot], s));
        if ((rc = hnsw_dedup_md_device(ma.out_ids, a.out_rows, a.out_scores, a.out_n, out_cap, d.metric, d.id_base, k5, nq,
                                       sc->cand.as<uint32_t>(), sc->hn_labels.as<uint32_t>(), sc->cand_cnt.as<uint32_t>(), s)))
            return rc;
        if ((rc = rerank_f32_device(ix->d_raw, ix->raw_pitch_elems, ix->d_raw_mags, ix->size, d.dim, sc->qraw.as<float>(),
                                    ix->raw_pitch_elems, sc->qraw_mags.as<float>(), nq, sc->cand.as<uint32_t>(),
                                    sc->cand_cnt.as<uint32_t>(), k5, p->k, d.id_base, d_ids, d_scores, d_counts, s,
                                    sc->hn_labels.as<uint32_t>(), sc->cur_keys)))
            return rc;
    } else {
        // one warp per query (hnsw_warp.cu); CDB_HNSW_F_CTA selects the round-1 CTA-per-query kernel for A/B measurements
        a.flags = g_hnsw_flags.load();
        a.prof = ix->hn_prof_on ? ix->hn_prof.as<unsigned long long>() : nullptr;
        if ((rc = (a.flags & CDB_HNSW_F_CTA) ? hnsw_search_device(a, s) : hnsw_search_warp_device(a, s))) return rc;
        CDB_CUDA_TRY(cudaEventRecord(ix->ring1[slot], s));
        if ((rc = hnsw_dedup_device(a.out_rows, a.out_scores, a.out_n, out_cap, d.metric, ix->graph.root_row, d.id_base, k5, nq,
                                    sc->cand.as<uint32_t>(), sc->cand_cnt.as<uint32_t>(), s)))
            return rc;
        if ((rc = rerank_f32_device(ix->d_raw, ix->raw_pitch_elems, ix->d_raw_mags, ix->size, d.dim, sc->qraw.as<float>(),
                                    ix->raw_pitch_elems, sc->qraw_mags.as<float>(), nq, sc->cand.as<uint32_t>(),
                                    sc->cand_cnt.as<uint32_t>(), k5, p->k, d.id_base, d_ids, d_scores, d_counts, s, nullptr,
                                    sc->cur_keys)))
            return rc;
    }
    if (d_err) {
        err32_to_u8_kernel<<<(nq + 255) / 256, 256, 0, s>>>(a.err32, d_err, nq);
        CDB_LAUNCH_CHECK();
    }
    CDB_CUDA_TRY(cudaEventRecord(sc->ev[1], s));
    CDB_CUDA_TRY(cudaEventRecord(sc->ev[2], s));
    sc->ev_valid = true;
    return CDB_OK;
}

// rigorous bound on |approximate cosine - reference cosine| of the fp16 tensor-core prefilter
// (two fp16 roundings, fp32 tensor accumulation, f32 norms; DESIGN.md section 5)
static float prefilter_eps(uint32_t dim) { return 1.0e-3f + 8.0e-7f * (float)dim; }

static cdb_status search_chunk_locked(cdb_index *ix, Scratch *sc, const float *d_queries, uint32_t nq, const cdb_search_params *p,
                                      uint32_t *d_ids, float *d_scores, uint32_t *d_counts, uint8_t *d_err, cudaStream_t s) {
    const cdb_index_desc &d = ix->desc;
    CDB_REQUIRE(p->k >= 1 && p->k <= 1024, "k must be in 1..1024");
    if (nq == 0) return CDB_OK;
    cdb_status rc;
    if (p->mode == CDB_MODE_HNSW) return hnsw_search_locked(ix, sc, d_queries, nq, p, d_ids, d_scores, d_counts, d_err, s);
    if (p->mode != CDB_MODE_BRUTE_RAW && p->mode != CDB_MODE_BRUTE_CODES) {
        set_error("unknown search mode");
        return CDB_INVALID_PARAMS;
    }
    const bool raw = p->mode == CDB_MODE_BRUTE_RAW;
    if (raw) CDB_REQUIRE(ix->d_raw, "BRUTE_RAW needs raw f32 rows (F32 storage or keep_raw_f32)");
    if (raw) CDB_REQUIRE(ix->raw_missing == 0, "rows appended as codes still lack their raw f32 rows (cdb_index_set_raw_f32 / cdb_index_fill_raw_from_itoe)");
    const int st = raw ? CDB_ST_F32 : d.storage_type;
    const int metric = raw ? CDB_METRIC_COSINE : d.metric;
    if (!raw && (rc = arm_status(metric, st)) != CDB_OK) {
        set_error("metric/storage arm is an Err in the reference (StorageMismatch / unimplemented)");
        return rc;
    }
    const uint32_t pitch = raw ? ix->raw_pitch_elems * 4 : ix->row_pitch;
    // ---- wgmma prefilter + exact re-rank: identical results, far fewer exact dot products.
    // Needs k proper (non-degenerate) rows for the bound to exist, and few enough odd degenerate rows to carry them on
    // every candidate list (tensor_scan.cu).
    const bool tensor_ok = raw && ix->d_xh && !p->exact_only && nq >= 4 && ix->size >= 16384 && p->k <= 64 &&
                           ix->n_odd_rows <= TS_MAX_ODD && ix->size - ix->n_allzero_rows - ix->n_odd_rows >= p->k &&
                           tensor_scan_smem_bytes(p->k) <= 227 * 1024 && (nq + 127) / 128 <= (uint32_t)ix->sm_count;
    // search_internal: quantize the query with the index's storage type and range (hnsw/mod.rs:399-403);
    // raw mode keeps f32 and |q| = sequential fold (vector_store.rs:412)
    if ((rc = sc->q_codes.ensure((size_t)nq * pitch)) || (rc = sc->q_mags.ensure((size_t)nq * 4))) return rc;
    if (!tensor_ok) {   // (the prefilter path prepares its queries in one fused launch below)
        CDB_CUDA_TRY(cudaMemsetAsync(sc->q_codes.p, 0, (size_t)nq * pitch, s));
        if ((rc = quantize_rows_device(d_queries, nq, d.dim, st, d.range_lo, d.range_hi, sc->q_codes.as<uint8_t>(), pitch,
                                       sc->q_mags.as<float>(), nullptr, 0, s)))
            return rc;
    }
    const int slot = (int)(ix->n_search.fetch_add(1) % cdb_index::EV_RING);
    CDB_CUDA_TRY(cudaEventRecord(sc->ev[0], s));

    const uint32_t *qsel = nullptr;
    if (tensor_ok) {
        const uint32_t mt = (nq + 127) / 128;
        // candidate slots per query (<= 64 MB in total): long lists only arise for few queries, and a query whose list
        // overflows is re-done alone by the selective exact scan
        const uint32_t cap = p->prefilter_k ? p->prefilter_k : (nq <= 256 ? 32768u : (nq <= 1024 ? 16384u : 8192u));
        if ((rc = sc->qh.ensure((size_t)mt * 128 * ix->xh_pitch * 2)) || (rc = sc->gthr.ensure((size_t)mt * 128 * 64 * 4)) ||
            (rc = sc->cand.ensure((size_t)nq * cap * 4)) || (rc = sc->cand_cnt.ensure((size_t)nq * 4)) ||
            (rc = sc->progress.ensure(8192)) || (rc = sc->qsel.ensure((size_t)(nq + 1) * 4)) || (rc = sc->err32.ensure((size_t)nq * 4)))
            return rc;
        uint32_t *flags = sc->flags.as<uint32_t>();  // [0] queries of the last search that needed the exact scan, [3] searches with a fallback
        const bool has_deg = ix->n_allzero_rows + ix->n_odd_rows > 0;
        if ((rc = prep_queries_device(d_queries, nq, d.dim, sc->q_codes.as<float>(), pitch / 4, sc->q_mags.as<float>(), sc->qh.p,
                                      ix->xh_pitch, sc->gthr.as<int>(), ix->deg.as<uint32_t>(), has_deg, d.id_base,
                                      sc->cand.as<uint32_t>(), cap, sc->cand_cnt.as<uint32_t>(), sc->err32.as<uint32_t>(), d_err,
                                      sc->progress.as<uint32_t>(), s)))
            return rc;
        CDB_CUDA_TRY(cudaEventRecord(ix->ring0[slot], s));
        if ((rc = tensor_scan_device(ix->d_xh, sc->qh.p, ix->xh_pitch, ix->size, nq, d.dim, p->k, 2.0f * prefilter_eps(d.dim),
                                     d.id_base, sc->gthr.as<int>(), sc->cand.as<uint32_t>(), sc->cand_cnt.as<uint32_t>(), cap,
                                     sc->progress.as<uint32_t>(), ix->deg.as<uint32_t>(), has_deg, ix->sm_count, s, /*prepared=*/true)))
            return rc;
        CDB_CUDA_TRY(cudaEventRecord(ix->ring1[slot], s));
        if ((rc = rerank_f32_device(ix->d_raw, ix->raw_pitch_elems, ix->d_raw_mags, ix->size, d.dim, sc->q_codes.as<float>(),
                                    pitch / 4, sc->q_mags.as<float>(), nq, sc->cand.as<uint32_t>(), sc->cand_cnt.as<uint32_t>(),
                                    cap, p->k, d.id_base, d_ids, d_scores, d_counts, s, nullptr, sc->cur_keys)))
            return rc;
        if ((rc = select_fallback_device(sc->cand_cnt.as<uint32_t>(), cap, sc->q_mags.as<float>(), nq, sc->qsel.as<uint32_t>(), flags, s)))
            return rc;
        ix->stat_tensor_searches++;
        qsel = sc->qsel.as<uint32_t>();  // the exact scan below only runs (on the device's own decision) for the queries listed there
    }
    // ---- exact integer scoring on wgmma u8: u8 codes in place, sub-byte codes through the digit copy
    const uint8_t *u8_rows = !raw ? (st == CDB_ST_U8 ? ix->d_codes : ix->d_digits) : nullptr;
    const bool u8_ok = u8_rows && !p->exact_only && (metric == CDB_METRIC_COSINE || metric == CDB_METRIC_DOT_PRODUCT) &&
                       ix->size >= 16384 && p->k <= 64 && tensor_u8_smem_bytes(p->k) <= 227 * 1024 &&
                       (nq + 127) / 128 <= (uint32_t)ix->sm_count;
    if (u8_ok) {
        const uint32_t mt = (nq + 127) / 128;
        const uint32_t upitch = st == CDB_ST_U8 ? ix->row_pitch : ix->digit_pitch;
        const uint32_t cap = p->prefilter_k ? p->prefilter_k : (nq <= 256 ? 16384u : (nq <= 1024 ? 4096u : 2048u));
        if ((rc = sc->qh.ensure((size_t)mt * 128 * upitch)) || (rc = sc->gthr.ensure((size_t)mt * 128 * 64 * 4)) ||
            (rc = sc->cand.ensure((size_t)nq * cap * 8)) || (rc = sc->cand_cnt.ensure((size_t)nq * 4)) ||
            (rc = sc->progress.ensure(8192)) || (rc = sc->err32.ensure((size_t)nq * 4)))
            return rc;
        if ((rc = sc->qsel.ensure((size_t)(nq + 1) * 4))) return rc;
        uint32_t *flags = sc->flags.as<uint32_t>();
        CDB_CUDA_TRY(cudaMemsetAsync(sc->err32.p, 0, (size_t)nq * 4, s));
        CDB_CUDA_TRY(cudaMemsetAsync(sc->qh.p, 0, (size_t)mt * 128 * upitch, s));
        if (st == CDB_ST_U8)
            CDB_CUDA_TRY(cudaMemcpyAsync(sc->qh.p, sc->q_codes.p, (size_t)nq * upitch, cudaMemcpyDeviceToDevice, s));
        else if ((rc = unpack_digits_device(sc->q_codes.as<uint8_t>(), pitch, nq, d.dim, st, sc->qh.as<uint8_t>(), upitch, s)))
            return rc;
        CDB_CUDA_TRY(cudaEventRecord(ix->ring0[slot], s));
        if ((rc = tensor_u8_scan_device(u8_rows, sc->qh.as<uint8_t>(), upitch, ix->size, nq, d.dim, p->k, metric, ix->d_mags,
                                        sc->q_mags.as<float>(), d.id_base, sc->gthr.as<int>(), sc->cand.as<uint64_t>(),
                                        sc->cand_cnt.as<uint32_t>(), cap, sc->err32.as<uint32_t>(), sc->progress.as<uint32_t>(),
                                        d_ids, d_scores, d_counts, ix->sm_count, s, sc->cur_keys)))
            return rc;
        CDB_CUDA_TRY(cudaEventRecord(ix->ring1[slot], s));
        if ((rc = select_fallback_device(sc->cand_cnt.as<uint32_t>(), cap, nullptr, nq, sc->qsel.as<uint32_t>(), flags, s))) return rc;
        if (d_err) {
            err32_to_u8_kernel<<<(nq + 255) / 256, 256, 0, s>>>(sc->err32.as<uint32_t>(), d_err, nq);
            CDB_LAUNCH_CHECK();
        }
        ix->stat_tensor_searches++;
        qsel = sc->qsel.as<uint32_t>();
    }
    {
        // exact scan: unconditional when no tensor-core path applies, otherwise a device-side conditional fallback
        // (its kernels return immediately unless qsel lists queries the tensor-core path could not answer) -- no host sync
        const bool fast = qsel != nullptr;
        if (!fast) CDB_CUDA_TRY(cudaEventRecord(ix->ring0[slot], s));
        if ((rc = exact_scan_locked(ix, sc, raw, st, metric, pitch, nq, p->k, d_ids, d_scores, d_counts, d_err, s, qsel))) return rc;
        if (!fast) CDB_CUDA_TRY(cudaEventRecord(ix->ring1[slot], s));
    }
    CDB_CUDA_TRY(cudaEventRecord(sc->ev[1], s));
    CDB_CUDA_TRY(cudaEventRecord(sc->ev[2], s));
    sc->ev_valid = true;
    return CDB_OK;
}

// Batches are processed in chunks of <= 2048 queries (16 query tiles of 128): 132 SMs then split into 8 whole
// CTA groups (128 CTAs) for the tensor-core kernels, and per-chunk scratch stays bounded.
static cdb_status search_device_locked(cdb_index *ix, Scratch *sc, const float *d_queries, uint32_t nq, const cdb_search_params *p,
                                       uint32_t *d_ids, float *d_scores, uint32_t *d_counts, uint8_t *d_err, cudaStream_t s) {
    // the handle's scratch arena is reused by every search: a search enqueued on a different stream than the previous
    // one must wait for it (stream-ordered hand-over, no host sync)
    if (sc->ev_valid && sc->last_stream != s) CDB_CUDA_TRY(cudaStreamWaitEvent(s, sc->ev[2], 0));
    sc->last_stream = s;
    const uint32_t CH = 2048;
    for (uint32_t off = 0; off < nq; off += CH) {
        const uint32_t m = nq - off < CH ? nq - off : CH;
        sc->cur_keys = sc->keys_out ? sc->keys_out + (size_t)off * p->k : nullptr;
        cdb_status rc = search_chunk_locked(ix, sc, d_queries + (size_t)off * ix->desc.dim, m, p, d_ids + (size_t)off * p->k,
                                            d_scores + (size_t)off * p->k, d_counts + off, d_err ? d_err + off : nullptr, s);
        if (rc) return rc;
    }
    return CDB_OK;
}

}  // extern "C"
namespace cdb {
// shard_group.cu: search one shard with device buffers on `s`; d_keys ([nq][k], may be null) receives the packed keys
cdb_status index_search_device_keys(cdb_index *ix, const float *d_queries, uint32_t nq, const cdb_search_params *p, uint32_t *d_ids,
                                    float *d_scores, uint32_t *d_counts, uint8_t *d_err, uint64_t *d_keys, cudaStream_t s) {
    std::shared_lock<std::shared_mutex> lock(ix->rw);
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    CDB_REQUIRE(p->k >= 1 && p->k <= 1024, "k must be in 1..1024");
    Lease l;
    cdb_status rc = lease_scratch(ix, l);
    if (rc) return rc;
    Scratch *sc = l.sc;
    sc->keys_out = d_keys;
    rc = search_device_locked(ix, sc, d_queries, nq, p, d_ids, d_scores, d_counts, d_err, s ? s : sc->stream);
    sc->keys_out = sc->cur_keys = nullptr;
    return rc;
}
int index_device(const cdb_index *ix) { return ix->desc.device; }
uint32_t index_dim(const cdb_index *ix) { return ix->desc.dim; }
int index_result_metric(const cdb_index *ix, int mode) { return mode == CDB_MODE_BRUTE_CODES ? ix->desc.metric : CDB_METRIC_COSINE; }
}  // namespace cdb
extern "C" {

cdb_status cdb_search_batch_device(cdb_index *ix, const float *d_queries, uint32_t nq, const cdb_search_params *p,
                                   uint32_t *d_ids, float *d_scores, uint32_t *d_counts, uint8_t *d_err, void *stream) {
    CDB_REQUIRE(ix && p && (d_queries || !nq) && (d_ids || !nq) && (d_scores || !nq), "null argument");
    std::shared_lock<std::shared_mutex> lock(ix->rw);
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    Lease l;
    cdb_status rc = lease_scratch(ix, l);
    if (rc) return rc;
    Scratch *sc = l.sc;
    cudaStream_t s = stream ? (cudaStream_t)stream : sc->stream;
    if (!d_counts) {
        if ((rc = sc->io_counts.ensure((size_t)nq * 4))) return rc;
        d_counts = sc->io_counts.as<uint32_t>();
    }
    // asynchronous: the set goes back to the pool when this call returns; the next search that leases it orders itself
    // behind this one on the device (event hand-over in search_device_locked)
    return search_device_locked(ix, sc, d_queries, nq, p, d_ids, d_scores, d_counts, d_err, s);
}

cdb_status cdb_search_batch(cdb_index *ix, const float *queries, uint32_t nq, const cdb_search_params *p, uint32_t *out_ids,
                            float *out_scores, uint32_t *out_counts, uint8_t *err_flags) {
    CDB_REQUIRE(ix && p && (queries || !nq) && (out_ids || !nq) && (out_scores || !nq), "null argument");
    std::shared_lock<std::shared_mutex> lock(ix->rw);
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    if (!nq) return CDB_OK;
    CDB_REQUIRE(p->k >= 1 && p->k <= 1024, "k must be in 1..1024");
    Lease l;
    cdb_status rc = lease_scratch(ix, l);
    if (rc) return rc;
    Scratch *sc = l.sc;
    cudaStream_t s = sc->stream;
    const size_t nk = (size_t)nq * p->k;
    if ((rc = sc->io_q.ensure((size_t)nq * ix->desc.dim * 4)) || (rc = sc->io_ids.ensure(nk * 4)) ||
        (rc = sc->io_scores.ensure(nk * 4)) || (rc = sc->io_counts.ensure((size_t)nq * 4)) || (rc = sc->io_err.ensure(nq)))
        return rc;
    CDB_CUDA_TRY(cudaMemcpyAsync(sc->io_q.p, queries, (size_t)nq * ix->desc.dim * 4, cudaMemcpyHostToDevice, s));
    rc = search_device_locked(ix, sc, sc->io_q.as<float>(), nq, p, sc->io_ids.as<uint32_t>(), sc->io_scores.as<float>(),
                              sc->io_counts.as<uint32_t>(), sc->io_err.as<uint8_t>(), s);
    if (rc) return rc;
    CDB_CUDA_TRY(cudaMemcpyAsync(out_ids, sc->io_ids.p, nk * 4, cudaMemcpyDeviceToHost, s));
    CDB_CUDA_TRY(cudaMemcpyAsync(out_scores, sc->io_scores.p, nk * 4, cudaMemcpyDeviceToHost, s));
    if (out_counts) CDB_CUDA_TRY(cudaMemcpyAsync(out_counts, sc->io_counts.p, (size_t)nq * 4, cudaMemcpyDeviceToHost, s));
    if (err_flags) CDB_CUDA_TRY(cudaMemcpyAsync(err_flags, sc->io_err.p, nq, cudaMemcpyDeviceToHost, s));
    CDB_CUDA_TRY(cudaStreamSynchronize(s));
    return CDB_OK;
}

cdb_status cdb_search_batch_filtered(cdb_index *ix, const float *queries, uint32_t nq, const cdb_search_params *p,
                                     const uint32_t *filter_offsets, const int8_t *filter_dims, const uint8_t *has_filter,
                                     uint32_t *out_ids, float *out_scores, uint32_t *out_counts, uint8_t *err_flags) {
    CDB_REQUIRE(ix && p && (queries || !nq) && (out_ids || !nq) && (out_scores || !nq), "null argument");
    CDB_REQUIRE(p->mode == CDB_MODE_HNSW, "metadata filters apply to CDB_MODE_HNSW");
    CDB_REQUIRE(!has_filter || filter_offsets, "has_filter needs filter_offsets");
    std::shared_lock<std::shared_mutex> lock(ix->rw);
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    if (!nq) return CDB_OK;
    CDB_REQUIRE(p->k >= 1 && p->k <= 1024, "k must be in 1..1024");
    CDB_REQUIRE(ix->has_md, "metadata filters need cdb_index_set_graph_metadata");
    Lease l;
    cdb_status rc = lease_scratch(ix, l);
    if (rc) return rc;
    Scratch *sc = l.sc;
    cudaStream_t s = sc->stream;
    const size_t nk = (size_t)nq * p->k;
    if ((rc = sc->io_q.ensure((size_t)nq * ix->desc.dim * 4)) || (rc = sc->io_ids.ensure(nk * 4)) ||
        (rc = sc->io_scores.ensure(nk * 4)) || (rc = sc->io_counts.ensure((size_t)nq * 4)) || (rc = sc->io_err.ensure(nq)))
        return rc;
    const uint32_t *d_off = nullptr;
    const int8_t *d_dims = nullptr;
    const uint8_t *d_has = nullptr;
    if (has_filter) {
        uint32_t total = 0;
        for (uint32_t q = 0; q < nq; ++q) {
            CDB_REQUIRE(filter_offsets[q] <= filter_offsets[q + 1], "filter_offsets must be non-decreasing");
            CDB_REQUIRE(!has_filter[q] || filter_offsets[q + 1] - filter_offsets[q] <= 4096, "too many filters for one query");
        }
        total = filter_offsets[nq];
        CDB_REQUIRE(filter_dims || !total, "null filter_dims");
        if ((rc = sc->flt_off.ensure((size_t)(nq + 1) * 4)) || (rc = sc->flt_has.ensure(nq)) ||
            (rc = sc->flt_dims.ensure((size_t)total * ix->md_dims + 1)))
            return rc;
        CDB_CUDA_TRY(cudaMemcpyAsync(sc->flt_off.p, filter_offsets, (size_t)(nq + 1) * 4, cudaMemcpyHostToDevice, s));
        CDB_CUDA_TRY(cudaMemcpyAsync(sc->flt_has.p, has_filter, nq, cudaMemcpyHostToDevice, s));
        if (total) CDB_CUDA_TRY(cudaMemcpyAsync(sc->flt_dims.p, filter_dims, (size_t)total * ix->md_dims, cudaMemcpyHostToDevice, s));
        d_off = sc->flt_off.as<uint32_t>(); d_dims = sc->flt_dims.as<int8_t>(); d_has = sc->flt_has.as<uint8_t>();
    }
    CDB_CUDA_TRY(cudaMemcpyAsync(sc->io_q.p, queries, (size_t)nq * ix->desc.dim * 4, cudaMemcpyHostToDevice, s));
    if (sc->ev_valid && sc->last_stream != s) CDB_CUDA_TRY(cudaStreamWaitEvent(s, sc->ev[2], 0));
    sc->last_stream = s;
    const uint32_t CH = 2048;
    for (uint32_t q0 = 0; q0 < nq; q0 += CH) {
        const uint32_t m = std::min(CH, nq - q0);
        rc = hnsw_search_locked(ix, sc, sc->io_q.as<float>() + (size_t)q0 * ix->desc.dim, m, p, sc->io_ids.as<uint32_t>() + (size_t)q0 * p->k,
                                sc->io_scores.as<float>() + (size_t)q0 * p->k, sc->io_counts.as<uint32_t>() + q0,
                                sc->io_err.as<uint8_t>() + q0, s, d_off ? d_off + q0 : nullptr, d_dims, d_has ? d_has + q0 : nullptr);
        if (rc) return rc;
    }
    CDB_CUDA_TRY(cudaMemcpyAsync(out_ids, sc->io_ids.p, nk * 4, cudaMemcpyDeviceToHost, s));
    CDB_CUDA_TRY(cudaMemcpyAsync(out_scores, sc->io_scores.p, nk * 4, cudaMemcpyDeviceToHost, s));
    if (out_counts) CDB_CUDA_TRY(cudaMemcpyAsync(out_counts, sc->io_counts.p, (size_t)nq * 4, cudaMemcpyDeviceToHost, s));
    if (err_flags) CDB_CUDA_TRY(cudaMemcpyAsync(err_flags, sc->io_err.p, nq, cudaMemcpyDeviceToHost, s));
    CDB_CUDA_TRY(cudaStreamSynchronize(s));
    return CDB_OK;
}

// ------------------------------------------------------------------ S2 / S3

cdb_status cdb_score_ids(cdb_index *ix, const float *query, const uint32_t *ids, uint32_t n, float *out, int32_t *out_status) {
    CDB_REQUIRE(ix && query && (ids || !n) && (out || !n) && (out_status || !n), "null argument");
    std::shared_lock<std::shared_mutex> lock(ix->rw);
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    if (!n) return CDB_OK;
    const cdb_index_desc &d = ix->desc;
    Lease l;
    cdb_status rc = lease_scratch(ix, l);
    if (rc) return rc;
    Scratch *sc = l.sc;
    cudaStream_t s = sc->stream;
    // the set's buffers may still be read by an asynchronous search enqueued on a caller stream: order behind it
    if (sc->ev_valid && sc->last_stream != s) CDB_CUDA_TRY(cudaStreamWaitEvent(s, sc->ev[2], 0));
    sc->last_stream = s;
    if ((rc = sc->io_q.ensure((size_t)d.dim * 4)) || (rc = sc->q_codes.ensure(ix->row_pitch)) || (rc = sc->q_mags.ensure(4)) ||
        (rc = sc->io_ids.ensure((size_t)n * 4)) || (rc = sc->io_scores.ensure((size_t)n * 4)) || (rc = sc->misc.ensure((size_t)n * 4)))
        return rc;
    CDB_CUDA_TRY(cudaMemcpyAsync(sc->io_q.p, query, (size_t)d.dim * 4, cudaMemcpyHostToDevice, s));
    CDB_CUDA_TRY(cudaMemcpyAsync(sc->io_ids.p, ids, (size_t)n * 4, cudaMemcpyHostToDevice, s));
    CDB_CUDA_TRY(cudaMemsetAsync(sc->q_codes.p, 0, ix->row_pitch, s));
    if ((rc = quantize_rows_device(sc->io_q.as<float>(), 1, d.dim, d.storage_type, d.range_lo, d.range_hi,
                                   sc->q_codes.as<uint8_t>(), ix->row_pitch, sc->q_mags.as<float>(), nullptr, 0, s)))
        return rc;
    float qmag = 0.0f;
    CDB_CUDA_TRY(cudaMemcpyAsync(&qmag, sc->q_mags.p, 4, cudaMemcpyDeviceToHost, s));
    CDB_CUDA_TRY(cudaStreamSynchronize(s));
    if ((rc = score_ids_device(d.metric, d.storage_type, d.dim, sc->q_codes.as<uint8_t>(), qmag, ix->d_codes, ix->d_mags,
                               ix->row_pitch, ix->size, sc->io_ids.as<uint32_t>(), n, sc->io_scores.as<float>(),
                               sc->misc.as<int32_t>(), s)))
        return rc;
    CDB_CUDA_TRY(cudaMemcpyAsync(out, sc->io_scores.p, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
    CDB_CUDA_TRY(cudaMemcpyAsync(out_status, sc->misc.p, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
    CDB_CUDA_TRY(cudaStreamSynchronize(s));
    return CDB_OK;
}

cdb_status cdb_rerank_f32(cdb_index *ix, const float *query, const uint32_t *cand_ids, uint32_t n, uint32_t k,
                          uint32_t *out_ids, float *out_scores, uint32_t *out_count) {
    CDB_REQUIRE(ix && query && (cand_ids || !n) && out_ids && out_scores && k >= 1, "bad argument");
    std::shared_lock<std::shared_mutex> lock(ix->rw);
    CDB_REQUIRE(ix->d_raw, "re-rank needs raw f32 rows (F32 storage or keep_raw_f32)");
    CDB_REQUIRE(ix->raw_missing == 0, "rows appended as codes still lack their raw f32 rows (cdb_index_set_raw_f32 / cdb_index_fill_raw_from_itoe)");
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    const cdb_index_desc &d = ix->desc;
    Lease l;
    cdb_status rc = lease_scratch(ix, l);
    if (rc) return rc;
    Scratch *sc = l.sc;
    cudaStream_t s = sc->stream;
    if (sc->ev_valid && sc->last_stream != s) CDB_CUDA_TRY(cudaStreamWaitEvent(s, sc->ev[2], 0));
    sc->last_stream = s;
    const uint32_t qpitch = ix->raw_pitch_elems;
    if ((rc = sc->io_q.ensure((size_t)d.dim * 4)) || (rc = sc->q_codes.ensure((size_t)qpitch * 4)) || (rc = sc->q_mags.ensure(4)) ||
        (rc = sc->misc.ensure((size_t)(n ? n : 1) * 4)) || (rc = sc->io_ids.ensure((size_t)k * 4)) ||
        (rc = sc->io_scores.ensure((size_t)k * 4)) || (rc = sc->io_counts.ensure(4)))
        return rc;
    CDB_CUDA_TRY(cudaMemcpyAsync(sc->io_q.p, query, (size_t)d.dim * 4, cudaMemcpyHostToDevice, s));
    if (n) CDB_CUDA_TRY(cudaMemcpyAsync(sc->misc.p, cand_ids, (size_t)n * 4, cudaMemcpyHostToDevice, s));
    CDB_CUDA_TRY(cudaMemsetAsync(sc->q_codes.p, 0, (size_t)qpitch * 4, s));
    if ((rc = quantize_rows_device(sc->io_q.as<float>(), 1, d.dim, CDB_ST_F32, 0.f, 0.f, sc->q_codes.as<uint8_t>(), qpitch * 4,
                                   sc->q_mags.as<float>(), nullptr, 0, s)))
        return rc;
    if ((rc = rerank_f32_device(ix->d_raw, ix->raw_pitch_elems, ix->d_raw_mags, ix->size, d.dim, sc->q_codes.as<float>(), qpitch,
                                sc->q_mags.as<float>(), 1, sc->misc.as<uint32_t>(), nullptr, n, k, d.id_base, sc->io_ids.as<uint32_t>(),
                                sc->io_scores.as<float>(), sc->io_counts.as<uint32_t>(), s)))
        return rc;
    CDB_CUDA_TRY(cudaMemcpyAsync(out_ids, sc->io_ids.p, (size_t)k * 4, cudaMemcpyDeviceToHost, s));
    CDB_CUDA_TRY(cudaMemcpyAsync(out_scores, sc->io_scores.p, (size_t)k * 4, cudaMemcpyDeviceToHost, s));
    if (out_count) CDB_CUDA_TRY(cudaMemcpyAsync(out_count, sc->io_counts.p, 4, cudaMemcpyDeviceToHost, s));
    CDB_CUDA_TRY(cudaStreamSynchronize(s));
    return CDB_OK;
}

// ------------------------------------------------------------------ multi-GPU merge

cdb_status cdb_merge_topk_device(int32_t device, int32_t metric, const uint32_t *d_ids, const float *d_scores,
                                 uint32_t n_shards, uint32_t nq, uint32_t k, uint32_t *d_out_ids, float *d_out_scores,
                                 void *stream) {
    CDB_REQUIRE(d_ids && d_scores && d_out_ids && d_out_scores && n_shards >= 1 && k >= 1, "bad argument");
    CDB_CUDA_TRY(cudaSetDevice(device));
    cudaStream_t s = (cudaStream_t)stream;
    uint64_t *keys = nullptr;
    CDB_CUDA_TRY(cudaMallocAsync(&keys, (size_t)n_shards * nq * k * 8, s));
    cdb_status rc = pack_keys_device(metric, d_ids, d_scores, n_shards, nq, k, keys, s);
    if (!rc) rc = merge_partials_device(metric, keys, nq, n_shards, k, d_out_ids, d_out_scores, nullptr, s);
    cudaFreeAsync(keys, s);
    return rc;
}

cdb_status cdb_index_last_kernel_ms(const cdb_index *ix, float *scan_ms, float *total_ms) {
    CDB_REQUIRE(ix, "null index");
    if (scan_ms) *scan_ms = 0.f;
    if (total_ms) *total_ms = 0.f;
    const Scratch *sc = ix->last;           // set of the most recently finished search
    if (!sc || !sc->ev_valid) return CDB_OK;
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    CDB_CUDA_TRY(cudaEventSynchronize(sc->ev[2]));
    if (scan_ms) CDB_CUDA_TRY(cudaEventElapsedTime(scan_ms, sc->ev[0], sc->ev[1]));
    if (total_ms) CDB_CUDA_TRY(cudaEventElapsedTime(total_ms, sc->ev[0], sc->ev[2]));
    return CDB_OK;
}


cdb_status cdb_index_set_graph(cdb_index *ix, const cdb_graph_desc *gd) {
    CDB_REQUIRE(ix && gd && gd->level_counts && gd->node_row && gd->adjacency && gd->child, "null argument");
    CDB_REQUIRE(gd->num_levels <= 31, "too many levels");
    CDB_REQUIRE(gd->neighbors_count >= 1 && gd->neighbors_count <= 64 && gd->level0_neighbors_count >= 1 &&
                    gd->level0_neighbors_count <= 64, "neighbour counts must be in 1..64");
    std::unique_lock<std::shared_mutex> lock(ix->rw);
    CDB_REQUIRE(gd->level_counts[0] >= 1, "level 0 is empty");
    CDB_REQUIRE(gd->root_row < ix->size, "root_row out of range");
    CDB_REQUIRE(gd->entry < gd->level_counts[gd->num_levels], "entry out of range");
    for (uint32_t L = 0; L <= gd->num_levels; ++L) {   // every index the kernels will follow
        const uint32_t cnt = gd->level_counts[L], nb = L == 0 ? gd->level0_neighbors_count : gd->neighbors_count;
        CDB_REQUIRE(gd->node_row[L] && gd->adjacency[L] && (L == 0 || gd->child[L]), "null level array");
        for (uint32_t i = 0; i < cnt; ++i) {
            CDB_REQUIRE(gd->node_row[L][i] < ix->size, "node_row entry out of range");
            if (L > 0) CDB_REQUIRE(gd->child[L][i] < gd->level_counts[L - 1], "child entry out of range");
        }
        for (size_t t = 0; t < (size_t)cnt * nb; ++t)
            CDB_REQUIRE(gd->adjacency[L][t] == CDB_INVALID_ID || gd->adjacency[L][t] < cnt, "adjacency entry out of range");
    }
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    for (void *g : ix->graph_allocs) cudaFree(g);
    ix->graph_allocs.clear();
    for (void *g : ix->md_allocs) cudaFree(g);
    ix->md_allocs.clear();
    ix->has_md = false;
    ix->has_graph = false;
    const uint32_t L1 = gd->num_levels + 1;
    std::vector<const uint32_t *> nr(L1), ad(L1), ch(L1);
    auto upload = [&](const uint32_t *src, size_t n, const uint32_t **dst) -> cdb_status {
        void *p = nullptr;
        CDB_CUDA_TRY(cudaMalloc(&p, (n ? n : 1) * 4));
        ix->graph_allocs.push_back(p);
        if (n) CDB_CUDA_TRY(cudaMemcpy(p, src, n * 4, cudaMemcpyHostToDevice));
        *dst = (const uint32_t *)p;
        return CDB_OK;
    };
    cdb_status rc;
    for (uint32_t L = 0; L < L1; ++L) {
        const uint32_t cnt = gd->level_counts[L];
        const uint32_t nb = L == 0 ? gd->level0_neighbors_count : gd->neighbors_count;
        if ((rc = upload(gd->node_row[L], cnt, &nr[L])) || (rc = upload(gd->adjacency[L], (size_t)cnt * nb, &ad[L]))) return rc;
        if (L == 0) ch[L] = nullptr;
        else if ((rc = upload(gd->child[L], cnt, &ch[L]))) return rc;
    }
    const uint32_t *tbl[3] = {nullptr, nullptr, nullptr};
    const std::vector<const uint32_t *> *src[3] = {&nr, &ad, &ch};
    for (int t = 0; t < 3; ++t) {
        void *p = nullptr;
        CDB_CUDA_TRY(cudaMalloc(&p, L1 * sizeof(void *)));
        ix->graph_allocs.push_back(p);
        CDB_CUDA_TRY(cudaMemcpy(p, src[t]->data(), L1 * sizeof(void *), cudaMemcpyHostToDevice));
        tbl[t] = (const uint32_t *)p;
    }
    ix->g_nr = nr; ix->g_ad = ad; ix->g_ch = ch;
    ix->g_cnt.assign(gd->level_counts, gd->level_counts + L1);
    ix->graph.num_levels = gd->num_levels;
    ix->graph.nbrs = gd->neighbors_count;
    ix->graph.nbrs0 = gd->level0_neighbors_count;
    ix->graph.entry = gd->entry;
    ix->graph.root_row = gd->root_row;
    ix->graph.identity_mask = 0;
    for (uint32_t L = 0; L < L1; ++L) {   // levels whose node i is row i: the kernels skip the node_row lookup
        bool ident = true;
        for (uint32_t i = 0; i < gd->level_counts[L] && ident; ++i) ident = gd->node_row[L][i] == i;
        if (ident) ix->graph.identity_mask |= 1u << L;
    }
    ix->graph.node_row = reinterpret_cast<const uint32_t *const *>(tbl[0]);
    ix->graph.adj = reinterpret_cast<const uint32_t *const *>(tbl[1]);
    ix->graph.child = reinterpret_cast<const uint32_t *const *>(tbl[2]);
    ix->has_graph = true;
    return CDB_OK;
}

cdb_status cdb_index_set_graph_metadata(cdb_index *ix, const cdb_graph_metadata *md) {
    CDB_REQUIRE(ix && md && md->node_id && md->node_md, "null argument");
    CDB_REQUIRE(md->md_dims >= 1 && md->md_dims <= 4096, "md_dims must be in 1..4096");
    CDB_REQUIRE((md->md_bits && md->md_mags) || !md->n_md, "null metadata table");
    std::unique_lock<std::shared_mutex> lock(ix->rw);
    CDB_REQUIRE(ix->has_graph, "cdb_index_set_graph_metadata needs cdb_index_set_graph first");
    const uint32_t L1 = ix->graph.num_levels + 1;
    CDB_REQUIRE(md->pseudo_entry < ix->g_cnt[L1 - 1], "pseudo_entry out of range");
    for (uint32_t L = 0; L < L1; ++L) {
        CDB_REQUIRE(md->node_id[L] && md->node_md[L], "null level array");
        for (uint32_t i = 0; i < ix->g_cnt[L]; ++i)
            CDB_REQUIRE(md->node_md[L][i] == CDB_INVALID_ID || md->node_md[L][i] < md->n_md, "node_md entry out of range");
    }
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    for (void *g : ix->md_allocs) cudaFree(g);
    ix->md_allocs.clear();
    ix->has_md = false;
    auto upload = [&](const void *src, size_t bytes, const void **dst) -> cdb_status {
        void *p = nullptr;
        CDB_CUDA_TRY(cudaMalloc(&p, bytes ? bytes : 4));
        ix->md_allocs.push_back(p);
        if (bytes) CDB_CUDA_TRY(cudaMemcpy(p, src, bytes, cudaMemcpyHostToDevice));
        *dst = p;
        return CDB_OK;
    };
    cdb_status rc;
    std::vector<const void *> ids(L1), mds(L1);
    for (uint32_t L = 0; L < L1; ++L)
        if ((rc = upload(md->node_id[L], (size_t)ix->g_cnt[L] * 4, &ids[L])) || (rc = upload(md->node_md[L], (size_t)ix->g_cnt[L] * 4, &mds[L])))
            return rc;
    const void *t_id = nullptr, *t_md = nullptr, *bits = nullptr, *mags = nullptr;
    if ((rc = upload(ids.data(), L1 * sizeof(void *), &t_id)) || (rc = upload(mds.data(), L1 * sizeof(void *), &t_md)) ||
        (rc = upload(md->md_bits, (size_t)md->n_md * md->md_dims * 4, &bits)) || (rc = upload(md->md_mags, (size_t)md->n_md * 4, &mags)))
        return rc;
    ix->md_node_id = reinterpret_cast<const uint32_t *const *>(t_id);
    ix->md_node_md = reinterpret_cast<const uint32_t *const *>(t_md);
    ix->g_id.assign(L1, nullptr); ix->g_md.assign(L1, nullptr);
    for (uint32_t L = 0; L < L1; ++L) { ix->g_id[L] = (const uint32_t *)ids[L]; ix->g_md[L] = (const uint32_t *)mds[L]; }
    ix->md_bits = reinterpret_cast<const int32_t *>(bits);
    ix->md_mags = reinterpret_cast<const float *>(mags);
    ix->md_dims = md->md_dims;
    ix->md_pseudo_entry = md->pseudo_entry;
    ix->has_md = true;
    return CDB_OK;
}

cdb_status cdb_index_build_graph(cdb_index *ix, const cdb_build_params *bp) {
    CDB_REQUIRE(ix && bp, "null argument");
    CDB_REQUIRE(bp->neighbors_count >= 1 && bp->neighbors_count <= 64 && bp->level0_neighbors_count >= 1 &&
                    bp->level0_neighbors_count <= 64, "neighbour counts must be in 1..64");
    CDB_REQUIRE(bp->ef_construction >= 1 && bp->ef_construction <= 4096 && bp->shortlist_size >= 1 && bp->shortlist_size <= 64 &&
                    bp->num_levels <= 15, "bad build parameters");
    std::unique_lock<std::shared_mutex> lock(ix->rw);
    CDB_REQUIRE(ix->size >= 1 && ix->size + 1 <= ix->desc.capacity, "build needs >= 1 row and capacity for the root row");
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    cdb_status rc;
    if ((rc = arm_status(ix->desc.metric, ix->desc.storage_type)) != CDB_OK) {
        set_error("metric/storage arm is an Err in the reference");
        return rc;
    }
    const uint32_t n = (uint32_t)ix->size;
    // root vector: uniform in [range_lo, range_hi) (vector_store.rs:57-64)
    std::vector<float> root(ix->desc.dim);
    for (uint32_t c = 0; c < ix->desc.dim; ++c)
        root[c] = ix->desc.range_lo + (synth_value(bp->seed ^ 0x526F6F74ull, c) + 1.0f) * 0.5f * (ix->desc.range_hi - ix->desc.range_lo);
    if ((rc = append_f32_locked(ix, root.data(), 1))) return rc;
    for (void *g : ix->md_allocs) cudaFree(g);
    ix->md_allocs.clear();
    ix->has_md = false;
    for (void *g : ix->graph_allocs) cudaFree(g);
    ix->graph_allocs.clear();
    ix->has_graph = false;
    HnScoreCtx sc{ix->d_codes, ix->row_pitch, ix->d_mags, ix->desc.dim, ix->desc.storage_type, ix->desc.metric, n};
    rc = hnsw_build_device(sc, n, bp->num_levels, bp->neighbors_count, bp->level0_neighbors_count, bp->ef_construction,
                           bp->shortlist_size, bp->max_batch, bp->seed, &ix->graph, &ix->graph_allocs, &ix->g_cnt, &ix->g_nr,
                           &ix->g_ad, &ix->g_ch, ix->stream);
    if (rc) return rc;
    ix->has_graph = true;
    return CDB_OK;
}

cdb_status cdb_index_build_graph_replicas(cdb_index *ix, const cdb_build_params *bp, const cdb_replica_build *rb, uint8_t *out_failed) {
    CDB_REQUIRE(ix && bp && rb, "null argument");
    CDB_REQUIRE(bp->neighbors_count >= 1 && bp->neighbors_count <= 64 && bp->level0_neighbors_count >= 1 &&
                    bp->level0_neighbors_count <= 64, "neighbour counts must be in 1..64");
    CDB_REQUIRE(bp->ef_construction >= 1 && bp->ef_construction <= 4096 && bp->shortlist_size >= 1 && bp->shortlist_size <= 64 &&
                    bp->num_levels <= 15, "bad build parameters");
    CDB_REQUIRE(rb->md_dims >= 1 && rb->md_dims <= 4096, "md_dims must be in 1..4096");
    CDB_REQUIRE((rb->row && rb->node_id && rb->base_id && rb->md_row && rb->max_level) || !rb->n_nodes, "null replica list");
    CDB_REQUIRE((rb->md_bits && rb->md_mags) || !rb->n_md, "null metadata table");
    CDB_REQUIRE(rb->pseudo_root_md < rb->n_md, "the pseudo root needs a metadata row");
    CDB_REQUIRE(rb->main_root_md == CDB_INVALID_ID || rb->main_root_md < rb->n_md, "main_root_md out of range");
    std::unique_lock<std::shared_mutex> lock(ix->rw);
    CDB_REQUIRE(ix->size + 2 <= ix->desc.capacity, "build needs capacity for the two root rows");
    const uint32_t n = (uint32_t)ix->size;
    for (uint32_t t = 0; t < rb->n_nodes; ++t) {
        CDB_REQUIRE(rb->row[t] == CDB_INVALID_ID || rb->row[t] < n, "replica row out of range");
        CDB_REQUIRE(rb->md_row[t] == CDB_INVALID_ID || rb->md_row[t] < rb->n_md, "replica md_row out of range");
    }
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    cdb_status rc;
    if ((rc = arm_status(ix->desc.metric, ix->desc.storage_type)) != CDB_OK) {
        set_error("metric/storage arm is an Err in the reference");
        return rc;
    }
    // main root: uniform in [range_lo, range_hi) (vector_store.rs:57-64); pseudo root: pseudo_node_vector = zeros (metadata/mod.rs:214-216)
    std::vector<float> roots(2 * (size_t)ix->desc.dim, 0.0f);
    for (uint32_t c = 0; c < ix->desc.dim; ++c)
        roots[c] = ix->desc.range_lo + (synth_value(bp->seed ^ 0x526F6F74ull, c) + 1.0f) * 0.5f * (ix->desc.range_hi - ix->desc.range_lo);
    if ((rc = append_f32_locked(ix, roots.data(), 2))) return rc;
    for (void *g : ix->md_allocs) cudaFree(g);
    ix->md_allocs.clear();
    ix->has_md = false;
    for (void *g : ix->graph_allocs) cudaFree(g);
    ix->graph_allocs.clear();
    ix->has_graph = false;
    std::vector<uint32_t> rows(rb->row, rb->row + rb->n_nodes);
    for (auto &r : rows) if (r == CDB_INVALID_ID) r = n + 1;   // pseudo replicas reuse the pseudo root's prop_value (vector_store.rs:661)
    ReplicaHost rh{rb->n_nodes, rows.data(), rb->node_id, rb->base_id, rb->md_row, rb->max_level, rb->md_dims, rb->n_md,
                   rb->md_bits, rb->md_mags, n, rb->main_root_md, n + 1, rb->pseudo_root_md};
    HnScoreCtx sc{ix->d_codes, ix->row_pitch, ix->d_mags, ix->desc.dim, ix->desc.storage_type, ix->desc.metric, n};
    ReplicaGraphDev mdv{};
    std::vector<uint8_t> failed;
    rc = hnsw_build_replicas_device(sc, rh, bp->num_levels, bp->neighbors_count, bp->level0_neighbors_count, bp->ef_construction,
                                    bp->shortlist_size, bp->max_batch, &ix->graph, &ix->graph_allocs, &ix->g_cnt, &ix->g_nr,
                                    &ix->g_ad, &ix->g_ch, &mdv, &failed, ix->stream);
    if (rc) return rc;
    ix->has_graph = true;
    ix->md_node_id = mdv.node_id; ix->md_node_md = mdv.node_md;
    ix->g_id = mdv.h_node_id; ix->g_md = mdv.h_node_md;
    ix->md_bits = mdv.md_bits; ix->md_mags = mdv.md_mags;
    ix->md_dims = mdv.md_dims; ix->md_pseudo_entry = mdv.pseudo_entry;
    ix->has_md = true;   // the arrays live in graph_allocs
    if (out_failed) std::copy(failed.begin(), failed.end(), out_failed);
    return CDB_OK;
}

cdb_status cdb_index_read_graph_metadata_level(const cdb_index *ix, uint32_t level, uint32_t *node_id, uint32_t *node_md) {
    CDB_REQUIRE(ix && ix->has_graph && ix->has_md && level <= ix->graph.num_levels, "no graph metadata / bad level");
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    const uint32_t cnt = ix->g_cnt[level];
    if (node_id) CDB_CUDA_TRY(cudaMemcpy(node_id, ix->g_id[level], (size_t)cnt * 4, cudaMemcpyDeviceToHost));
    if (node_md) CDB_CUDA_TRY(cudaMemcpy(node_md, ix->g_md[level], (size_t)cnt * 4, cudaMemcpyDeviceToHost));
    return CDB_OK;
}

cdb_status cdb_index_graph_info(const cdb_index *ix, uint32_t *info5, uint32_t *level_counts) {
    CDB_REQUIRE(ix && info5, "null argument");
    CDB_REQUIRE(ix->has_graph, "no graph");
    info5[0] = ix->graph.num_levels; info5[1] = ix->graph.nbrs; info5[2] = ix->graph.nbrs0; info5[3] = ix->graph.entry; info5[4] = ix->graph.root_row;
    if (level_counts) for (size_t i = 0; i < ix->g_cnt.size(); ++i) level_counts[i] = ix->g_cnt[i];
    return CDB_OK;
}

cdb_status cdb_index_read_graph_level(const cdb_index *ix, uint32_t level, uint32_t *node_row, uint32_t *adjacency, uint32_t *child) {
    CDB_REQUIRE(ix && ix->has_graph && level <= ix->graph.num_levels, "no graph / bad level");
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    const uint32_t cnt = ix->g_cnt[level], nb = level == 0 ? ix->graph.nbrs0 : ix->graph.nbrs;
    if (node_row) CDB_CUDA_TRY(cudaMemcpy(node_row, ix->g_nr[level], (size_t)cnt * 4, cudaMemcpyDeviceToHost));
    if (adjacency) CDB_CUDA_TRY(cudaMemcpy(adjacency, ix->g_ad[level], (size_t)cnt * nb * 4, cudaMemcpyDeviceToHost));
    if (child && level > 0) CDB_CUDA_TRY(cudaMemcpy(child, ix->g_ch[level], (size_t)cnt * 4, cudaMemcpyDeviceToHost));
    return CDB_OK;
}

cdb_status cdb_index_hnsw_counters(const cdb_index *ix, uint64_t *out2) {
    CDB_REQUIRE(ix && out2, "null argument");
    out2[0] = out2[1] = 0;
    if (!ix->hn_counters.p) return CDB_OK;
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    CDB_CUDA_TRY(cudaMemcpy(out2, ix->hn_counters.p, 16, cudaMemcpyDeviceToHost));
    return CDB_OK;
}

cdb_status cdb_debug_set_hnsw_flags(uint32_t flags) {
    g_hnsw_flags.store(flags == 0xFFFFFFFFu ? CDB_HNSW_F_DEFAULT : flags);
    return CDB_OK;
}

cdb_status cdb_index_hnsw_profile(cdb_index *ix, int32_t enable, uint64_t *out) {
    CDB_REQUIRE(ix, "null index");
    std::unique_lock<std::shared_mutex> lock(ix->rw);
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    CDB_CUDA_TRY(cudaDeviceSynchronize());
    if (out) {
        for (int i = 0; i < CDB_HNSW_PROF_SLOTS; ++i) out[i] = 0;
        if (ix->hn_prof.p) CDB_CUDA_TRY(cudaMemcpy(out, ix->hn_prof.p, CDB_HNSW_PROF_SLOTS * 8, cudaMemcpyDeviceToHost));
    }
    if (enable) {
        cdb_status rc = ix->hn_prof.ensure(CDB_HNSW_PROF_SLOTS * 8);
        if (rc) return rc;
        CDB_CUDA_TRY(cudaMemset(ix->hn_prof.p, 0, CDB_HNSW_PROF_SLOTS * 8));
    }
    ix->hn_prof_on = enable != 0;
    return CDB_OK;
}

// cumulative fallback count = sum over the pool's sets; "last" values come from the most recently finished search
static cdb_status read_pool_flags(const cdb_index *ix, uint64_t *fallbacks, uint64_t *last_fallback_queries) {
    *fallbacks = 0; *last_fallback_queries = 0;
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    CDB_CUDA_TRY(cudaDeviceSynchronize());
    for (const auto &u : ix->pool) {
        uint32_t fl[4] = {0, 0, 0, 0};
        if (u->flags.p) CDB_CUDA_TRY(cudaMemcpy(fl, u->flags.p, 16, cudaMemcpyDeviceToHost));
        *fallbacks += fl[3];
        if (u.get() == ix->last) *last_fallback_queries = fl[0];
    }
    return CDB_OK;
}

cdb_status cdb_index_stats(const cdb_index *ix, uint64_t *out4) {
    CDB_REQUIRE(ix && out4, "null argument");
    uint64_t fb = 0, lq = 0;
    cdb_status rc = read_pool_flags(ix, &fb, &lq);
    if (rc) return rc;
    out4[0] = ix->stat_tensor_searches.load();
    out4[1] = fb;
    out4[2] = ix->n_allzero_rows + ix->n_odd_rows;
    out4[3] = ix->d_xh ? 1 : 0;
    return CDB_OK;
}

cdb_status cdb_index_stats_ex(const cdb_index *ix, uint64_t *out, uint32_t n) {
    CDB_REQUIRE(ix && (out || !n), "null argument");
    uint64_t fb = 0, lq = 0;
    cdb_status rc = read_pool_flags(ix, &fb, &lq);
    if (rc) return rc;
    const uint64_t v[CDB_STATS_FIELDS] = {ix->stat_tensor_searches.load(), fb, ix->n_allzero_rows, ix->n_odd_rows,
                                          ix->d_xh ? 1ull : 0ull, lq};
    for (uint32_t i = 0; i < n && i < CDB_STATS_FIELDS; ++i) out[i] = v[i];
    return CDB_OK;
}

cdb_status cdb_index_last_candidate_counts(const cdb_index *ix, uint32_t n, uint32_t *out) {
    CDB_REQUIRE(ix && out, "null argument");
    const Scratch *sc = ix->last;
    CDB_REQUIRE(sc && sc->cand_cnt.p && (size_t)n * 4 <= sc->cand_cnt.cap, "no prefilter search of that size has run");
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    CDB_CUDA_TRY(cudaMemcpy(out, sc->cand_cnt.p, (size_t)n * 4, cudaMemcpyDeviceToHost));
    return CDB_OK;
}

cdb_status cdb_index_scan_ms_history(const cdb_index *ix, uint32_t n, float *out, uint32_t *out_n) {
    CDB_REQUIRE(ix && out && out_n, "null argument");
    CDB_CUDA_TRY(cudaSetDevice(ix->desc.device));
    const uint64_t ns = ix->n_search.load();
    uint64_t have = ns < (uint64_t)cdb_index::EV_RING ? ns : (uint64_t)cdb_index::EV_RING;
    uint32_t m = n < have ? n : (uint32_t)have;
    for (uint32_t i = 0; i < m; ++i) {  // oldest of the last m first
        int slot = (int)((ns - m + i) % cdb_index::EV_RING);
        CDB_CUDA_TRY(cudaEventSynchronize(ix->ring1[slot]));
        CDB_CUDA_TRY(cudaEventElapsedTime(out + i, ix->ring0[slot], ix->ring1[slot]));
    }
    *out_n = m;
    return CDB_OK;
}

}  // extern "C"
