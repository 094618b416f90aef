// metadata.cuh -- the metadata-filter arms of the cosine metric (device side).
//   VectorData::replica_node_kind                 src/models/types.rs:223-243
//   CosineSimilarity::calculate, match (y, x)     src/distance/cosine.rs:34-102
//   cosine_similarity_mdims                       src/distance/cosine.rs:243-259
// Only the cosine metric looks at metadata (dotproduct.rs / euclidean.rs / hamming.rs score the quantized vectors alone).
#pragma once
#include "scorers.cuh"

namespace cdb {

constexpr int MD_KIND_PSEUDO = 0, MD_KIND_BASE = 1, MD_KIND_METADATA = 2;
constexpr uint32_t MD_PSEUDO_ID_LO = 0xFFFFFFFFu - 257u, MD_PSEUDO_ID_HI = 0xFFFFFFFFu - 2u;   // types.rs:232

// one side of DistanceFunction::calculate: VectorData { id, quantized_vec, metadata }
struct MdSide {
    const void *code;
    float mag;
    uint32_t pp;             // plane pitch of `code`
    bool has_id;
    uint32_t id;
    const int32_t *md_bits;  // nullptr = metadata: None
    float md_mag;
};

__device__ __forceinline__ int md_kind(const MdSide &v) {
    if (!v.md_bits || v.md_mag == 0.0f) return MD_KIND_BASE;
    if (v.has_id && v.id >= MD_PSEUDO_ID_LO && v.id <= MD_PSEUDO_ID_HI) return MD_KIND_PSEUDO;
    return MD_KIND_METADATA;
}

// dot_product_f32 (8 FMA lanes, hadd tree, scalar tail) over the i32 dims converted to f32, / (x.mag * y.mag)
__device__ inline int md_mdims_cosine(const MdSide &x, const MdSide &y, uint32_t M, float *out) {
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.0f;
    const uint32_t chunks = M / 8;
    for (uint32_t i = 0; i < chunks; ++i) {
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = __fmaf_rn((float)x.md_bits[8 * i + j], (float)y.md_bits[8 * i + j], acc[j]);
    }
    const float lo = __fadd_rn(__fadd_rn(acc[0], acc[1]), __fadd_rn(acc[2], acc[3]));
    const float hi = __fadd_rn(__fadd_rn(acc[4], acc[5]), __fadd_rn(acc[6], acc[7]));
    float r = __fadd_rn(lo, hi);
    for (uint32_t t = chunks * 8; t < M; ++t) r = __fadd_rn(r, __fmul_rn((float)x.md_bits[t], (float)y.md_bits[t]));
    const float den = __fmul_rn(x.md_mag, y.md_mag);
    if (den == 0.0f) return CDB_CALCULATION_ERROR;   // cosine.rs:230-231
    *out = canon_nan(__fdiv_rn(r, den));
    return CDB_OK;
}

// The arm of DistanceMetric::calculate(x, y) with metadata (x = query side / fvec_data, y = node side): MD_ARM_VECTOR when
// the result is the vector metric of the pair, else the arm's status (and *out).  Only the vector arms read the codes, so a
// caller with its own vector chain (hnsw_warp.cu) skips it for the constant arms.
constexpr int MD_ARM_VECTOR = -1;
__device__ inline int md_arm(int metric, uint32_t M, const MdSide &x, const MdSide &y, float *out) {
    if (metric != CDB_METRIC_COSINE) return MD_ARM_VECTOR;
    const int xk = md_kind(x), yk = md_kind(y);
    if (yk == MD_KIND_BASE && xk == MD_KIND_BASE) return MD_ARM_VECTOR;
    if (yk == MD_KIND_PSEUDO && xk == MD_KIND_PSEUDO) return md_mdims_cosine(x, y, M, out);
    if (yk == MD_KIND_PSEUDO && xk == MD_KIND_METADATA) {   // a metadata node strongly (mis)matches a pseudo node
        bool same = true;
        for (uint32_t t = 0; t < M; ++t) same &= x.md_bits[t] == y.md_bits[t];
        *out = same ? 1.0f : -1.0f;
        return CDB_OK;
    }
    if (yk == MD_KIND_METADATA && xk == MD_KIND_METADATA) {
        float mc;
        const int rc = md_mdims_cosine(x, y, M, &mc);
        if (rc != CDB_OK) return rc;
        if (mc > 0.99f) return MD_ARM_VECTOR;
        *out = -1.0f;
        return CDB_OK;
    }
    if (yk == MD_KIND_BASE && xk == MD_KIND_METADATA) { *out = 0.0f; return CDB_OK; }
    return CDB_UNREACHABLE_ARM;   // (Pseudo,Base) (Base,Pseudo) (Metadata,Pseudo) (Metadata,Base): unreachable!() in the reference
}

__device__ inline int md_pair_distance(int metric, int st, uint32_t dim, uint32_t M, const MdSide &x, const MdSide &y, float *out) {
    const int rc = md_arm(metric, M, x, y, out);
    return rc == MD_ARM_VECTOR ? pair_distance(metric, st, dim, x.code, x.mag, x.pp, y.code, y.mag, y.pp, out) : rc;
}

__device__ __forceinline__ uint32_t md_err_flag(int rc) {
    return rc == CDB_CALCULATION_ERROR ? (uint32_t)CDB_ERRFLAG_CALCULATION : rc == CDB_UNREACHABLE_ARM ? (uint32_t)CDB_ERRFLAG_UNREACHABLE : 2u;
}

}  // namespace cdb
