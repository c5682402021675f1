// Exact fp32 distance kernels in the oracle's pinned arithmetic (host API).
//
// Every dot product / norm / squared difference is accumulated with fmaf in ascending component
// order, exactly as oracle/oracle.c does, so results can be compared bit for bit.  These kernels
// are (a) the re-scoring stage behind every tensor-core candidate scan, (b) the certified fallback
// of brute force, (c) the filtered / exotic-shape path.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <functional>

#include <cuvs/distance/distance.h>

#include "common.hpp"  // filter_view

namespace b200 {

// Row types: the rows x of row_norms, exact_distance_tile and rescore_topk are float, __half, int8_t or uint8_t.  Narrow
// elements are widened on load, so a narrow row gives the same bits as its fp32 copy.  Queries are always fp32.

/** out[i] = sum_k x[i,k]^2 (ascending k, fmaf). */
template <typename T>
void row_norms(cudaStream_t stream, const T* x, int64_t n, int d, int64_t ld, float* out);

/** out[i] = 1 / sqrt(xn[i]) from squared norms, and 0 where xn[i] is 0: the per-row scale of the cosine metric.  A zero row
 *  scales to the zero vector, so its cosine distance to anything is 1.  out may alias xn. */
void rsqrt_rows(cudaStream_t stream, const float* xn, int64_t n, float* out);

/** x[i, :d] *= 1 / |x_i| in place (row_norms + rsqrt_rows, then one fp32 multiply per element); zero rows stay zero. */
void normalize_rows(cudaStream_t stream, float* x, int64_t n, int d, int64_t ld);

/**
 * Dense distance tile: out[i, j] = dist(q_i, x_j) for i < nq, j < n, in the metric's *selection*
 * form (squared for the L2Sqrt variants; plain dot for InnerProduct).  qn/xn: squared row norms
 * (needed for L2*Expanded and Cosine, may be null otherwise).  Filtered-out pairs get the worst
 * value.  `q_row0` is the global query index of row 0 (bitmap addressing).  self_clamp: finish_distance's self-neighbour rule
 * for expanded L2 (false: clamp at 0 only, as k-means assignment does).
 */
template <typename T>
void exact_distance_tile(cudaStream_t stream, const float* q, int64_t nq, int64_t ldq, const T* x, int64_t n,
                         int64_t ldx, int d, const float* qn, const float* xn, cuvsDistanceType metric, float* out,
                         int64_t ldo, filter_view filt, int64_t q_row0, bool self_clamp = true);

/**
 * Re-score candidates exactly and keep the best k per query.
 *   cand_pos [nq, kc]  uint32 row positions into x (0xffffffff = empty slot)
 *   src_ids            optional int64 map position -> source id (null: identity)
 * Output rows are sorted best-first, ties towards the smaller *source id*; missing entries get
 * id `pad_id` and +/-FLT_MAX.  kc <= 256 runs one warp per query; 256 < kc <= 2048 (k <= kc) one CTA per query with the
 * same arithmetic and ranking.  self_clamp: as for exact_distance_tile.
 */
template <typename T>
void rescore_topk(cudaStream_t stream, const float* q, int64_t nq, int64_t ldq, const T* x, int64_t ldx, int d,
                  const float* qn, const float* xn, cuvsDistanceType metric, const uint32_t* cand_pos, int kc,
                  const int64_t* src_ids, int k, int64_t* out_idx, float* out_dist, int64_t pad_id, bool self_clamp = true);

/** dst[dst_rows[i]] = src[src_rows[i]] for n rows of `width` elements (a null row map is the identity).  T: float, int64_t,
 *  uint32_t. */
template <typename T>
void copy_rows(cudaStream_t s, const T* src, const int64_t* src_rows, T* dst, const int64_t* dst_rows, int64_t n, int64_t width);

/** The exact fallback of a certified search: flags [nq + 1] (device) marks the queries a certificate rejected and flags[nq]
 *  counts them (recorded by set_last_flagged).  answer(rows, n, idx, dist) writes the k results of the n flagged rows (device,
 *  ascending) to idx / dist [n, k], which replace those rows of out_idx / out_dist [nq, k].  Synchronises the stream. */
void rerun_flagged(cudaStream_t s, const int* flags, int64_t nq, int k, int64_t* out_idx, float* out_dist,
                   const std::function<void(const int64_t* rows, int64_t n, int64_t* idx, float* dist)>& answer);

/** How a raw scan score s of the tensor-core engine maps to the metric's selection form, and the
 *  error budget of that approximation:  A = sa*s + sb*|q|^2 + sc,  eps = eps_rel * (eq*|q|^2 + ec). */
struct approx_map {
  float sa = 1.f, sb = 0.f, sc = 0.f;
  float eps_rel = 0.f, eq = 0.f, ec = 0.f;
};

/** out[q] = the smallest last entry of the sorted lists of KC (score) in row q of cs [nq, row_stride]: every row a full list
 *  dropped scores at least that much (+inf when no list is full). */
void list_floors(cudaStream_t s, const float* cs, int64_t nq, int64_t row_stride, int KC, float* out);

/**
 * The certificate of a candidate scan (DESIGN.md §3), one warp per query: flags[q] = 1 (flags[nq] counts them; this call
 * zeroes it first) unless the exact k-th distance out_dist[q, k-1] (selection form) beats the approximate score A of every
 * row outside the kc candidates (cand_score / cand_pos [nq, kc], raw engine units) by more than the budget of `amap`.  Rows
 * outside exist when the candidate list is full, or, with a floor (raw units, +inf: none), below the rows that never entered
 * a list.  exact_ints (8-bit scans): the budget is 0 while eq |q|^2 + ec < 2^23, where every value involved is an exact
 * integer.
 */
void certify_candidates(cudaStream_t s, const float* cand_score, const uint32_t* cand_pos, int kc, const float* floor,
                        const float* qn, const float* out_dist, int k, const approx_map& amap, bool select_min, bool exact_ints,
                        int64_t nq, int* flags);

/** In-place sqrt (L2Sqrt*) or sign/offset fix-ups applied after selection. */
void postprocess_distances(cudaStream_t stream, float* dist, int64_t count, cuvsDistanceType metric);

}  // namespace b200
