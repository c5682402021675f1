// Batched top-k selection and shard-merge primitives (host API).
//
// Stands in for cuvs::selection::select_k (cpp/include/cuvs/selection/select_k.hpp:70-198, whose
// arithmetic lives in RAFT: cpp/src/selection/select_k.cuh:39-51) and
// cuvs::neighbors::knn_merge_parts (cpp/src/neighbors/detail/knn_merge_parts.cuh:24-170).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace b200 {

enum idx_kind : int { IDX_NONE = 0, IDX_I64 = 1, IDX_U32 = 2, IDX_I32 = 3 };

/**
 * For each of `batch` rows of `len` floats pick the k best (smallest when select_min), sorted
 * best-first; ties go to the smaller column position.  `in_idx` (kind `in_kind`, may be null)
 * supplies the payload, otherwise the payload is the column position.  Missing entries
 * (len < k) are padded with +/-FLT_MAX and the all-ones index.
 * `in_ld` is the row pitch of in_val/in_idx in elements (>= len).
 * `batch_dev` (device, may be null): the rows to select are the first *batch_dev <= batch; `batch` sizes the launch.
 */
void select_k(cudaStream_t stream, const float* in_val, const void* in_idx, idx_kind in_kind, int64_t batch,
              int64_t len, int64_t in_ld, int k, float* out_val, void* out_idx, idx_kind out_kind, bool select_min,
              const int* batch_dev = nullptr);

/** Largest k of select_k and select_k_segments. */
constexpr int kSelectMaxK = 2048;

/**
 * select_k over rows that are segments of one array: row r is in_val[seg_off[r] .. seg_off[r] + seg_len[r]) (device arrays,
 * seg_len[r] <= max_len), and its column c is reported as position pos_base[r] + c.  Same order, tie rule and padding as
 * select_k; out_* are [batch, k].
 */
void select_k_segments(cudaStream_t stream, const float* in_val, const int64_t* seg_off, const uint32_t* seg_len,
                       const uint32_t* pos_base, int64_t batch, int64_t max_len, int k, float* out_val, uint32_t* out_pos,
                       bool select_min);

/**
 * Merge per-part top-k lists: in_* are [n_parts * n_rows, k] (part-major), out_* [n_rows, k].
 * `translations` (device int64[n_parts] or null) is added to the ids of each part.
 */
void knn_merge_parts(cudaStream_t stream, const float* in_keys, const int64_t* in_vals, float* out_keys,
                     int64_t* out_vals, int64_t n_parts, int64_t n_rows, int k, const int64_t* translations_dev,
                     bool select_min);

}  // namespace b200
