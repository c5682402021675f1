// IVF-PQ fine scan that streams the 8-bit PQ CODES from HBM and decodes them on the SM (host API).
//
// Replaces the reference's compute_similarity kernel family
//   cpp/src/neighbors/ivf_pq/detail/jit_lto_kernels/compute_similarity_impl.cuh:77-173 (LUT in smem, one CTA per
//   (query, probe), interleaved 16-byte code chunks: cpp/include/cuvs/neighbors/ivf_pq.hpp:235-296)
// on H100.  score(x) = sum_j lut[j][code_j(x)] is |r - y(x)|^2 with r the rotated query residual and y(x) the
// concatenation of the codebook entries the codes select; instead of one shared-memory LUT gather per (query, row, subspace)
// this kernel gathers each ROW's entries once (64 conflict-free 4-byte shared-memory reads), writes the decoded bf16 row
// into a swizzled operand tile and lets the tensor cores contract it against all the queries that probe the list.
// HBM traffic per row: pq_dim code bytes + 4 bytes of |y|^2/2 — the codes are never expanded in memory.
// See scan_pq.cu for the kernel, DESIGN.md §5 for the layout and the roofline.
#pragma once
#include "scan_tc.cuh"

#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <cstdint>

namespace b200 {

/** Bytes of one 128-row tile block of the code stream: 128 * pq_dim transposed code bytes + 128 fp32 half-norms. */
inline int64_t pq_stream_tile_bytes(int pq_dim) { return 128 * static_cast<int64_t>(pq_dim) + 512; }

/** True when the (device, index shape) combination is served by the code-streaming kernel: sm_90, 8-bit codes, one
 *  codebook per subspace, pq_len == 2 (one 32-bit bf16x2 word per code) and pq_dim 32 or 64 (rot_dim 64 / 128). */
bool pq_stream_supported(int device, int pq_dim, int pq_len, int pq_bits, bool per_subspace);

/**
 * Build the streamed form of the lists.
 *   codes    [rows_total, pq_dim]   one code per byte (lists padded to 128-row tiles)
 *   ids      [rows_total]           pad_id on padding rows
 *   pq_centers [pq_dim, 2, 256]     fp32 (rounded to bf16 here — the scan's arithmetic)
 *   stream   [rows_total / 128, pq_stream_tile_bytes]   per tile: for every 16-row group g and 32-subspace half h, lane l's
 *            16 bytes are code_{32h+l}(row 16g + i), i = 0..15 (a warp reads one row's 64 codes with conflict-free
 *            128-bit loads; the role of the reference's interleaved groups); then hn[128] fp32 = |y|^2/2 (0 for inner
 *            product, +inf on padding rows)
 *   cb_words [pq_dim/32][256][32]   bf16x2 word of (half, code, lane): bank == lane, so the gather of one row's 64 entries
 *            is conflict-free by construction
 */
void pq_stream_build(cudaStream_t s, const uint8_t* codes, const int64_t* ids, int64_t pad_id, int64_t rows_total, int pq_dim,
                     const float* pq_centers, bool ip, uint8_t* stream, uint32_t* cb_words);

/** The flat form back from the stream: codes [rows_total, pq_dim], one code per byte (getters, extend, serialize, LUT path). */
void pq_stream_to_flat(cudaStream_t s, const uint8_t* stream, int64_t rows_total, int pq_dim, uint8_t* codes);

/** False when CUVS_B200_PQ_NO_BOUND is set (not "0"): the filtering scan then takes no pruning bound, and the search runs no
 *  bound pre-pass (pq_bound_prime). */
bool pq_stream_bound_enabled();

/** Queries per work item the scan wants for an average of `pairs_per_list` probing queries per list (32, 64 or 128);
 *  KC = 0 (store epilogue) is not limited by candidate buffers. */
int pq_stream_group(double pairs_per_list, int KC, int passes);

/**
 * Scan.  Work items as in tc_scan_topk, except that an item covers `group` (= pq_stream_group) A rows instead of 128:
 * A rows = per-(query, probe) residual rows [a_rows, Kp] bf16 (q_lo: second plane for passes == 2, else null), B = the code
 * stream.  For every item and valid A row the kernel writes KC (score, position) candidates (unsorted, empty slots
 * (+inf, 0xffffffff)) at out_off + row * out_row_stride; score = hn - r.y as in tc_scan_topk; `bound` as in tc_scan_topk.
 * KC = 0 is the store epilogue (k > 64): the score of every list row goes to out_score[out_off + row * n_tiles * 128 + j],
 * j = row of the item's list (padding rows +inf); out_pos, out_row_stride and `bound` are unused, any group is accepted.
 */
void pq_stream_scan(cudaStream_t stream, int device, const __nv_bfloat16* q_hi, const __nv_bfloat16* q_lo, int64_t a_rows, int Kp,
                    const uint8_t* code_stream, const uint32_t* cb_words, int pq_dim, const tc_item* items_dev, int n_items,
                    const int* n_items_dev, int group, int KC, int passes, float* out_score, uint32_t* out_pos, int64_t out_row_stride,
                    const tc_bound* bound);

/**
 * Pruning-bound pre-pass of the filtering scan (KC > 0 with a bound): for each of the nq queries, scores the first rows of
 * its nearest probed list(s) in fp32 from the code stream and the pair's residual rows (q_hi, and q_lo with two passes), and
 * atomically lowers b_keys[q] (tc_bound key encoding, distance units: add[slot] + scale * score) to a value that is at least
 * the k-th best distance pq_stream_scan and the merge will find among those rows, raised far enough that every row of the
 * query's final top k still passes each item's starting threshold (DESIGN.md §5).  slot_of [nq, n_probes] (probes in rank
 * order), pair_list [slots], list_offsets [n_lists + 1] (padded row offsets), add [slots]; residual rows [slots, Kp] with
 * Kp = 2 * pq_dim; k <= 64.
 */
void pq_bound_prime(cudaStream_t s, int device, const uint8_t* code_stream, const uint32_t* cb_words, int pq_dim, const __nv_bfloat16* q_hi,
                    const __nv_bfloat16* q_lo, int Kp, int passes, const uint32_t* slot_of, const uint32_t* pair_list, const int64_t* list_offsets,
                    const float* add, float scale, int64_t nq, int n_probes, int k, int* b_keys);

}  // namespace b200
