// Tensor-core scan + fused top-k engine (host API).
//
// One kernel serves every dense "queries x rows -> k best rows per query" contraction of the hot
// path: brute force (a3 in SURVEY §8a), IVF coarse search (a7/a10), IVF-Flat list scans (a8), the
// k-means assignment step (a18).  Scores are  s(q, x) = hn[x] - q.x  (hn = |x|^2/2 for L2, 0 for
// inner product, +inf for padding rows), smaller is better; the caller maps them back to the
// metric.  See scan_tc.cu for the kernel and DESIGN.md §3 for the layout.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstdint>

namespace b200 {

constexpr int kTcTile = 128;  // rows of A (queries) and rows of B (dataset) per MMA tile
constexpr int kTcMaxK = 2048; // largest padded dimension (K <= 128: query tile resident in smem; above: streamed k-blocks)

/** One unit of work: 128 query rows against a contiguous range of 128-row dataset tiles. */
struct tc_item {
  uint32_t a_row0;      // first row in the A planes (any row; 128 rows are read)
  uint32_t b_row0;      // first row in the B planes (multiple of 128)
  uint32_t n_tiles;     // number of 128-row B tiles to scan
  uint32_t valid_rows;  // rows of the A tile that are real queries (<= 128)
  uint64_t out_off;     // element offset of (row 0, slot 0) in out_score/out_pos
};

/** items[m_tiles * splits]: every 128-row tile of the nq A rows against each of `splits` equal ranges of the b_tiles B tiles.
 *  Item i is (range i / m_tiles, A tile i % m_tiles): split-major, so CTAs that run at the same time stream the same B range
 *  (L2 reuse).  An item's out_off is (a_row0 * splits + s) * row_stride for range s: with an output row stride of
 *  splits * row_stride, each A row keeps its ranges' outputs side by side. */
void tc_split_items(cudaStream_t stream, tc_item* items, int m_tiles, int splits, int64_t nq, uint32_t b_tiles, int64_t row_stride);

/**
 * Optional cross-item pruning bound (the role of `query_kths` in the reference's compute_similarity kernel,
 * cpp/src/neighbors/ivf_pq/detail/jit_lto_kernels/compute_distances_impl.cuh:64-65,96): work items that scan different
 * row ranges for the SAME query share one running upper bound on that query's k'-th best value.  An item starts with
 *   thr = (bound[b] - add[a_row]) / scale      b = idx ? idx[a_row] : a_row
 * instead of +inf and publishes  add[a_row] + scale * (its k'-th best score)  with an atomic min when its list is full.
 * Values are stored as order-preserving ints (tc_bound_init_value = "+inf").  Rows dropped by the bound can never be
 * among the query's k' best, so results (and the brute-force certificate) are unchanged.
 */
struct tc_bound {
  int* keys           = nullptr;  // [n_bounds] ordered-int encoded floats
  const uint32_t* idx = nullptr;  // [a_rows] bound slot of every A row (null: the A row itself)
  const float* add    = nullptr;  // [a_rows] (null: 0)
  float scale         = 1.0f;
  int kth             = 0;        // the caller only needs each query's kth best (1..KC; 0 = KC): lists prune at, and publish,
                                  // their kth entry instead of their last one
};
constexpr int tc_bound_init_byte = 0x7f;  // memset value: 0x7f7f7f7f decodes to 3.39e38

inline int tc_pad_k(int d) { return (d + 63) / 64 * 64; }
inline int64_t tc_pad_rows(int64_t n) { return (n + kTcTile - 1) / kTcTile * kTcTile; }

/** Candidate lists the kernel emits per (item, query row): two epilogue threads per accumulator row, each owning
 *  64 of the tile's 128 columns.  Every list holds KC entries; list j sits at +j*KC. */
constexpr int kTcListsPerItem = 2;

/** True when the device/shape combination is served by the wgmma kernel (sm_90, padded dim <= kTcMaxK). */
bool tc_supported(int device, int d);

/**
 * Split an fp32 row-major matrix into bf16 hi / lo planes [rows_pad, Kp] (x ~= hi + lo, zero padded).
 * `scale` multiplies each row first when non-null (1/|x| for cosine).  lo may be null (hi only).
 */
void tc_split_planes(cudaStream_t stream, const float* x, int64_t n, int64_t ld, int d, int Kp, __nv_bfloat16* hi,
                     __nv_bfloat16* lo, int64_t rows_pad, const float* row_scale);

/**
 * Half-norm plane hx [rows_pad, 16] bf16 (32 bytes per row): columns 0..2 hold -hn[j] as three bf16 pieces (exact),
 * hn[j] = 0.5 * xn[j] (or 0 when xn == null) for j < n, +inf for n <= j < rows_pad; columns 3..15 are zero.  The scan
 * kernel feeds it to the tensor cores as one extra K = 16 step, so the accumulator is q.x - hn directly.
 */
void tc_half_norms(cudaStream_t stream, const float* xn, int64_t n, int64_t rows_pad, __nv_bfloat16* hx);
/** Same plane from ready-made half norms hn[rows_pad] (may hold +inf for rows to exclude). */
void tc_pack_half_norms(cudaStream_t stream, const float* hn, int64_t rows_pad, __nv_bfloat16* hx);

/**
 * Run the scan.  For every item and every valid row r the kernel writes kTcListsPerItem lists of KC
 * (score, position) pairs, each sorted best-first, at out_off + r * out_row_stride (+0..lists*KC-1); empty slots hold
 * (+inf, 0xffffffff).  `passes` = 3 uses hi*hi + lo*hi + hi*lo (fp32-grade products), 2 uses (hi + lo)*hi (exact when the B rows are
 * bf16 numbers, e.g. decoded PQ rows), 1 uses hi*hi.
 * KC must be 16 or 32 — or 0 for the dense "store" epilogue: all scores of the item are written to
 * out_score[out_off + r * out_row_stride + j], j = column offset inside the item's row range (out_pos unused).
 * out_row_stride == 0 (store only) makes the stride each item's own width, n_tiles * 128: the item's rows are written back
 * to back, as the per-pair score segments of an IVF search need (item_segments).
 * With KC > 0 and out_score == null nothing is written (a bound warm-up pass: only `bound` is updated).
 * `dynamic_schedule`: items are handed to CTAs through a global counter (adjacent items — e.g. the query groups of one
 * IVF list — run at the same time on different SMs and share the list's tiles through L2); false = static round-robin.
 * `n_items` is the host-known count or an upper bound; when `n_items_dev` is non-null the kernel reads the
 * exact count from it (work lists built on the device, no host round trip).
 */
void tc_scan_topk(cudaStream_t stream, int device, const __nv_bfloat16* a_hi, const __nv_bfloat16* a_lo,
                  int64_t a_rows_pad, const __nv_bfloat16* b_hi, const __nv_bfloat16* b_lo, int64_t b_rows_pad, int Kp,
                  const __nv_bfloat16* hx, const tc_item* items_dev, int n_items, const int* n_items_dev, int KC, int passes,
                  float* out_score, uint32_t* out_pos, int64_t out_row_stride, const tc_bound* bound = nullptr,
                  bool dynamic_schedule = true);

/**
 * 8-bit rows (DESIGN.md §4 "Row types").  Scores are exact integers, s = |x|^2 - 2 q.x (L2) or -q.x (inner product), handed to
 * the epilogue and written out as order-preserving fp32 keys: the float whose bits are s + kI8KeyBias (positive and finite
 * for every d <= 2048), so that the fused top-k, the pruning bound and the radix selects rank them exactly.  A row norm of
 * kI8PadNorm (padding rows, rows a filter hides) scores +inf.
 */
constexpr int kI8KeyBias = 1 << 30;
constexpr int kI8PadNorm = 0x7fffffff;
__device__ __forceinline__ float tc_i8_key(int s) { return __int_as_float(s + kI8KeyBias); }
__device__ __forceinline__ int tc_i8_score(float key) { return __float_as_int(key) - kI8KeyBias; }
inline int tc_pad_k_i8(int d) { return (d + 127) / 128 * 128; }

/** id stored on padding rows (the padding of IVF lists; any other int64, negative ones included, is a user id). */
constexpr int64_t kPadId = INT64_MIN;

/** norms[r] = the exact |x_r|^2 of the rows [n_rows, Kp] of a padded 8-bit plane (uint8 when `is_unsigned`), or kI8PadNorm
 *  where row r is not live.  A row is live when r < n_live and, given ids, ids[r] is not kPadId and the bitset keep_bits
 *  (n_bits bits, 1 = keep; null: all) keeps ids[r]. */
void tc_i8_norms(cudaStream_t stream, bool is_unsigned, const uint8_t* rows, int64_t n_rows, int64_t n_live, int Kp, const int64_t* ids,
                 const uint32_t* keep_bits, int64_t n_bits, int* norms);

/**
 * tc_scan_topk over 8-bit rows: A [a_rows_pad, Kp] and B [b_rows_pad, Kp] int8 (uint8 when `is_unsigned`), K-major, Kp a
 * multiple of 128; b_norm [b_rows_pad] the exact |x|^2 of each B row (kI8PadNorm: excluded), `l2` false for inner product.
 * Same work items, epilogues and outputs as tc_scan_topk with passes = 1, the scores being tc_i8_key's.
 * KC = 32 needs Kp = 128.
 */
void tc_scan_i8(cudaStream_t stream, int device, bool is_unsigned, const void* a, int64_t a_rows_pad, const void* b,
                int64_t b_rows_pad, int Kp, const int* b_norm, bool l2, const tc_item* items_dev, int n_items,
                const int* n_items_dev, int KC, float* out_score, uint32_t* out_pos, int64_t out_row_stride,
                const tc_bound* bound = nullptr, bool dynamic_schedule = true);

/**
 * tc_scan_topk over fp16 rows b [b_rows_pad, Kp] (zero padded, the bf16 planes' layout) with their half-norm plane hx, fused
 * top-KC (16 or 32) only.  fp16 queries: a_hi the query rows, a_lo and a_scale null; one pass of exact products.  fp32
 * queries: row r scaled by the power of two a_scale[r] [a_rows_pad] and split into fp16 a_hi + a_lo, two passes (hi + lo) * b;
 * the scores come out unscaled.  Scores and lists as tc_scan_topk's.
 */
void tc_scan_f16(cudaStream_t stream, int device, const __half* a_hi, const __half* a_lo, const float* a_scale, int64_t a_rows_pad,
                 const __half* b, int64_t b_rows_pad, int Kp, const __nv_bfloat16* hx, const tc_item* items_dev, int n_items, int KC,
                 float* out_score, uint32_t* out_pos, int64_t out_row_stride, const tc_bound* bound, bool dynamic_schedule);

}  // namespace b200
