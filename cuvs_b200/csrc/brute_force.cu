// Exact kNN ("brute force"): index + search + C boundary.
//
// Reference path being replaced (SURVEY §8a rows a1-a4):
//   index / build      cpp/src/neighbors/brute_force.cu:32-108, detail/knn_brute_force.cuh:778-818
//   search dispatch    detail/knn_brute_force.cuh:353-539 (fused SIMT kernel for k<=64 L2, tiled cuBLAS otherwise)
//   C wrapper          c/src/neighbors/brute_force.cpp:120-330
//
// Design (DESIGN.md §3): the index keeps, next to the fp32 rows and their norms, the rows
// split into two bf16 planes (x = hi + lo) padded to 128-row tiles.  Search is
//   1. candidate scan on wgmma (scan_tc.cu): s = |x|^2/2 - q.x with split-bf16 products, a
//      register top-k' per query row per dataset split, no distance matrix in HBM;
//   2. merge of the per-split lists (select_k.cu);
//   3. exact fp32 re-scoring of the k' candidates in the oracle's arithmetic (exact.cu);
//   4. a certificate (certify_candidates): if the k-th exact distance is not strictly below the worst
//      candidate's approximate distance minus the error budget, the query is flagged;
//   5. flagged queries (ties / duplicates at the k' boundary) are recomputed by the exact SIMT
//      path.  Result: identical to oracle/oracle.c::oracle_knn, bit for bit.
// Filtered search and shapes the tensor-core kernel does not cover (dim > 2048, k > 64)
// run on the exact SIMT path.
//
// Row types (DESIGN.md §3 "Row types"): float16, int8 and uint8 rows are kept in their own type.  float16 rows are scanned on
// fp16 wgmma, int8 / uint8 rows on the integer tensor cores (exact integer scores); cosine keeps the bf16 planes of the unit
// rows.  The re-score and the exact path read the typed rows and widen each element on load.
#include "common.hpp"
#include "exact.cuh"
#include "ivf_common.cuh"  // abs_max_host
#include "npy_io.hpp"
#include "scan_tc.cuh"
#include "select_k.cuh"
#include "timing.hpp"

#include <cuvs/neighbors/brute_force.h>
#include <cuvs_b200/ext.h>

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <fstream>
#include <memory>
#include <vector>

namespace b200 {

struct bf_index {
  int64_t n   = 0;
  int d       = 0;
  int device  = 0;
  cuvsDistanceType metric = L2Expanded;
  float metric_arg        = 2.0f;
  row_type type          = row_type::f32;  // the element type of the rows
  const float* data       = nullptr;  // float32 rows: [n, d] row-major on the device (view or data_own)
  owned<float> data_own;
  // float16 / int8 / uint8 rows, `ld` elements apart: the scan's zero-padded operand [rows_pad, Kp] when the scan reads them
  // (f16_scan, i8_scan), else [n, d]
  owned<uint8_t> rows;
  int64_t ld = 0;
  owned<float> norms;  // |x|^2 of the (widened) rows in the oracle's order (always kept: the certificate needs max norm)
  float xn_max = 0.f;
  // tensor-core side
  bool tc      = false;
  int Kp       = 0;  // padded K of the scan's operands (8-bit scans: tc_pad_k_i8)
  int64_t rows_pad = 0;
  owned<__nv_bfloat16> hi, lo;  // float32 rows, and cosine on every row type
  owned<__nv_bfloat16> hx;  // [rows_pad, 16] half-norm plane (scan_tc.cuh) of the bf16 and fp16 scans
  owned<float> inv_norm;  // cosine only
  owned<int> norms8;      // 8-bit scans: [rows_pad] exact |x|^2, kI8PadNorm on padding rows
  bool f16_scan() const { return tc && type == row_type::f16 && metric != CosineExpanded; }
  bool i8_scan() const { return tc && row_bytes(type) == 1 && metric != CosineExpanded; }
  template <typename T>
  const T* rows_as() const { return reinterpret_cast<const T*>(rows.data()); }
  int64_t device_bytes() const
  {
    return static_cast<int64_t>(data_own.size() * 4 + rows.size() + norms.size() * 4 + (hi.size() + lo.size() + hx.size()) * 2 +
                                inv_norm.size() * 4 + norms8.size() * 4);
  }
};

namespace {

// f(rows, ld): the index's rows in their own element type
template <typename F>
void with_rows(const bf_index& idx, F&& f)
{
  with_row_type(idx.type, [&](auto t) {
    using T = decltype(t);
    if constexpr (std::is_same_v<T, float>) f(idx.data, static_cast<int64_t>(idx.d));
    else f(idx.rows_as<T>(), idx.ld);
  });
}

bool metric_supported(cuvsDistanceType m)
{
  return m == L2Expanded || m == L2SqrtExpanded || m == L2Unexpanded || m == L2SqrtUnexpanded || m == InnerProduct ||
         m == CosineExpanded;
}

// column-major [n, d] elements of E bytes -> rows `ld` elements apart
template <typename E>
__global__ void transpose_into_kernel(const E* __restrict__ in, E* __restrict__ out, int64_t n, int d, int64_t ld)
{
  int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (t >= n * d) return;
  const int64_t r = t / d;
  const int c     = static_cast<int>(t % d);
  out[r * ld + c] = in[static_cast<int64_t>(c) * n + r];
}

// The A operand of a narrow scan from fp32 query rows that hold values of type T (exact): [rows_pad, Kp], zero padded
template <typename T>
__global__ void pack_queries_kernel(const float* __restrict__ q, int64_t nq, int d, int Kp, int64_t rows_pad, T* __restrict__ out)
{
  const int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (t >= rows_pad * Kp) return;
  const int64_t r = t / Kp;
  const int c     = static_cast<int>(t % Kp);
  const float v   = r < nq && c < d ? q[r * d + c] : 0.f;
  if constexpr (std::is_same_v<T, __half>) out[t] = __float2half_rn(v);
  else out[t] = static_cast<T>(static_cast<int>(v));
}

// fp32 query rows against fp16 rows: row r scaled by 2^e, e putting its largest |component| in [2^14, 2^15) (e clamped to
// [-60, 60]; a zero row keeps e = 0), then split into fp16 hi + lo.  scale[r] = 2^e (1 on padding rows).  One warp per row.
__global__ void split_f16_queries_kernel(const float* __restrict__ q, int64_t nq, int d, int Kp, int64_t rows_pad,
                                         __half* __restrict__ hi, __half* __restrict__ lo, float* __restrict__ scale)
{
  const int64_t r = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
  const int lane  = threadIdx.x & 31;
  if (r >= rows_pad) return;
  float m = 0.f;
  if (r < nq)
    for (int c = lane; c < d; c += 32) m = fmaxf(m, fabsf(q[r * d + c]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  int ex = 0;
  if (m > 0.f) {
    frexpf(m, &ex);  // m in [2^(ex-1), 2^ex)
    ex = min(60, max(-60, 15 - ex));
  }
  const float sc = ldexpf(1.0f, ex);
  for (int c = lane; c < Kp; c += 32) {
    const float v  = r < nq && c < d ? q[r * d + c] * sc : 0.f;
    const __half h = __float2half_rn(v);
    hi[r * Kp + c] = h;
    lo[r * Kp + c] = __float2half_rn(v - __half2float(h));
  }
  if (lane == 0) scale[r] = sc;
}

// 8-bit scan keys (tc_i8_key) -> the bf16 scan's units s = hn - q.x: half the integer score for L2, the score itself for inner
// product; +inf (empty slots) stays
__global__ void i8_keys_to_scores_kernel(float* __restrict__ v, int64_t count, float mul)
{
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= count) return;
  const float key = v[i];
  if (key < INFINITY) v[i] = mul * static_cast<float>(tc_i8_score(key));
}

int pick_splits(int m_tiles, int64_t b_tiles, int sms)
{
  int64_t s_max = std::max<int64_t>(1, std::min<int64_t>(32, b_tiles / 8));
  int best = 1;
  double best_eff = -1;
  for (int s = 1; s <= s_max; ++s) {
    int64_t items = static_cast<int64_t>(m_tiles) * s;
    int64_t waves = (items + sms - 1) / sms;
    double eff    = static_cast<double>(items) / static_cast<double>(waves * sms);
    if (eff > best_eff + 1e-9) { best_eff = eff; best = s; }
  }
  return best;
}

}  // namespace

// ------------------------------------------------------------------------------------ build
static bf_index* bf_build(resources* res, const DLTensor& ds, cuvsDistanceType metric, float metric_arg)
{
  B2_EXPECTS(ds.ndim == 2, "dataset must be a 2-D tensor");
  B2_EXPECTS(metric_supported(metric), "brute_force: unsupported metric %d", int(metric));
  auto idx        = std::make_unique<bf_index>();
  idx->n          = ds.shape[0];
  idx->d          = static_cast<int>(ds.shape[1]);
  idx->metric     = metric;
  idx->metric_arg = metric_arg;
  idx->device     = res->device;
  idx->type       = row_type_of(ds.dtype);
  auto stream     = res->stream;
  const bool c_contig = dl_is_c_contiguous(ds), f_contig = dl_is_f_contiguous(ds);
  B2_EXPECTS(c_contig || f_contig, "dataset input to cuvsBruteForceBuild must be contiguous (non-strided)");
  const float* src = dl_ptr<float>(ds);
  const size_t count = static_cast<size_t>(idx->n) * idx->d;
  idx->tc = tc_supported(res->device, idx->d) && idx->n >= 1 && idx->n < (int64_t(1) << 31);
  const bool l2 = (metric != InnerProduct && metric != CosineExpanded);
  if (idx->type != row_type::f32) {
    // float16 / int8 / uint8: the rows in their own type, in the scan's padded operand when the scan reads them
    const int es   = static_cast<int>(row_bytes(idx->type));
    idx->rows_pad  = tc_pad_rows(idx->n);
    const bool pad = idx->f16_scan() || idx->i8_scan();
    idx->Kp        = idx->type == row_type::f16 || metric == CosineExpanded ? tc_pad_k(idx->d) : tc_pad_k_i8(idx->d);
    idx->ld        = pad ? idx->Kp : idx->d;
    const int64_t rows = pad ? idx->rows_pad : idx->n;
    idx->rows.alloc(static_cast<size_t>(rows * idx->ld * es));
    if (pad) B2_CUDA(cudaMemsetAsync(idx->rows.data(), 0, idx->rows.size(), stream));
    if (count == 0) {
    } else if (c_contig) {
      B2_CUDA(cudaMemcpy2DAsync(idx->rows.data(), idx->ld * es, ds.data, static_cast<size_t>(idx->d) * es,
                                static_cast<size_t>(idx->d) * es, idx->n, cudaMemcpyDefault, stream));
    } else {
      dbuf<uint8_t> tmp(count * es, stream);
      B2_CUDA(cudaMemcpyAsync(tmp.data(), ds.data, count * es, cudaMemcpyDefault, stream));
      count_launch();
      if (es == 2)
        transpose_into_kernel<<<blocks_for(static_cast<int64_t>(count), 256), 256, 0, stream>>>(
          reinterpret_cast<const uint16_t*>(tmp.data()), reinterpret_cast<uint16_t*>(idx->rows.data()), idx->n, idx->d, idx->ld);
      else
        transpose_into_kernel<<<blocks_for(static_cast<int64_t>(count), 256), 256, 0, stream>>>(
          tmp.data(), idx->rows.data(), idx->n, idx->d, idx->ld);
      B2_CUDA(cudaGetLastError());
    }
  } else if (dl_is_device(ds) && ds.device.device_type != kDLCUDAHost && c_contig) {
    idx->data = src;  // non-owning view, like the reference (brute_force.cu:60-75)
  } else {
    idx->data_own.alloc(count);
    if (c_contig) {
      B2_CUDA(cudaMemcpyAsync(idx->data_own.data(), src, count * sizeof(float), cudaMemcpyDefault, stream));
    } else {
      dbuf<float> tmp(count, stream);
      B2_CUDA(cudaMemcpyAsync(tmp.data(), src, count * sizeof(float), cudaMemcpyDefault, stream));
      if (count)
        transpose_into_kernel<<<blocks_for(static_cast<int64_t>(count), 256), 256, 0, stream>>>(tmp.data(), idx->data_own.data(), idx->n,
                                                                                                idx->d, int64_t(idx->d));
      B2_CUDA(cudaGetLastError());
    }
    idx->data = idx->data_own.data();
  }
  idx->norms.alloc(static_cast<size_t>(std::max<int64_t>(idx->n, 1)));
  with_rows(*idx, [&](auto x, int64_t ld) { row_norms(stream, x, idx->n, idx->d, ld, idx->norms.data()); });
  // the norms are >= 0: their largest |value|.  A NaN norm (a row holding NaN) ranks above +inf, so xn_max is NaN; the
  // certificate's budget is then NaN and fails every query it is applied to: those queries take the exact path.
  const uint32_t xn_max_bits = abs_max_host(stream, idx->norms.data(), idx->n);
  std::memcpy(&idx->xn_max, &xn_max_bits, sizeof(float));
  if (idx->i8_scan()) {
    idx->norms8.alloc(static_cast<size_t>(idx->rows_pad));
    tc_i8_norms(stream, idx->type == row_type::u8, idx->rows.data(), idx->rows_pad, idx->n, idx->Kp, nullptr, nullptr, 0, idx->norms8.data());
  } else if (idx->f16_scan()) {
    idx->hx.alloc(static_cast<size_t>(idx->rows_pad) * 16);
    tc_half_norms(stream, l2 ? idx->norms.data() : nullptr, idx->n, idx->rows_pad, idx->hx.data());
  } else if (idx->tc) {
    idx->Kp       = tc_pad_k(idx->d);
    idx->rows_pad = tc_pad_rows(idx->n);
    idx->hi.alloc(static_cast<size_t>(idx->rows_pad) * idx->Kp);
    idx->lo.alloc(static_cast<size_t>(idx->rows_pad) * idx->Kp);
    idx->hx.alloc(static_cast<size_t>(idx->rows_pad) * 16);
    const float* scale = nullptr;
    if (metric == CosineExpanded) {
      idx->inv_norm.alloc(static_cast<size_t>(idx->n));
      rsqrt_rows(stream, idx->norms.data(), idx->n, idx->inv_norm.data());
      scale = idx->inv_norm.data();
    }
    if (idx->type == row_type::f32) {
      tc_split_planes(stream, idx->data, idx->n, idx->d, idx->d, idx->Kp, idx->hi.data(), idx->lo.data(), idx->rows_pad, scale);
    } else {
      // cosine over narrow rows: the planes of the unit rows from bounded chunks of widened rows, which are not kept
      const int64_t chunk = std::max<int64_t>(kTcTile, ((int64_t(1) << 24) / idx->d) / kTcTile * kTcTile);
      dbuf<float> w(static_cast<size_t>(std::min(chunk, idx->n) * idx->d), stream);
      for (int64_t r0 = 0; r0 < idx->n; r0 += chunk) {
        const int64_t c   = std::min(chunk, idx->n - r0);
        const int64_t pad = r0 + chunk >= idx->n ? idx->rows_pad - r0 : c;  // the last chunk zeroes the padding rows
        widen_async(stream, idx->rows.data() + r0 * idx->ld * row_bytes(idx->type), dtype_of(idx->type), c * idx->d, w.data());
        tc_split_planes(stream, w.data(), c, idx->d, idx->d, idx->Kp, idx->hi.data() + r0 * idx->Kp, idx->lo.data() + r0 * idx->Kp,
                        pad, scale + r0);
      }
    }
    tc_half_norms(stream, l2 ? idx->norms.data() : nullptr, idx->n, idx->rows_pad, idx->hx.data());
  }
  return idx.release();
}

// ------------------------------------------------------------------------------------ search
static void search_exact(resources* res, const bf_index& idx, const float* q, int64_t nq, int64_t q_row0, int k,
                         int64_t* out_idx, float* out_dist, filter_view filt)
{
  auto stream = res->stream;
  if (nq == 0) return;
  const bool select_min = metric_is_min_close(idx.metric);
  const bool need_norms = (idx.metric == L2Expanded || idx.metric == L2SqrtExpanded || idx.metric == CosineExpanded);
  dbuf<float> qn;
  if (need_norms) {
    qn.alloc(static_cast<size_t>(nq), stream);
    row_norms(stream, q, nq, idx.d, idx.d, qn.data());
  }
  const int64_t n_cols = std::max<int64_t>(idx.n, 1);
  int64_t chunk = std::max<int64_t>(1, std::min<int64_t>(nq, (int64_t(1) << 28) / n_cols));
  chunk         = std::min<int64_t>(chunk, 65535 * 64);
  dbuf<float> dist(static_cast<size_t>(chunk * n_cols), stream);
  for (int64_t q0 = 0; q0 < nq; q0 += chunk) {
    int64_t qc = std::min(chunk, nq - q0);
    with_rows(idx, [&](auto x, int64_t ld) {
      exact_distance_tile(stream, q + q0 * idx.d, qc, idx.d, x, idx.n, ld, idx.d, need_norms ? qn.data() + q0 : nullptr,
                          need_norms ? idx.norms.data() : nullptr, idx.metric, dist.data(), idx.n, filt, q_row0 + q0);
    });
    select_k(stream, dist.data(), nullptr, IDX_NONE, qc, idx.n, idx.n, k, out_dist + q0 * k, out_idx + q0 * k, IDX_I64,
             select_min);
  }
}

__global__ void mask_filtered_kernel(int64_t* idx, float* dist, int64_t count, bool select_min)
{
  int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= count) return;
  float worst = select_min ? FLT_MAX : -FLT_MAX;
  if (dist[i] == worst) idx[i] = -1;  // nothing (or only filtered-out rows) left for this slot
}

struct bf_cands {
  dbuf<float> score;    // [nq, KCm] raw engine scores s = hn - q.x (best first)
  dbuf<uint32_t> pos;   // [nq, KCm] row positions
  dbuf<float> qn;       // [nq] |q|^2
  dbuf<float> floor;    // [nq] (KCm > KC only) min over the scan's FULL candidate lists of the list's worst kept score
  int width = 0;        // entries per query row in score / pos (KCm, or everything the scan kept when that is less)
};

// Stage 1+2 of the search: wgmma scan over `splits` dataset ranges (lists of KC per column half and split) +
// merge to KCm per query (KCm == KC: the merged set's worst entry bounds everything outside it; KCm > KC, used for k above
// the fused list length: `out.floor` carries the bound for the rows that never entered a list).  The scan is split-bf16 over
// the bf16 planes, fp16 over fp16 rows (q_narrow: the queries hold fp16 values, one pass; else the scaled two-pass split) or
// 8-bit over 8-bit rows (q_narrow).  Scores come out in the bf16 scan's units, s = hn - q.x.
static void bf_tc_candidates(resources* res, const bf_index& idx, const float* q, int64_t nq, bool q_narrow, int KC, bf_cands& out,
                             int KCm = 0)
{
  if (KCm <= 0) KCm = KC;
  auto stream           = res->stream;
  const int64_t nq_pad  = tc_pad_rows(nq);
  const int m_tiles     = static_cast<int>(nq_pad / 128);
  const int64_t b_tiles = idx.rows_pad / 128;
  int splits            = pick_splits(m_tiles, b_tiles, res->sm_count ? res->sm_count : 132);
  // 8-bit lists of 16 at k > 16: enough lists per query that the merged width covers KCm
  if (idx.i8_scan()) splits = std::max(splits, (KCm + kTcListsPerItem * KC - 1) / (kTcListsPerItem * KC));
  const int n_items     = m_tiles * splits;

  out.qn.alloc(static_cast<size_t>(nq), stream);
  row_norms(stream, q, nq, idx.d, idx.d, out.qn.data());
  dbuf<float> qscale;
  dbuf<__nv_bfloat16> qhi, qlo;
  dbuf<__half> qh, ql;
  dbuf<uint8_t> q8;
  const int64_t a_elems = nq_pad * idx.Kp;
  if (idx.i8_scan()) {
    B2_EXPECTS(q_narrow, "brute_force: an 8-bit index is scanned with queries of its own type");
    q8.alloc(static_cast<size_t>(a_elems), stream);
    count_launch();
    if (idx.type == row_type::u8)
      pack_queries_kernel<<<blocks_for(a_elems, 256), 256, 0, stream>>>(q, nq, idx.d, idx.Kp, nq_pad, q8.data());
    else
      pack_queries_kernel<<<blocks_for(a_elems, 256), 256, 0, stream>>>(q, nq, idx.d, idx.Kp, nq_pad, reinterpret_cast<int8_t*>(q8.data()));
    B2_CUDA(cudaGetLastError());
  } else if (idx.f16_scan()) {
    qh.alloc(static_cast<size_t>(a_elems), stream);
    count_launch();
    if (q_narrow) {
      pack_queries_kernel<<<blocks_for(a_elems, 256), 256, 0, stream>>>(q, nq, idx.d, idx.Kp, nq_pad, qh.data());
    } else {
      ql.alloc(static_cast<size_t>(a_elems), stream);
      qscale.alloc(static_cast<size_t>(nq_pad), stream);
      split_f16_queries_kernel<<<blocks_for(nq_pad * 32, 256), 256, 0, stream>>>(q, nq, idx.d, idx.Kp, nq_pad, qh.data(), ql.data(),
                                                                                 qscale.data());
    }
    B2_CUDA(cudaGetLastError());
  } else {
    if (idx.metric == CosineExpanded) {
      qscale.alloc(static_cast<size_t>(nq), stream);
      rsqrt_rows(stream, out.qn.data(), nq, qscale.data());
    }
    qhi.alloc(static_cast<size_t>(a_elems), stream);
    qlo.alloc(static_cast<size_t>(a_elems), stream);
    tc_split_planes(stream, q, nq, idx.d, idx.d, idx.Kp, qhi.data(), qlo.data(), nq_pad, qscale.data());
  }

  dbuf<tc_item> items(static_cast<size_t>(n_items), stream);
  const int KCW = KC * kTcListsPerItem;  // candidates per (item, query row)
  tc_split_items(stream, items.data(), m_tiles, splits, nq, static_cast<uint32_t>(b_tiles), KCW);

  const int64_t row_stride = static_cast<int64_t>(splits) * KCW;
  dbuf<float> cs(static_cast<size_t>(nq_pad) * row_stride, stream);
  dbuf<uint32_t> cp(static_cast<size_t>(nq_pad) * row_stride, stream);
  // the splits of one query row share a running k'-th-best bound (scores are comparable: same query)
  dbuf<int> bkeys(static_cast<size_t>(nq_pad), stream);
  B2_CUDA(cudaMemsetAsync(bkeys.data(), tc_bound_init_byte, sizeof(int) * nq_pad, stream));
  tc_bound bnd;
  bnd.keys = bkeys.data();
  // equal-sized items in split-major order: static round-robin keeps each column range L2 resident
  if (idx.i8_scan()) {
    tc_scan_i8(stream, res->device, idx.type == row_type::u8, q8.data(), nq_pad, idx.rows.data(), idx.rows_pad, idx.Kp, idx.norms8.data(),
               idx.metric != InnerProduct, items.data(), n_items, nullptr, KC, cs.data(), cp.data(), row_stride, &bnd, false);
    count_launch();
    const int64_t cnt = nq_pad * row_stride;
    i8_keys_to_scores_kernel<<<blocks_for(cnt, 256), 256, 0, stream>>>(cs.data(), cnt, idx.metric == InnerProduct ? 1.0f : 0.5f);
    B2_CUDA(cudaGetLastError());
  } else if (idx.f16_scan()) {
    tc_scan_f16(stream, res->device, qh.data(), ql.data(), qscale.data(), nq_pad, idx.rows_as<__half>(), idx.rows_pad, idx.Kp,
                idx.hx.data(), items.data(), n_items, KC, cs.data(), cp.data(), row_stride, &bnd, false);
  } else {
    tc_scan_topk(stream, res->device, qhi.data(), qlo.data(), nq_pad, idx.hi.data(), idx.lo.data(), idx.rows_pad, idx.Kp,
                 idx.hx.data(), items.data(), n_items, nullptr, KC, 3, cs.data(), cp.data(), row_stride, &bnd, false);
  }
  if (KCm > KC) {
    out.floor.alloc(static_cast<size_t>(nq), stream);
    list_floors(stream, cs.data(), nq, row_stride, KC, out.floor.data());
  }
  out.width = static_cast<int>(std::min<int64_t>(row_stride, KCm));
  if (row_stride > KCm) {
    out.score.alloc(static_cast<size_t>(nq) * KCm, stream);
    out.pos.alloc(static_cast<size_t>(nq) * KCm, stream);
    select_k(stream, cs.data(), cp.data(), IDX_U32, nq, row_stride, row_stride, KCm, out.score.data(), out.pos.data(), IDX_U32, true);
  } else {
    out.score = std::move(cs);
    out.pos   = std::move(cp);
  }
}

static approx_map bf_approx_map(const bf_index& idx)
{
  approx_map am;
  // Relative to |q|^2 + max|x|^2 (DESIGN.md §3): the split-bf16 products are within 3*2^-18*2|q||x| <= 2^-16.4 of exact, and
  // the fp32 accumulation of Kp products adds up to ~Kp*2^-24 (Kp/16 wgmma k-steps of 16).  max(2^-15, 2^-16 + Kp*2^-24)
  // covers both; it is 2^-15 up to Kp = 256 (so the d <= 128 searches keep their budget) and 2^-13 + 2^-16 at Kp = 2048.
  // fp16 scans (exact products, or a split query within 2^-21 |q||x|) stay inside the same budget.
  am.eps_rel = std::max(1.0f / 32768.0f, 1.0f / 65536.0f + static_cast<float>(idx.Kp) / 16777216.0f);
  // 8-bit scans score exact integers; the budget covers the fp32 re-score's rounding against them (<= 2d ulps of
  // |q|^2 + |x|^2 for a sum of d products or squared differences and its finish) and the scores' conversion to fp32.  Below
  // |q|^2 + max|x|^2 = 2^23 there is no rounding at all and the budget is 0 (certify_candidates' exact_ints).
  if (idx.i8_scan()) am.eps_rel = static_cast<float>(2 * idx.Kp + 8) / 16777216.0f;
  if (idx.metric == InnerProduct) { am.sa = -1.f; am.eq = 1.f; am.ec = idx.xn_max; }
  else if (idx.metric == CosineExpanded) { am.sa = 1.f; am.sc = 1.f; am.eq = 0.f; am.ec = 2.f; }
  else { am.sa = 2.f; am.sb = 1.f; am.eq = 1.f; am.ec = idx.xn_max; }
  return am;
}

// qt: fp32 queries; q_narrow when they are the widened values of queries of the index's own narrow type
static void bf_search(resources* res, const bf_index& idx, const DLTensor& qt, const DLTensor& nt, const DLTensor& dt,
                      cuvsFilter prefilter, bool q_narrow)
{
  auto stream      = res->stream;
  const int64_t nq = qt.shape[0];
  const int k      = static_cast<int>(nt.shape[1]);
  B2_EXPECTS(k >= 1, "k must be >= 1");
  int64_t* out_idx = dl_ptr<int64_t>(nt);
  float* out_dist  = dl_ptr<float>(dt);
  if (nq == 0) return;

  // queries: row-major view or a transposed copy
  const float* q = dl_ptr<float>(qt);
  dbuf<float> qcopy;
  if (!dl_is_c_contiguous(qt)) {
    B2_EXPECTS(dl_is_f_contiguous(qt), "queries input to cuvsBruteForceSearch must be contiguous (non-strided)");
    qcopy.alloc(static_cast<size_t>(nq) * idx.d, stream);
    transpose_into_kernel<<<blocks_for(nq * idx.d, 256), 256, 0, stream>>>(q, qcopy.data(), nq, idx.d, int64_t(idx.d));
    B2_CUDA(cudaGetLastError());
    q = qcopy.data();
  }

  filter_view filt = read_prefilter(prefilter, true, "Unsupported prefilter type");
  if (filt.kind) filt.n_samples = idx.n;  // the bitmap's row length

  const bool select_min = metric_is_min_close(idx.metric);
  // k <= 24: fused lists of 16 / 32, merged to the list length.  24 < k <= 64 (the reference's fused range,
  // knn_brute_force.cuh:447-451): fused lists of 32 per (column half, split), merged to 64 / 96 candidates, and the
  // certificate additionally uses the lists' own worst entries (bf_cands::floor) — a row of the true top-k can only be missing
  // when more than 32 of them fall into one list, which the certificate detects (flagged queries take the exact path).
  const bool use_tc     = idx.tc && filt.kind == 0 && k <= 64 && idx.n > 0;
  set_last_flagged(0);
  if (!use_tc) {
    search_exact(res, idx, q, nq, 0, k, out_idx, out_dist, filt);
    if (filt.kind)
      mask_filtered_kernel<<<static_cast<unsigned>((nq * k + 255) / 256), 256, 0, stream>>>(out_idx, out_dist, nq * k, select_min);
    postprocess_distances(stream, out_dist, nq * k, idx.metric);
    return;
  }

  // ---- tensor-core candidate scan
  // (the fused 8-bit top-32 exists at Kp = 128 only: wider 8-bit rows take lists of 16, merged to KCm with the floor bound)
  const bool kc32 = !idx.i8_scan() || idx.Kp == 128;
  const int KC    = k <= 10 || !kc32 ? 16 : 32;
  const int KCm   = k <= 10 ? 16 : (k <= 24 ? 32 : (k <= 48 ? 64 : 96));
  bf_cands cand;
  bf_tc_candidates(res, idx, q, nq, q_narrow, KC, cand, KCm);

  // ---- exact re-scoring
  const bool need_xn = (idx.metric == L2Expanded || idx.metric == L2SqrtExpanded || idx.metric == CosineExpanded);
  with_rows(idx, [&](auto x, int64_t ld) {
    rescore_topk(stream, q, nq, idx.d, x, ld, idx.d, cand.qn.data(), need_xn ? idx.norms.data() : nullptr, idx.metric,
                 cand.pos.data(), cand.width, nullptr, k, out_idx, out_dist, -1);
  });

  // ---- certificate, and the exact path for flagged queries (rare: exact ties / duplicates at the k' boundary)
  dbuf<int> flags(static_cast<size_t>(nq) + 1, stream);
  certify_candidates(stream, cand.score.data(), cand.pos.data(), cand.width, cand.floor.data(), cand.qn.data(), out_dist, k,
                     bf_approx_map(idx), select_min, idx.i8_scan(), nq, flags.data());
  // search_exact answers every query on its own, and these run unfiltered, so the gathered rows get the same bits
  rerun_flagged(stream, flags.data(), nq, k, out_idx, out_dist, [&](const int64_t* rows, int64_t n, int64_t* fi, float* fd) {
    dbuf<float> fq(static_cast<size_t>(n) * idx.d, stream);
    copy_rows(stream, q, rows, fq.data(), nullptr, n, idx.d);
    search_exact(res, idx, fq.data(), n, 0, k, fi, fd, filter_view{});
  });
  postprocess_distances(stream, out_dist, nq * k, idx.metric);
}

}  // namespace b200

using namespace b200;

// ------------------------------------------------------------------------------------ C boundary
extern "C" {

cuvsError_t cuvsBruteForceIndexCreate(cuvsBruteForceIndex_t* index)
{
  return guarded([=] {
    B2_EXPECTS(index != nullptr, "index is null");
    *index = new cuvsBruteForceIndex{};
  });
}

cuvsError_t cuvsBruteForceIndexDestroy(cuvsBruteForceIndex_t index)
{
  return guarded([=] {
    if (!index) return;
    drop_index<bf_index>(index);
    delete index;
  });
}

cuvsError_t cuvsBruteForceBuild(cuvsResources_t res, DLManagedTensor* dataset_tensor, cuvsDistanceType metric,
                                float metric_arg, cuvsBruteForceIndex_t index)
{
  return guarded([=] {
    auto r = as_res(res);
    B2_EXPECTS(dataset_tensor != nullptr && index != nullptr, "null argument");
    const DLTensor& ds = dataset_tensor->dl_tensor;
    // float32, float16, int8 or uint8 rows (c/src/neighbors/brute_force.cpp:60-110), each kept in its own type
    B2_EXPECTS(dl_is_dataset_dtype(ds), "Unsupported dataset DLtensor dtype: %d and bits: %d", ds.dtype.code, ds.dtype.bits);
    drop_index<bf_index>(index);
    set_index(index, bf_build(r, ds, metric, metric_arg), ds.dtype);
  });
}

cuvsError_t cuvsBruteForceSearch(cuvsResources_t res, cuvsBruteForceIndex_t index, DLManagedTensor* queries_tensor,
                                 DLManagedTensor* neighbors_tensor, DLManagedTensor* distances_tensor, cuvsFilter prefilter)
{
  return guarded([=] {
    auto r = as_res(res);
    B2_EXPECTS(queries_tensor && neighbors_tensor && distances_tensor, "null argument");
    auto& idx                 = index_of<bf_index>(index);
    const DLTensor& queries   = queries_tensor->dl_tensor;
    const DLTensor& neighbors = neighbors_tensor->dl_tensor;
    const DLTensor& distances = distances_tensor->dl_tensor;
    check_search_tensors(queries, neighbors, distances, idx.d, false);
    B2_EXPECTS(queries.dtype.code == index->dtype.code, "type mismatch between index and queries");
    if (dl_is(queries, kDLFloat, 32)) {
      bf_search(r, idx, queries, neighbors, distances, prefilter, false);
    } else if (dl_is_dataset_dtype(queries) && queries.dtype.bits == index->dtype.bits) {
      f32_rows w;
      widen_to_f32(r, queries, w);
      bf_search(r, idx, w.t, neighbors, distances, prefilter, true);
    } else {
      B2_FAIL("Unsupported queries DLtensor dtype: %d and bits: %d", queries.dtype.code, queries.dtype.bits);
    }
  });
}

cuvsError_t cuvsB200BruteForceCandidates(cuvsResources_t res, cuvsBruteForceIndex_t index, DLManagedTensor* queries,
                                         DLManagedTensor* cand_pos, DLManagedTensor* cand_score)
{
  return guarded([=] {
    auto r = as_res(res);
    B2_EXPECTS(queries && cand_pos && cand_score, "null argument");
    auto& idx           = index_of<bf_index>(index);
    const DLTensor& q   = queries->dl_tensor;
    const DLTensor& cp  = cand_pos->dl_tensor;
    const DLTensor& cs  = cand_score->dl_tensor;
    B2_EXPECTS(idx.tc, "index has no tensor-core planes on this device");
    // float32 queries, or (as cuvsBruteForceSearch accepts them) queries of the index's own type
    const bool q_f32 = dl_is(q, kDLFloat, 32);
    B2_EXPECTS((q_f32 || (dl_is_dataset_dtype(q) && q.dtype.bits == index->dtype.bits)) && dl_is_device(q) && dl_is_c_contiguous(q) &&
                 q.ndim == 2 && q.shape[1] == idx.d, "bad queries");
    B2_EXPECTS(q.dtype.code == index->dtype.code, "type mismatch between index and queries");
    const int KC = static_cast<int>(cp.shape[1]);
    B2_EXPECTS((KC == 16 || KC == 32) && dl_is(cp, kDLUInt, 32) && dl_is(cs, kDLFloat, 32) && cp.shape[0] == q.shape[0] &&
                 cs.shape[0] == q.shape[0] && cs.shape[1] == KC, "bad candidate tensors");
    B2_EXPECTS(KC == 16 || !idx.i8_scan() || idx.Kp == 128, "the 8-bit scan keeps lists of 32 at padded widths of 128 only");
    f32_rows w;
    widen_to_f32(r, q, w);
    bf_cands c;
    bf_tc_candidates(r, idx, dl_ptr<float>(w.t), q.shape[0], !q_f32, KC, c);
    B2_CUDA(cudaMemcpyAsync(dl_ptr<void>(cp), c.pos.data(), sizeof(uint32_t) * q.shape[0] * KC, cudaMemcpyDeviceToDevice, r->stream));
    B2_CUDA(cudaMemcpyAsync(dl_ptr<void>(cs), c.score.data(), sizeof(float) * q.shape[0] * KC, cudaMemcpyDeviceToDevice, r->stream));
    B2_CUDA(cudaStreamSynchronize(r->stream));
  });
}

// Serialization: 4-char numpy-style dtype tag of the rows ("<f4\0", "<f2\0", "|i1\0" or "|u1\0"), then n, dim, metric,
// metric_arg, the n x dim rows in that type.
// (Own container; the reference's brute_force_serialize.cu writes RAFT mdspans — compatibility is a
// "next" item, SURVEY §8f n1.)
cuvsError_t cuvsBruteForceSerialize(cuvsResources_t res, const char* filename, cuvsBruteForceIndex_t index)
{
  return guarded([=] {
    auto r = as_res(res);
    B2_EXPECTS(filename, "null argument");
    auto& idx    = index_of<bf_index>(index);
    const size_t es = row_bytes(idx.type);
    std::vector<char> host(static_cast<size_t>(idx.n) * idx.d * es);
    const void* src      = idx.type == row_type::f32 ? static_cast<const void*>(idx.data) : idx.rows.data();
    const size_t pitch   = static_cast<size_t>(idx.type == row_type::f32 ? idx.d : idx.ld) * es;
    if (!host.empty())
      B2_CUDA(cudaMemcpy2DAsync(host.data(), static_cast<size_t>(idx.d) * es, src, pitch, static_cast<size_t>(idx.d) * es, idx.n,
                                cudaMemcpyDeviceToHost, r->stream));
    B2_CUDA(cudaStreamSynchronize(r->stream));
    std::ofstream os(filename, std::ios::out | std::ios::binary);
    B2_EXPECTS(bool(os), "Cannot open file %s", filename);
    const char* descr = npy::file_dtype_for(dtype_of(idx.type)).descr;  // "<f4", "<f2", "|i1", "|u1"
    const char tag[4] = {descr[0], descr[1], descr[2], 0};
    os.write(tag, 4);
    int64_t n = idx.n, d = idx.d;
    int32_t m = int(idx.metric);
    os.write(reinterpret_cast<const char*>(&n), 8);
    os.write(reinterpret_cast<const char*>(&d), 8);
    os.write(reinterpret_cast<const char*>(&m), 4);
    os.write(reinterpret_cast<const char*>(&idx.metric_arg), 4);
    os.write(host.data(), static_cast<std::streamsize>(host.size()));
    B2_EXPECTS(bool(os), "Error writing %s", filename);
  });
}

cuvsError_t cuvsBruteForceDeserialize(cuvsResources_t res, const char* filename, cuvsBruteForceIndex_t index)
{
  return guarded([=] {
    auto r = as_res(res);
    B2_EXPECTS(index && filename, "null argument");
    std::ifstream is(filename, std::ios::in | std::ios::binary);
    B2_EXPECTS(bool(is), "Cannot open file %s", filename);
    char tag[4]{};
    B2_EXPECTS(bool(is.read(tag, 4)), "Invalid or truncated index header in file %s", filename);
    const npy::file_dtype* ft = npy::file_dtype_named(std::string(tag, 3));
    B2_EXPECTS(ft != nullptr, "Unsupported index dtype in %s", filename);
    int64_t n = 0, d = 0;
    int32_t m = 0;
    float marg = 0;
    is.read(reinterpret_cast<char*>(&n), 8);
    is.read(reinterpret_cast<char*>(&d), 8);
    is.read(reinterpret_cast<char*>(&m), 4);
    is.read(reinterpret_cast<char*>(&marg), 4);
    B2_EXPECTS(bool(is) && n >= 0 && d > 0, "Invalid index header in file %s", filename);
    std::vector<char> host(static_cast<size_t>(n) * d * ft->size);
    is.read(host.data(), static_cast<std::streamsize>(host.size()));
    B2_EXPECTS(bool(is), "Truncated index file %s", filename);
    const dl_view rows(host.data(), DLDevice{kDLCPU, 0}, ft->dl, n, d);
    drop_index<bf_index>(index);
    set_index(index, bf_build(r, rows.t(), static_cast<cuvsDistanceType>(m), marg), rows.t().dtype);
  });
}

cuvsError_t cuvsB200BruteForceIndexInfo(cuvsBruteForceIndex_t index, int* row_type, int64_t* device_bytes)
{
  return guarded([=] {
    B2_EXPECTS(row_type && device_bytes, "null argument");
    auto& idx     = index_of<bf_index>(index);
    *row_type     = static_cast<int>(idx.type);
    *device_bytes = idx.device_bytes();
  });
}

}  // extern "C"
