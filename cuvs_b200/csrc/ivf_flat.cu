// IVF-Flat: index, build / extend, search, C boundary.
//
// Reference path being replaced (SURVEY §8a rows a6-a8, a13):
//   index / list layout   cpp/include/cuvs/neighbors/ivf_flat.hpp:139-300
//   build / extend        cpp/src/neighbors/ivf_flat/ivf_flat_build.cuh:109-520 (balanced k-means + list fill)
//   search_impl           cpp/src/neighbors/ivf_flat/ivf_flat_search.cuh:41-309
//   interleaved_scan      cpp/src/neighbors/ivf_flat/detail/jit_lto_kernels/interleaved_scan_impl.cuh:70-206
//   C wrapper             c/src/neighbors/ivf_flat.cpp
//
// Search (DESIGN.md §4):
//   1. coarse: dense wgmma score block queries x centres (split-bf16, fp32-grade) + select_k(n_probes)
//   2. (query, probe) pairs are bucketed by list on the device (ivf_common.cu)
//   3. fine:   per (list, <=128 probing queries) work item, wgmma scan of the list's bf16 residual rows x - c with the
//              fused top-k' epilogue — each list tile is read once per 128 probing queries, not once per query.
//              k > 64: the same scan with the store epilogue writes every (pair, list row) score to the pair's dense
//              segment, and a segmented select keeps each pair's kc2 = min(2k, 2048) best (the reference's non-fused
//              formulation, ivf_flat_search.cuh:238-295)
//   4. per query: gather the candidates of its probes, keep the best few by approximate score, re-score
//      them exactly in fp32 (sum (q-x)^2 / q.x — the reference's fine-scan arithmetic) and emit ids.
//   5. certificate: a query whose k-th exact distance is not safely below every row the candidates left out (the bf16 score's
//      error budget) is searched again with every row of its probed lists scored exactly, so every query returns the
//      oracle's answer over its probed lists.
// int8 / uint8 indexes in L2 or inner product keep their rows as bytes and scan them on the integer tensor cores, whose scores
// are exact: steps 3-4 rank by exact integer keys and need no re-score or certificate (ivf_flat_search_i8, DESIGN.md §4
// "Row types").
#include "common.hpp"
#include "exact.cuh"
#include "exact_device.cuh"
#include "ivf_common.cuh"
#include "ivf_lists.cuh"
#include "npy_io.hpp"
#include "select_k.cuh"
#include "timing.hpp"

#include <cuvs/neighbors/ivf_flat.h>
#include <cuvs_b200/ext.h>

#include <cuda_fp16.h>

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <fstream>
#include <memory>
#include <vector>

namespace b200 {

struct ivf_flat_index {
  int device              = 0;
  cuvsDistanceType metric = L2Expanded;
  float metric_arg        = 2.0f;
  int dim                 = 0;
  uint32_t n_lists        = 0;
  bool adaptive_centers   = false;
  uint32_t kmeans_n_iters = 20;
  double kmeans_trainset_fraction = 0.5;
  owned<float> centers;  // [n_lists, dim]
  owned<float> centers_unit;  // cosine: [n_lists, dim] the unit centres the scan's residuals are taken from
  tc_rows centers_tc;    // split planes + |c|^2/2 (0 for inner product)
  list_layout lists;
  owned<float> data;         // [rows_total, dim], list-major, zero padding rows
  owned<int64_t> ids;        // [rows_total], kPadId on padding rows
  owned<float> xn;           // [rows_total] |x|^2 (the exact re-score)
  owned<float> rn;           // [rows_total] |x - c|^2 of the residual rows below
  owned<__nv_bfloat16> hi;   // [rows_total, Kp] bf16 residuals x - c of each row's list centre (cosine: x/|x| - c/|c|)
  owned<__nv_bfloat16> hx;   // [rows_total, 16] half-norm plane: |x - c|^2/2 (0 for inner product), +inf on padding rows (scan_tc.cuh)
  // (cosine is scanned as L2 over the unit vectors, 2 - 2 q.x = |q - x|^2: the error then follows |q - c|, not |q| = 1)
  owned<float> rn_max;       // [n_lists] max |x - c|^2 over the list's rows (the certificate's error budget)
  owned<float> cn;           // [n_lists] |c|^2 of the fp32 centres (the inner-product budget)
  int Kp = 0;
  // 8-bit lists (row_type s8 / u8; DESIGN.md §4 "Row types"): data, hi, hx, xn, rn and rn_max stay empty
  row_type type = row_type::f32;
  owned<uint8_t> rows8;      // [rows_total, Kp8] the rows' bytes, zero padding rows and columns
  owned<int> norms8;         // [rows_total] exact |x|^2, kI8PadNorm on padding rows
  int Kp8 = 0;
};

namespace {

// How an index stores its list rows: fp32 (float32 and float16 datasets, and cosine on 8-bit ones), or the 8-bit rows themselves.
row_type row_type_for(DLDataType t, cuvsDistanceType metric)
{
  const row_type rt = row_type_of(t);
  if (metric == CosineExpanded || row_bytes(rt) != 1) return row_type::f32;  // a cosine distance is no integer function of the rows
  return rt;
}

// 8-bit rows from a widened chunk x (integer values as fp32): one thread per byte of a padded row, written to row dst_rows[r]
__global__ void narrow_rows_kernel(const float* __restrict__ x, int64_t n, int dim, int Kp8, const int64_t* __restrict__ dst_rows,
                                   uint8_t* __restrict__ out)
{
  const int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (t >= n * Kp8) return;
  const int64_t r = t / Kp8;
  const int j     = static_cast<int>(t % Kp8);
  const int64_t o = dst_rows[r];
  if (o < 0) return;
  out[o * Kp8 + j] = j < dim ? static_cast<uint8_t>(static_cast<int>(x[r * dim + j])) : uint8_t(0);
}

// The A rows of an 8-bit scan: the bytes of each pair slot's query (slots past the live pairs: zero), 16 per thread
__global__ void pair_query_bytes_kernel(const float* __restrict__ q, int dim, int Kp8, const uint32_t* __restrict__ pair_query,
                                        const int* __restrict__ n_live, int64_t rows, uint8_t* __restrict__ out)
{
  const int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int w     = Kp8 / 16;
  if (t >= rows * w) return;
  const int64_t slot = t / w;
  const int j0       = static_cast<int>(t % w) * 16;
  uint32_t v[4]      = {0, 0, 0, 0};
  if (slot < *n_live) {
    const float* qr = q + static_cast<int64_t>(pair_query[slot]) * dim;
#pragma unroll
    for (int b = 0; b < 16; ++b)
      if (j0 + b < dim) v[b >> 2] |= (static_cast<uint32_t>(static_cast<int>(qr[j0 + b])) & 0xffu) << (8 * (b & 3));
  }
  reinterpret_cast<uint4*>(out)[t] = make_uint4(v[0], v[1], v[2], v[3]);
}

// exact |q|^2 of a query row holding integer values; every thread of the block calls it and gets the sum
__device__ int block_query_norm(const float* __restrict__ qr, int dim)
{
  __shared__ int part[32];
  int acc = 0;
  for (int j = threadIdx.x; j < dim; j += blockDim.x) {
    const int v = static_cast<int>(qr[j]);
    acc += v * v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  int total = 0;
  for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) total += part[w];
  return total;
}

// a merged candidate that names a row: not an empty slot (FLT_MAX or +inf, position 0xffffffff) nor a row the filter hid (+inf)
__device__ __forceinline__ bool i8_live(float key, uint32_t pos) { return pos != 0xffffffffu && __float_as_uint(key) < 0x7f000000u; }
// the exact distance of a key's score s, rounded once: |q - x|^2 = s + |q|^2 (L2), q.x = -s (inner product)
__device__ __forceinline__ float i8_distance(float key, int qn, bool ip)
{
  const int s = tc_i8_score(key);
  return ip ? __int2float_rn(-s) : __int2float_rn(s + qn);
}

// 8-bit search, one block per query: its kc2 merged candidates (key, position), sorted by key, give the k best by (distance, id).
// Equal keys are equal distances, so a candidate's rank is the number of candidates ahead of its run of equal keys plus the
// members of the run with a smaller id.  Missing slots: (INT64_MAX, +-FLT_MAX).
__global__ void i8_finish_kernel(const float* __restrict__ ms, const uint32_t* __restrict__ mp, int kc2, const int64_t* __restrict__ ids,
                                 const float* __restrict__ q, int dim, bool ip, int k, int64_t* __restrict__ out_idx,
                                 float* __restrict__ out_dist)
{
  const int64_t qi    = blockIdx.x;
  const int qn        = block_query_norm(q + qi * dim, dim);
  const float* key    = ms + qi * kc2;
  const uint32_t* pos = mp + qi * kc2;
  for (int j = threadIdx.x; j < k; j += blockDim.x) {
    out_idx[qi * k + j]  = INT64_MAX;
    out_dist[qi * k + j] = ip ? -FLT_MAX : FLT_MAX;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < kc2; j += blockDim.x) {
    const float kj = key[j];
    if (!i8_live(kj, pos[j])) continue;
    const int64_t id = ids[pos[j]];
    int lo = j;
    while (lo > 0 && key[lo - 1] == kj) --lo;
    int rank = lo;
    for (int i = lo; i < kc2 && key[i] == kj && rank < k; ++i)
      if (i != j && i8_live(key[i], pos[i]) && ids[pos[i]] < id) ++rank;
    if (rank >= k) continue;
    out_idx[qi * k + rank]  = id;
    out_dist[qi * k + rank] = i8_distance(kj, qn, ip);
  }
}

// cuvsB200IvfFlatCandidates on an 8-bit index: the kc2 merged candidates with their exact distances in the scan's units
// (|q - x|^2, or -q.x) and, as their bound, half an ulp of that distance, the only error left being its rounding to fp32.
__global__ void i8_candidates_kernel(const float* __restrict__ ms, const uint32_t* __restrict__ mp, int kc2, const int64_t* __restrict__ ids,
                                     const float* __restrict__ q, int dim, bool ip, int64_t* __restrict__ out_ids,
                                     float* __restrict__ out_dist, float* __restrict__ out_bound)
{
  const int64_t qi = blockIdx.x;
  const int qn     = block_query_norm(q + qi * dim, dim);
  for (int j = threadIdx.x; j < kc2; j += blockDim.x) {
    const int64_t i = qi * kc2 + j;
    const bool live = i8_live(ms[i], mp[i]);
    const float d   = live ? i8_distance(ms[i], qn, ip) : INFINITY;
    out_ids[i]      = live ? ids[mp[i]] : INT64_MAX;
    out_dist[i]     = ip && live ? -d : d;
    out_bound[i]    = live ? fmaxf(fabsf(d), 1.f) * 0x1p-24f : INFINITY;
  }
}

// The centres the scan's residuals are taken from: the unit centres for cosine (the rows and queries are unit there too).
const float* residual_centers(const ivf_flat_index& idx)
{
  return idx.metric == CosineExpanded ? idx.centers_unit.data() : idx.centers.data();
}
// The metric the scan ranks by: cosine ranks as L2 over unit vectors.
cuvsDistanceType scan_metric(const ivf_flat_index& idx) { return idx.metric == CosineExpanded ? L2Expanded : idx.metric; }
// The metric the exact re-score computes: the reference's fine-scan arithmetic, sum (q - x)^2, for every L2 metric.
cuvsDistanceType fine_metric(const ivf_flat_index& idx) { return is_ip(idx.metric) ? idx.metric : L2Unexpanded; }

// One warp per list row: hi = bf16(x * scale - c_l) and rn = |x * scale - c_l|^2 (fp32), with l the row's list (the last with
// offsets[l] <= row) and scale = row_scale[row] (null: 1).  Padding rows get a zero residual.
__global__ void residual_rows_kernel(const float* __restrict__ x, const int64_t* __restrict__ ids, const float* __restrict__ row_scale,
                                     int64_t rows, int dim, int Kp, const float* __restrict__ centers,
                                     const int64_t* __restrict__ offsets, int64_t n_lists, __nv_bfloat16* __restrict__ hi,
                                     float* __restrict__ rn)
{
  const int64_t r = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
  const int lane  = threadIdx.x & 31;
  if (r >= rows) return;
  const bool pad = ids[r] == kPadId;
  int64_t lo = 0, up = n_lists;
  while (up - lo > 1) {
    const int64_t mid = (lo + up) >> 1;
    if (offsets[mid] <= r) lo = mid;
    else up = mid;
  }
  const float sc  = row_scale ? row_scale[r] : 1.f;
  const float* xr = x + r * dim;
  const float* cr = centers + lo * dim;
  float nrm       = 0.f;
  for (int j = lane; j < Kp; j += 32) {
    const float v = (!pad && j < dim) ? xr[j] * sc - cr[j] : 0.f;
    hi[r * Kp + j] = __float2bfloat16_rn(v);
    nrm            = fmaf(v, v, nrm);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) nrm += __shfl_xor_sync(0xffffffffu, nrm, o);
  if (lane == 0) rn[r] = nrm;
}

__global__ void half_norms_masked_kernel(const float* __restrict__ xn, const int64_t* __restrict__ ids, int64_t n, bool zero,
                                         float* __restrict__ hn)
{
  int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  hn[i] = ids[i] == kPadId ? INFINITY : (zero ? 0.f : 0.5f * xn[i]);
}

// same, additionally hiding every row whose source id is not kept by the bitset (bit = 1 keeps): the filtered search
// scans against this temporary plane, so excluded rows score -inf inside the tensor-core kernel and can never be candidates
__global__ void half_norms_filtered_kernel(const float* __restrict__ xn, const int64_t* __restrict__ ids, int64_t n, bool zero,
                                           const uint32_t* __restrict__ bits, int64_t n_bits, float* __restrict__ hn)
{
  int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const int64_t id = ids[i];
  const bool keep  = id >= 0 && id < n_bits && ((bits[id >> 5] >> (id & 31)) & 1u);
  hn[i]            = keep ? (zero ? 0.f : 0.5f * xn[i]) : INFINITY;
}

// k > 64: candidates whose scan score is not finite (rows hidden by the filter) become empty slots of the re-score
__global__ void drop_nonfinite_kernel(const float* __restrict__ score, uint32_t* __restrict__ pos, int64_t n)
{
  int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i < n && !isfinite(score[i])) pos[i] = 0xffffffffu;
}

// rn_max[l] = max of rn over the rows of list l (padding rows hold 0); one warp per list
__global__ void list_max_kernel(const float* __restrict__ rn, const int64_t* __restrict__ offsets, int64_t n_lists, float* __restrict__ out)
{
  const int64_t l = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
  const int lane  = threadIdx.x & 31;
  if (l >= n_lists) return;
  float m = 0.f;
  for (int64_t r = offsets[l] + lane; r < offsets[l + 1]; r += 32) m = fmaxf(m, rn[r]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) out[l] = m;
}

// Error budget of the fine scan's approximate distance A = add + scale * score of a row x of a pair (q, list l) against the
// exact fp32 distance F the re-score computes, in A's units (DESIGN.md §4, "Certificate").  Q = |q - c| (inner product: |q|),
// R = max |x - c| over the list (rn_max), C = |c|:
//   bf16 rounding of both residual rows        scale (2^-8 + 2^-16) Q R
//   fp32 tensor-core accumulation over Kp + 16  scale (Kp + 20) 2^-22 (1.01 Q R + hn), hn = R^2 / 2 (L2, cosine) or 0
//   fp32 rounding of add, rn, the sum and F     (2 dim + 16) 2^-23 (Q + R)^2, inner product (2 dim + 16) 2^-23 Q (2 C + R)
//   cosine: unit rows and queries vs the exact  (2 dim + 16) 2^-21
//     1 - q.x / (|q| |x|), taken twice
// Each term bounds its rounding step as documented; how the MMA orders and rounds its fp32 sums inside one instruction is not,
// so the budget is checked against the errors the scan makes (tests/test_ivf_flat_near_duplicates_gpu.py::budget_ratio,
// DESIGN.md §4): they stay below 0.4 of it, and below 0.25 except where a row nearly repeats the query.
struct flat_budget {
  float c_bf, c_acc, c_fp, c_abs;
  bool ip;
  __device__ float eps(float Q, float R, float C) const
  {
    if (ip) return (c_bf + 1.01f * c_acc) * Q * R + c_fp * Q * (2.f * C + R);
    return c_bf * Q * R + c_acc * (1.01f * Q * R + 0.5f * R * R) + c_fp * (Q + R) * (Q + R) + c_abs;
  }
};

flat_budget make_budget(const ivf_flat_index& idx, float scale)
{
  flat_budget b;
  b.ip    = idx.metric == InnerProduct;
  b.c_bf  = scale * (1.f / 256.f + 1.f / 65536.f);
  b.c_acc = scale * static_cast<float>(idx.Kp + 20) * (1.f / 4194304.f);
  b.c_fp  = static_cast<float>(2 * idx.dim + 16) * (1.f / 8388608.f);
  b.c_abs = idx.metric == CosineExpanded ? 4.f * b.c_fp : 0.f;
  return b;
}

// The certificate (DESIGN.md §4).  Every row of the query's probed lists that is not among its kc2 merged candidates has A at
// least `floor`, the minimum of
//   * the kc2-th merged candidate (ms, sorted), for the rows the merge dropped;
//   * the last entry of every full per-pair list (a column half of KC, or a pair's segment of kc2 at k > 64), for the rows a
//     list dropped: last[q, p * nl + j] for list j of probe p (gather_probe_candidates), +inf where a list is not full;
// and the rows the shared pruning bound rejected score above some full list's L-th entry, hence above `floor` too.  Such a row
// has F >= floor - eps, so when the exact k-th distance (kth, in A's units) is strictly below floor - eps no row outside can
// enter the top k, and the re-score of the candidates is the oracle's answer.  eps is the largest budget of the query's pairs,
// except pairs whose every row is provably farther than kth (triangle inequality: |q - x| >= Q - R, or -q.x >= add - Q R).
// Otherwise the query is flagged (flags[nq] counts them).  One warp per query, its lanes over the probes.
__global__ void certify_kernel(const float* __restrict__ out_dist, int k, int fine, const float* __restrict__ ms, int kc2,
                               const float* __restrict__ last, int nl, const uint32_t* __restrict__ probes,
                               const uint32_t* __restrict__ slot_of, int n_probes, const float* __restrict__ add,
                               const float* __restrict__ qn, const float* __restrict__ rn_max, const float* __restrict__ cn,
                               flat_budget bud, int64_t nq, int* __restrict__ flags)
{
  const int64_t q = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
  const int lane  = threadIdx.x & 31;
  if (q >= nq) return;
  const float kd = out_dist[q * k + k - 1];
  // the exact k-th distance in A's units; a missing k-th neighbour (+-FLT_MAX) is FLT_MAX
  const float kth = fine == InnerProduct ? -kd : (fine == CosineExpanded && kd < FLT_MAX ? 2.f * kd : kd);
  float floor     = lane == 0 ? ms[q * kc2 + kc2 - 1] : INFINITY;
  float eps       = 0.f;
  const float qi  = bud.ip ? sqrtf(qn[q]) : 0.f;
  for (int p = lane; p < n_probes; p += 32) {
    const uint32_t slot = slot_of[q * n_probes + p];
    if (slot == 0xffffffffu) continue;
    const float* g = last + (q * n_probes + p) * nl;
    for (int j = 0; j < nl; ++j) floor = fminf(floor, g[j]);
    const float a    = add[slot];
    const uint32_t l = probes[q * n_probes + p];
    const float R    = sqrtf(rn_max[l]);
    const float Q    = bud.ip ? qi : sqrtf(fmaxf(a, 0.f));
    const float e_p  = bud.eps(Q, R, bud.ip ? sqrtf(cn[l]) : 0.f);
    const float lower = bud.ip ? a - Q * R - e_p : (Q > R ? (Q - R) * (Q - R) - e_p : -INFINITY);
    if (lower > kth) continue;
    eps = fmaxf(eps, e_p);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    floor = fminf(floor, __shfl_xor_sync(0xffffffffu, floor, o));
    eps   = fmaxf(eps, __shfl_xor_sync(0xffffffffu, eps, o));
  }
  if (lane != 0) return;
  const int flag = kth < floor - eps ? 0 : 1;
  flags[q]       = flag;
  if (flag) atomicAdd(flags + nq, 1);
}

__device__ __forceinline__ bool row_kept(int64_t id, const uint32_t* __restrict__ keep_bits, int64_t n_bits)
{
  return id != kPadId && (keep_bits == nullptr || (id >= 0 && id < n_bits && ((keep_bits[id >> 5] >> (id & 31)) & 1u)));
}

// k <= 64: the exact fallback on the device, the CTAs taking the queries in turn; they pass over a query the certificate
// accepted, so the search needs no host round trip.  A flagged query scores every row of its probed lists exactly, negated for
// inner product so that smaller is better.  Rows better than the running k-th best (distance, id) collect in shared memory,
// which is sorted and cut back to k whenever it may overflow; the k best by (distance, id), rescore_topk's ranking, overwrite
// the query's output row (selection form; missing: pad id and +-FLT_MAX).
constexpr int kFbThreads = 256, kFbCap = 1024;
__global__ void __launch_bounds__(kFbThreads)
exact_fallback_kernel(const int* __restrict__ flags, const uint32_t* __restrict__ probes, int n_probes, const int64_t* __restrict__ offsets,
                      const float* __restrict__ q, int dim, const float* __restrict__ x, const float* __restrict__ qn,
                      const float* __restrict__ xn, const int64_t* __restrict__ ids, int fine, const uint32_t* __restrict__ keep_bits,
                      int64_t n_bits, int k, int64_t nq, int64_t* __restrict__ out_idx, float* __restrict__ out_dist)
{
  __shared__ float sd[kFbCap];
  __shared__ int64_t si[kFbCap];
  __shared__ int cnt;
  __shared__ float thr_d;
  __shared__ int64_t thr_i;
  const bool ip = fine == InnerProduct;
  auto compact = [&]() {  // sort the cnt entries by (distance, id), keep the k best and their k-th as the threshold
    const int n = cnt;
    for (int i = n + threadIdx.x; i < kFbCap; i += kFbThreads) { sd[i] = INFINITY; si[i] = INT64_MAX; }
    __syncthreads();
    block_bitonic_sort(sd, si, nullptr, kFbCap, [&](int a, int b) { return sd[a] < sd[b] || (sd[a] == sd[b] && si[a] < si[b]); });
    if (threadIdx.x == 0) {
      cnt = min(n, k);
      if (n >= k) { thr_d = sd[k - 1]; thr_i = si[k - 1]; }
    }
    __syncthreads();
  };
  for (int64_t qi = blockIdx.x; qi < nq; qi += gridDim.x) {
    if (!flags[qi]) continue;
    __syncthreads();  // the previous query's rows are written
    if (threadIdx.x == 0) { cnt = 0; thr_d = INFINITY; thr_i = INT64_MAX; }
    __syncthreads();
    const float* qr = q + qi * dim;
    for (int p = 0; p < n_probes; ++p) {
      const uint32_t l = probes[qi * n_probes + p];
      if (l == 0xffffffffu) continue;
      const int64_t r1 = offsets[l + 1];
      for (int64_t base = offsets[l]; base < r1; base += kFbThreads) {
        const int64_t r = base + threadIdx.x;
        if (r < r1) {
          const int64_t id = ids[r];
          if (row_kept(id, keep_bits, n_bits)) {
            // scalar reads: the float4 form makes this kernel spill, and both give the same bits
            const float e = finish_distance(exact_accumulate(qr, x + r * dim, dim, false, fine), qn[qi], xn[r], fine);
            const float d = ip ? -e : e;
            if (d < thr_d || (d == thr_d && id < thr_i)) {
              const int at = atomicAdd(&cnt, 1);
              sd[at] = d;
              si[at] = id;
            }
          }
        }
        __syncthreads();
        const bool full = cnt > kFbCap - kFbThreads;  // every thread reads it before any adds to it again
        __syncthreads();
        if (full) compact();
      }
    }
    compact();
    for (int j = threadIdx.x; j < k; j += kFbThreads) {
      const bool have     = j < cnt;
      out_idx[qi * k + j]  = have ? si[j] : INT64_MAX;
      out_dist[qi * k + j] = have ? (ip ? -sd[j] : sd[j]) : (ip ? -FLT_MAX : FLT_MAX);
    }
  }
}

// k > 64: the exact fallback's scan.  The score of every (pair, list row) is the row's exact distance (negated for inner
// product), so the segmented select keeps each pair's k best by the very value the re-score recomputes.  Padding rows and rows
// the bitset hides score +inf.  One CTA per live pair slot, one thread per row.
__global__ void exact_segments_kernel(const float* __restrict__ q, int dim, const float* __restrict__ x, const float* __restrict__ qn,
                                      const float* __restrict__ xn, const int64_t* __restrict__ ids, int fine,
                                      const uint32_t* __restrict__ pair_query, const uint32_t* __restrict__ pair_list,
                                      const int* __restrict__ n_live, const int64_t* __restrict__ offsets,
                                      const int64_t* __restrict__ seg_off, const uint32_t* __restrict__ keep_bits, int64_t n_bits,
                                      float* __restrict__ scores)
{
  const int64_t slot = blockIdx.x;
  if (slot >= *n_live) return;
  const int64_t qi = pair_query[slot];
  const uint32_t l = pair_list[slot];
  const float* qr  = q + qi * dim;
  float* out       = scores + seg_off[slot];
  const bool vec4  = exact_vec4(q, dim, x, dim, dim);
  for (int64_t r = offsets[l] + threadIdx.x; r < offsets[l + 1]; r += blockDim.x) {
    if (!row_kept(ids[r], keep_bits, n_bits)) { out[r - offsets[l]] = INFINITY; continue; }
    const float v = finish_distance(exact_accumulate(qr, x + r * dim, dim, vec4, fine), qn[qi], xn[r], fine);
    out[r - offsets[l]] = fine == InnerProduct ? -v : v;
  }
}

// cuvsB200IvfFlatCandidates: per merged candidate (q, c) at index row pos, its source id (INT64_MAX for an empty slot) and the
// budget of its own pair, the probe of q whose list holds the row (flat_budget::eps, as certify_kernel takes it).
__global__ void candidate_budget_kernel(const uint32_t* __restrict__ pos, const int64_t* __restrict__ src_ids,
                                        const int64_t* __restrict__ offsets, int64_t n_lists, const uint32_t* __restrict__ probes,
                                        const uint32_t* __restrict__ slot_of, int n_probes, int kc2, const float* __restrict__ add,
                                        const float* __restrict__ qn, const float* __restrict__ rn_max, const float* __restrict__ cn,
                                        flat_budget bud, int64_t n, int64_t* __restrict__ ids, float* __restrict__ bound)
{
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const uint32_t r = pos[i];
  ids[i]           = r == 0xffffffffu ? INT64_MAX : src_ids[r];
  float eps        = INFINITY;
  if (r != 0xffffffffu) {
    int64_t lo = 0, up = n_lists;  // the list holding row r: the last with offsets[l] <= r
    while (up - lo > 1) {
      const int64_t mid = (lo + up) >> 1;
      if (offsets[mid] <= r) lo = mid;
      else up = mid;
    }
    const int64_t q = i / kc2;
    for (int p = 0; p < n_probes; ++p) {
      const uint32_t slot = slot_of[q * n_probes + p];
      if (slot == 0xffffffffu || probes[q * n_probes + p] != static_cast<uint32_t>(lo)) continue;
      const float Q = bud.ip ? sqrtf(qn[q]) : sqrtf(fmaxf(add[slot], 0.f));
      eps           = bud.eps(Q, sqrtf(rn_max[lo]), bud.ip ? sqrtf(cn[lo]) : 0.f);
    }
  }
  bound[i] = eps;
}

// The scan's side of the list rows (DESIGN.md §4): bf16 residuals against the row's list centre and their half norms.  Rebuilt
// whenever the rows change (extend, load); the centres change only while the index is empty.
void refresh_tc_side(resources* res, ivf_flat_index& idx)
{
  auto s          = res->stream;
  const int64_t R = idx.lists.rows_total;
  idx.Kp          = tc_pad_k(idx.dim);
  idx.hi.alloc(static_cast<size_t>(std::max<int64_t>(R, 128)) * idx.Kp);
  idx.hx.alloc(static_cast<size_t>(std::max<int64_t>(R, 128)) * 16);
  idx.xn.alloc(static_cast<size_t>(std::max<int64_t>(R, 128)));
  idx.rn.alloc(static_cast<size_t>(std::max<int64_t>(R, 128)));
  idx.rn_max.alloc(static_cast<size_t>(idx.n_lists));
  B2_CUDA(cudaMemsetAsync(idx.rn_max.data(), 0, sizeof(float) * idx.n_lists, s));
  if (R == 0) return;
  row_norms(s, idx.data.data(), R, idx.dim, idx.dim, idx.xn.data());
  dbuf<float> scale;
  if (idx.metric == CosineExpanded) {
    scale.alloc(static_cast<size_t>(R), s);
    rsqrt_rows(s, idx.xn.data(), R, scale.data());
  }
  count_launch(2);
  residual_rows_kernel<<<blocks_for(R * 32, 256), 256, 0, s>>>(idx.data.data(), idx.ids.data(), scale.data(), R, idx.dim, idx.Kp,
                                                                residual_centers(idx), idx.lists.d_offsets.data(), idx.n_lists,
                                                                idx.hi.data(), idx.rn.data());
  dbuf<float> hn(static_cast<size_t>(R), s);
  half_norms_masked_kernel<<<blocks_for(R, 256), 256, 0, s>>>(idx.rn.data(), idx.ids.data(), R, !is_l2(scan_metric(idx)), hn.data());
  count_launch();
  list_max_kernel<<<blocks_for(idx.n_lists * 32, 256), 256, 0, s>>>(idx.rn.data(), idx.lists.d_offsets.data(), idx.n_lists, idx.rn_max.data());
  B2_CUDA(cudaGetLastError());
  tc_pack_half_norms(s, hn.data(), R, idx.hx.data());
}

// The scan's side of 8-bit list rows: their exact norms (kI8PadNorm on padding rows).  Rebuilt whenever the rows change.
void refresh_i8_side(resources* res, ivf_flat_index& idx)
{
  const int64_t R = idx.lists.rows_total;
  idx.norms8.alloc(static_cast<size_t>(std::max<int64_t>(R, 128)));
  if (R == 0) return;
  tc_i8_norms(res->stream, idx.type == row_type::u8, idx.rows8.data(), R, R, idx.Kp8, idx.ids.data(), nullptr, 0, idx.norms8.data());
}

void refresh_centers_tc(resources* res, ivf_flat_index& idx)
{
  auto s = res->stream;
  idx.cn.alloc(static_cast<size_t>(idx.n_lists));
  float* cn = idx.cn.data();
  row_norms(s, idx.centers.data(), idx.n_lists, idx.dim, idx.dim, cn);
  dbuf<float> scale;
  if (idx.metric == CosineExpanded) {
    scale.alloc(static_cast<size_t>(idx.n_lists), s);
    rsqrt_rows(s, cn, idx.n_lists, scale.data());
    idx.centers_unit.alloc(static_cast<size_t>(idx.n_lists) * idx.dim);
    B2_CUDA(cudaMemcpyAsync(idx.centers_unit.data(), idx.centers.data(), sizeof(float) * idx.n_lists * idx.dim, cudaMemcpyDeviceToDevice, s));
    normalize_rows(s, idx.centers_unit.data(), idx.n_lists, idx.dim, idx.dim);
  }
  idx.centers_tc.build(s, idx.centers.data(), idx.n_lists, idx.dim, is_l2(idx.metric) ? cn : nullptr, true, scale.data());
}

// Insert the rows of `t` ([n, dim], device or host: fp32, or int8 / uint8 for an index of that row type) with ids new_ids[i]
// (device) or id0 + i, then refresh the derived rows once.  A cosine row is labelled from its unit bf16 planes, as a cosine
// query is in the coarse search.  8-bit rows are labelled from a widened chunk at a time and stored as bytes.
void ivf_flat_extend(resources* res, ivf_flat_index& idx, const DLTensor& t, const int64_t* new_ids, int64_t id0)
{
  auto s = res->stream;
  if (t.shape[0] == 0) return;
  auto label = [&](const float* x, int64_t n, uint32_t* labels) {
    tc_rows_tmp xp;
    dbuf<float> scale;
    if (idx.metric == CosineExpanded) {
      dbuf<float> xn(static_cast<size_t>(n), s);
      row_norms(s, x, n, idx.dim, idx.dim, xn.data());
      scale.alloc(static_cast<size_t>(n), s);
      rsqrt_rows(s, xn.data(), n, scale.data());
    }
    xp.build(s, x, n, idx.dim, true, 0, scale.data());
    assign_nearest(res, xp.hi.data(), xp.lo.data(), n, xp.rows_pad, xp.Kp, idx.centers_tc, labels, nullptr);
  };
  auto write = [&](const float* x, int64_t n, uint32_t*, const int64_t* dst_rows, float* data) {
    scatter_rows(s, x, n, int64_t(idx.dim), dst_rows, data);
  };
  if (idx.type != row_type::f32) {
    auto write8 = [&](const float* x, int64_t n, uint32_t*, const int64_t* dst_rows, uint8_t* rows) {
      count_launch();
      narrow_rows_kernel<<<blocks_for(n * idx.Kp8, 256), 256, 0, s>>>(x, n, idx.dim, idx.Kp8, dst_rows, rows);
      B2_CUDA(cudaGetLastError());
    };
    insert_rows<uint8_t>(res, t, idx.lists, idx.rows8, idx.Kp8, idx.ids, new_ids, id0, label, write8);
    refresh_i8_side(res, idx);
    return;
  }
  insert_rows<float>(res, t, idx.lists, idx.data, idx.dim, idx.ids, new_ids, id0, label, write);
  refresh_tc_side(res, idx);
}

// The derived rows of the index's row type
void refresh_rows(resources* res, ivf_flat_index& idx)
{
  if (idx.type != row_type::f32) refresh_i8_side(res, idx);
  else refresh_tc_side(res, idx);
}

ivf_flat_index* ivf_flat_build(resources* res, const cuvsIvfFlatIndexParams& p, const DLTensor& ds)
{
  B2_EXPECTS(ds.ndim == 2, "dataset must be a 2-D tensor");
  B2_EXPECTS(dl_is_c_contiguous(ds), "dataset must be row-major contiguous");
  B2_EXPECTS(is_l2(p.metric) || p.metric == InnerProduct || p.metric == CosineExpanded, "ivf_flat: unsupported metric %d", int(p.metric));
  const int64_t n = ds.shape[0];
  const int d     = static_cast<int>(ds.shape[1]);
  B2_EXPECTS(n >= 1 && d >= 1, "empty dataset");
  B2_EXPECTS(p.n_lists >= 1 && static_cast<int64_t>(p.n_lists) <= n, "n_lists (%u) must be in [1, n_rows]", p.n_lists);
  B2_EXPECTS(tc_supported(res->device, d), "ivf_flat: dim %d is not supported: it pads to more than %d columns, the widest the tensor-core kernels take", d, kTcMaxK);
  auto idx               = std::make_unique<ivf_flat_index>();
  idx->device            = res->device;
  idx->metric            = p.metric;
  idx->metric_arg        = p.metric_arg;
  idx->dim               = d;
  idx->n_lists           = p.n_lists;
  idx->adaptive_centers  = p.adaptive_centers;
  idx->kmeans_n_iters    = p.kmeans_n_iters;
  idx->kmeans_trainset_fraction = p.kmeans_trainset_fraction;
  idx->type              = row_type_for(ds.dtype, p.metric);
  idx->Kp8               = tc_pad_k_i8(d);
  B2_EXPECTS(idx->type != row_type::f32 || dl_is(ds, kDLFloat, 32), "ivf_flat_build: float16 rows, and 8-bit rows of a cosine index, must be widened to float32 first");
  auto s = res->stream;

  int64_t n_train   = 0;
  dbuf<float> train = train_subsample(s, ds, p.n_lists, p.kmeans_trainset_fraction, n_train);
  idx->centers.alloc(static_cast<size_t>(p.n_lists) * d);
  kmeans_train(res, train.data(), n_train, d, p.n_lists, std::max<uint32_t>(p.kmeans_n_iters, 1), idx->centers.data(), true, true,
               nullptr, nullptr);
  refresh_centers_tc(res, *idx);
  std::vector<int64_t> zero(p.n_lists, 0);
  idx->lists.set_sizes(s, zero);
  if (p.add_data_on_build) ivf_flat_extend(res, *idx, ds, nullptr, 0);
  else refresh_rows(res, *idx);
  return idx.release();
}

// The merged candidates of a search and their error budget, as the certificate sees them (cuvsB200IvfFlatCandidates).
struct flat_candidates {
  int64_t* ids;  // [nq, kc2]
  float* dist;   // [nq, kc2] approximate distance, add + scale * score
  float* bound;  // [nq, kc2] error budget of each candidate's own pair
};

// k > 64: the exact fallback.  The k > 64 steps with exact scores over the lists the nq queries q probe (probes [nq, n_probes],
// the search's own: its coarse selection is exact per query), written postprocessed to out_idx / out_dist [nq, k].  A query's
// workspace here (kc = k) is no larger than in the search (kc = min(2k, 2048)), so the flagged queries of a batch fit its budget.
void exact_probed_search(resources* res, const ivf_flat_index& idx, const float* q, int64_t nq, const uint32_t* probes,
                         uint32_t n_probes, const uint32_t* keep_bits, int64_t n_bits, int k, int64_t* out_idx, float* out_dist)
{
  auto s                     = res->stream;
  const cuvsDistanceType fine = fine_metric(idx);
  dbuf<float> qn(static_cast<size_t>(nq), s);
  row_norms(s, q, nq, idx.dim, idx.dim, qn.data());
  probe_buckets pb;
  bucket_probes(res, probes, nq, static_cast<int>(n_probes), idx.n_lists, idx.lists.d_offsets.data(), 0, pb);
  dbuf<float> cs;
  dbuf<uint32_t> cp;
  large_k_select(s, pb, idx.lists, nq, n_probes, k, [&](float* scores, const int64_t* seg_off) {
    count_launch();
    exact_segments_kernel<<<static_cast<unsigned>(std::max<int64_t>(pb.n_pairs, 1)), 128, 0, s>>>(
      q, idx.dim, idx.data.data(), qn.data(), idx.xn.data(), idx.ids.data(), int(fine), pb.pair_query.data(), pb.pair_list.data(),
      pb.n_items.data() + 1, idx.lists.d_offsets.data(), seg_off, keep_bits, n_bits, scores);
    B2_CUDA(cudaGetLastError());
  }, cs, cp);
  const int64_t cand_w = static_cast<int64_t>(n_probes) * k;
  dbuf<float> gs(static_cast<size_t>(nq) * cand_w, s);
  dbuf<uint32_t> gp(static_cast<size_t>(nq) * cand_w, s);
  gather_probe_candidates(s, cs.data(), cp.data(), pb.slot_of.data(), nullptr, 1.f, INFINITY, nq, static_cast<int>(n_probes), k,
                          gs.data(), gp.data());
  dbuf<float> ms(static_cast<size_t>(nq) * k, s);
  dbuf<uint32_t> mp(static_cast<size_t>(nq) * k, s);
  select_k(s, gs.data(), gp.data(), IDX_U32, nq, cand_w, cand_w, k, ms.data(), mp.data(), IDX_U32, true);
  count_launch();
  drop_nonfinite_kernel<<<blocks_for(nq * k, 256), 256, 0, s>>>(ms.data(), mp.data(), nq * k);
  B2_CUDA(cudaGetLastError());
  rescore_topk(s, q, nq, idx.dim, idx.data.data(), idx.dim, idx.dim, qn.data(), idx.xn.data(), fine, mp.data(), k, idx.ids.data(), k,
               out_idx, out_dist, INT64_MAX);
  postprocess_distances(s, out_dist, nq * k, idx.metric);
}

// Search of an 8-bit index (DESIGN.md §4 "Row types").  q [nq, dim] fp32 holds the queries' integer values.  The coarse search
// is the fp32 one; the fine scan multiplies the pairs' query bytes with the list bytes on the integer tensor cores and ranks by
// exact keys (tc_i8_key), so the merged candidates are the exact best of the probed lists: no re-score, no certificate.
//   want <= 16 (32 at Kp8 = 128): the fused epilogue, lists of KC >= want per column half; each holds every row of its half
//   that can be among the query's want best, and the shared pruning bound stops at each list's want-th key.
//   otherwise: the store scan and the segmented select keep each pair's want best, which hold the query's want best.
// want is k, or the kc2 candidates cuvsB200IvfFlatCandidates asks for (dump).
void ivf_flat_search_i8(resources* res, const ivf_flat_index& idx, uint32_t n_probes, const DLTensor& qt, const DLTensor& nt,
                        const DLTensor& dt, const uint32_t* keep_bits, int64_t n_bits, const flat_candidates* dump)
{
  auto s           = res->stream;
  const int64_t nq = qt.shape[0];
  const int k      = static_cast<int>(nt.shape[1]);
  const int want   = dump ? std::max(32, 2 * k) : k;
  const int KC     = want <= 16 ? 16 : (want <= 32 && idx.Kp8 == 128 ? 32 : 0);
  // Query batching.  Per pair: its query bytes, the bound slot, 2 x KC candidates (score, position) and their per-query gather.
  // Store scan, per query: dense scores over its n_probes largest lists, each pair's want best and their gather (16 bytes each),
  // pair bookkeeping, and the merged want.
  const int64_t store_bytes = KC != 0 ? 0
                                      : large_k_rows_per_query(idx.lists, n_probes) * 4 +
                                          static_cast<int64_t>(n_probes) * (16 * want + idx.Kp8 + 32) + static_cast<int64_t>(want) * 8;
  const int64_t batch = query_batch_size(idx.Kp8 + 4 + 2 * 32 * 8 + 16, n_probes, store_bytes, "CUVS_B200_FLAT_LARGE_K_BUDGET_MB");
  B2_EXPECTS(dump == nullptr || nq <= batch, "ivf_flat candidates: %lld queries do not fit one batch", (long long)nq);
  if (search_in_batches(batch, qt, nt, dt, [&](const DLTensor& qs, const DLTensor& ns, const DLTensor& ds) {
        ivf_flat_search_i8(res, idx, n_probes, qs, ns, ds, keep_bits, n_bits, nullptr);
      }))
    return;
  const float* q   = dl_ptr<float>(qt);
  const bool ip    = idx.metric == InnerProduct;

  // ---- 1. coarse (as for fp32 rows)
  tc_rows_tmp qp;
  qp.build(s, q, nq, idx.dim, true, 0, nullptr);
  dbuf<uint32_t> probes(static_cast<size_t>(nq) * n_probes, s);
  coarse_select(res, qp, idx.centers_tc, static_cast<int>(n_probes), probes.data(), nullptr);

  // ---- 1b. bitset pre-filter: hidden rows get the padding norm and score +inf
  const int64_t R  = idx.lists.rows_total;
  const int* norms = idx.norms8.data();
  dbuf<int> norms_f;
  if (keep_bits != nullptr && R > 0) {
    norms_f.alloc(static_cast<size_t>(std::max<int64_t>(R, 128)), s);
    tc_i8_norms(s, idx.type == row_type::u8, idx.rows8.data(), R, R, idx.Kp8, idx.ids.data(), keep_bits, n_bits, norms_f.data());
    norms = norms_f.data();
  }

  // ---- 2. pairs by list, and their query bytes
  const int KCW = KC * kTcListsPerItem;
  probe_buckets pb;
  bucket_probes(res, probes.data(), nq, static_cast<int>(n_probes), idx.n_lists, idx.lists.d_offsets.data(), KCW, pb);
  const int64_t a_rows = pb.n_pairs + 128;
  dbuf<uint8_t> a(static_cast<size_t>(a_rows) * idx.Kp8, s);
  count_launch();
  pair_query_bytes_kernel<<<blocks_for(a_rows * idx.Kp8 / 16, 256), 256, 0, s>>>(q, idx.dim, idx.Kp8, pb.pair_query.data(), pb.n_items.data() + 1,
                                                                            a_rows, a.data());
  B2_CUDA(cudaGetLastError());

  // ---- 3. fine scan on the integer tensor cores
  const bool u8       = idx.type == row_type::u8;
  const int64_t b_rows = std::max<int64_t>(R, 128);
  dbuf<float> cs;
  dbuf<uint32_t> cp;
  int L = KCW;  // candidates per pair
  if (KC == 0) {
    large_k_select(s, pb, idx.lists, nq, n_probes, want, [&](float* scores, const int64_t* seg_off) {
      item_segments(s, pb, seg_off);
      timed_section ts("ivf_flat_scan", s);
      tc_scan_i8(s, res->device, u8, a.data(), a_rows, idx.rows8.data(), b_rows, idx.Kp8, norms, !ip, pb.items.data(), pb.max_items,
                 pb.n_items.data(), 0, scores, nullptr, 0);
    }, cs, cp);
    L = want;
  } else {
    cs.alloc(static_cast<size_t>(pb.n_pairs) * KCW, s);
    cp.alloc(static_cast<size_t>(pb.n_pairs) * KCW, s);
    dbuf<int> bkeys(static_cast<size_t>(nq), s);
    B2_CUDA(cudaMemsetAsync(bkeys.data(), tc_bound_init_byte, sizeof(int) * nq, s));
    tc_bound bnd;
    bnd.keys = bkeys.data();
    bnd.idx  = pb.pair_query.data();
    bnd.kth  = want < KC ? want : 0;
    timed_section ts("ivf_flat_scan", s);
    tc_scan_i8(s, res->device, u8, a.data(), a_rows, idx.rows8.data(), b_rows, idx.Kp8, norms, !ip, pb.items.data(), pb.max_items,
               pb.n_items.data(), KC, cs.data(), cp.data(), KCW, &bnd);
  }

  // ---- 4. per query: the want best keys of its pairs, then the k best by (distance, id)
  const int64_t cand_w = static_cast<int64_t>(n_probes) * L;
  dbuf<float> gs(static_cast<size_t>(nq) * cand_w, s);
  dbuf<uint32_t> gp(static_cast<size_t>(nq) * cand_w, s);
  gather_probe_candidates(s, cs.data(), cp.data(), pb.slot_of.data(), nullptr, 1.f, INFINITY, nq, static_cast<int>(n_probes), L,
                          gs.data(), gp.data());
  const int kc2 = static_cast<int>(std::min<int64_t>(cand_w, want));
  dbuf<float> ms(static_cast<size_t>(nq) * kc2, s);
  dbuf<uint32_t> mp(static_cast<size_t>(nq) * kc2, s);
  select_k(s, gs.data(), gp.data(), IDX_U32, nq, cand_w, cand_w, kc2, ms.data(), mp.data(), IDX_U32, true);
  count_launch();
  if (dump) {
    B2_EXPECTS(kc2 == want, "ivf_flat candidates: n_probes too small for %d candidates", want);
    i8_candidates_kernel<<<static_cast<unsigned>(nq), 256, 0, s>>>(ms.data(), mp.data(), kc2, idx.ids.data(), q, idx.dim, ip, dump->ids,
                                                                   dump->dist, dump->bound);
    B2_CUDA(cudaGetLastError());
    B2_CUDA(cudaStreamSynchronize(s));
    return;
  }
  i8_finish_kernel<<<static_cast<unsigned>(nq), 256, 0, s>>>(ms.data(), mp.data(), kc2, idx.ids.data(), q, idx.dim, ip, k,
                                                             dl_ptr<int64_t>(nt), dl_ptr<float>(dt));
  B2_CUDA(cudaGetLastError());
  postprocess_distances(s, dl_ptr<float>(dt), nq * k, idx.metric);
  set_last_flagged(0);
}

// dump: stop after the certificate and copy its inputs out (one query batch).
void ivf_flat_search(resources* res, const ivf_flat_index& idx, uint32_t n_probes, const DLTensor& qt, const DLTensor& nt,
                     const DLTensor& dt, const uint32_t* keep_bits = nullptr, int64_t n_bits = 0,
                     const flat_candidates* dump = nullptr)
{
  auto s           = res->stream;
  const int64_t nq = qt.shape[0];
  const int k      = static_cast<int>(nt.shape[1]);
  B2_EXPECTS(k >= 1 && k <= kSelectMaxK, "ivf_flat search: k must be in [1, %d] (got %d)", kSelectMaxK, k);
  B2_EXPECTS(n_probes >= 1, "n_probes must be >= 1");
  if (nq == 0) return;
  n_probes         = std::min<uint32_t>(n_probes, idx.n_lists);
  if (idx.type != row_type::f32) return ivf_flat_search_i8(res, idx, n_probes, qt, nt, dt, keep_bits, n_bits, dump);
  // k > 64 (DESIGN.md §4 "k > 64"): the scan stores every (pair, list row) score and a segmented select keeps kc2 per pair.
  const bool large_k = k > 64;
  const int large_kc = std::min(2 * k, kSelectMaxK);
  // Query batching.  Per (query, probe) pair: the bf16 query residual row and its offset, 2 x KC candidate slots and their
  // per-query concatenation.  k > 64, per query: dense scores (bounded by its n_probes largest lists), each pair's kc2 best and their
  // per-query gather (8 + 8 bytes each), the gathered bf16 query rows, slot bookkeeping (32 bytes per pair) and the merged kc2.
  const int64_t large_k_bytes = !large_k ? 0
                                         : large_k_rows_per_query(idx.lists, n_probes) * 4 +
                                             static_cast<int64_t>(n_probes) * (16 * large_kc + 2 * idx.Kp + 32) +
                                             static_cast<int64_t>(large_kc) * 8;
  const int64_t batch = query_batch_size(idx.Kp * 2 + 4 + 2 * 64 * 8 + 16, n_probes, large_k_bytes, "CUVS_B200_FLAT_LARGE_K_BUDGET_MB");
  B2_EXPECTS(dump == nullptr || nq <= batch, "ivf_flat candidates: %lld queries do not fit one batch", (long long)nq);
  if (search_in_batches(batch, qt, nt, dt, [&](const DLTensor& qs, const DLTensor& ns, const DLTensor& ds) {
        ivf_flat_search(res, idx, n_probes, qs, ns, ds, keep_bits, n_bits);
      }))
    return;
  const float* q   = dl_ptr<float>(qt);
  int64_t* out_idx = dl_ptr<int64_t>(nt);
  float* out_dist  = dl_ptr<float>(dt);

  // ---- 1. coarse
  dbuf<float> qn(static_cast<size_t>(nq), s);
  row_norms(s, q, nq, idx.dim, idx.dim, qn.data());
  dbuf<float> qscale;
  if (idx.metric == CosineExpanded) {
    qscale.alloc(static_cast<size_t>(nq), s);
    rsqrt_rows(s, qn.data(), nq, qscale.data());
  }
  tc_rows_tmp qp;
  qp.build(s, q, nq, idx.dim, true, 0, qscale.data());
  dbuf<uint32_t> probes(static_cast<size_t>(nq) * n_probes, s);
  coarse_select(res, qp, idx.centers_tc, static_cast<int>(n_probes), probes.data(), nullptr);

  // ---- 1b. bitset pre-filter (cuvs::neighbors::filtering::bitset_filter): one pass over the half-norm plane (the exact
  // fallback reads the bitset itself)
  dbuf<__nv_bfloat16> hx_f;
  const __nv_bfloat16* hx = idx.hx.data();
  if (keep_bits != nullptr && idx.lists.rows_total > 0) {
    const int64_t R = idx.lists.rows_total;
    dbuf<float> hn(static_cast<size_t>(R), s);
    hx_f.alloc(static_cast<size_t>(std::max<int64_t>(R, 128)) * 16, s);
    count_launch();
    half_norms_filtered_kernel<<<blocks_for(R, 256), 256, 0, s>>>(idx.rn.data(), idx.ids.data(), R, !is_l2(scan_metric(idx)), keep_bits, n_bits,
                                                                   hn.data());
    B2_CUDA(cudaGetLastError());
    tc_pack_half_norms(s, hn.data(), R, hx_f.data());
    hx = hx_f.data();
  }

  // ---- 2. bucket (query, probe) pairs by list
  // The scan ranks rows by a ONE-pass bf16 score; the exact fp32 re-score below only sees what survives it.  Keep slack
  // between k and the per-list capacity (and the shared pruning bound, which tracks the KC-th best): a true top-k row whose
  // bf16 score ranks a few places late must still be a candidate.  k <= 10 -> 16 slots, k <= 32 -> 32 slots; the bound is
  // only used when KC >= 1.5 k.  Step 5 certifies the result.
  // k > 64: no fused top-k (KC = 0, the store epilogue); each pair keeps its kc2 best from its dense score segment.
  const int KC    = large_k ? 0 : ((k + k / 2 <= 16) ? 16 : 32);
  const bool use_bound = !large_k && KC >= k + k / 2;
  int KCW         = KC * kTcListsPerItem;
  probe_buckets pb;
  bucket_probes(res, probes.data(), nq, static_cast<int>(n_probes), idx.n_lists, idx.lists.d_offsets.data(), KCW, pb);
  const cuvsDistanceType fine = fine_metric(idx);

  // ---- 3. fine scan: per-pair query residuals (A) x list residuals (B).  Scores of different pairs compare as distances,
  // add[slot] + scale * score (pair_residual_rows); cosine scores the unit query as L2 (scan_metric).
  residual_rows a;
  dbuf<float> add;
  float scale = 1.f;
  {
    const float* qf = q;
    dbuf<float> q_unit;
    if (idx.metric == CosineExpanded) {
      q_unit.alloc(static_cast<size_t>(nq) * idx.dim, s);
      B2_CUDA(cudaMemcpyAsync(q_unit.data(), q, sizeof(float) * nq * idx.dim, cudaMemcpyDeviceToDevice, s));
      normalize_rows(s, q_unit.data(), nq, idx.dim, idx.dim);
      qf = q_unit.data();
    }
    scale = pair_residual_rows(s, qf, residual_centers(idx), idx.dim, idx.Kp, scan_metric(idx), pb, false, a, add);
  }
  dbuf<float> cs;
  dbuf<uint32_t> cp;
  if (large_k) {
    // every (pair, list row) score goes to the pair's dense segment; each pair keeps its kc2 best rows
    large_k_select(s, pb, idx.lists, nq, n_probes, large_kc, [&](float* scores, const int64_t* seg_off) {
      item_segments(s, pb, seg_off);
      timed_section ts("ivf_flat_scan", s);
      tc_scan_topk(s, res->device, a.hi.data(), nullptr, a.rows, idx.hi.data(), nullptr, std::max<int64_t>(idx.lists.rows_total, 128),
                   idx.Kp, hx, pb.items.data(), pb.max_items, pb.n_items.data(), 0, 1, scores, nullptr, 0 /*per item*/);
    }, cs, cp);
    KCW = large_kc;
  } else {
    cs.alloc(static_cast<size_t>(pb.n_pairs) * KCW, s);
    cp.alloc(static_cast<size_t>(pb.n_pairs) * KCW, s);
    // probes of one query share a running bound on its k'-th best distance, add[slot] + scale * score
    dbuf<int> bkeys(static_cast<size_t>(nq), s);
    B2_CUDA(cudaMemsetAsync(bkeys.data(), tc_bound_init_byte, sizeof(int) * nq, s));
    tc_bound bnd;
    bnd.keys  = bkeys.data();
    bnd.idx   = pb.pair_query.data();
    bnd.add   = add.data();
    bnd.scale = scale;
    timed_section ts("ivf_flat_scan", s);
    tc_scan_topk(s, res->device, a.hi.data(), nullptr, a.rows, idx.hi.data(), nullptr, std::max<int64_t>(idx.lists.rows_total, 128),
                 idx.Kp, hx, pb.items.data(), pb.max_items, pb.n_items.data(), KC, 1, cs.data(), cp.data(), KCW, use_bound ? &bnd : nullptr);
  }

  // ---- 4. per query: merge probes by approximate score, exact re-score, ids
  const int64_t cand_w = static_cast<int64_t>(n_probes) * KCW;
  dbuf<float> gs(static_cast<size_t>(nq) * cand_w, s);
  dbuf<uint32_t> gp(static_cast<size_t>(nq) * cand_w, s);
  // empty entries +inf: FLT_MAX made the ivf_flat bench search ~3 % slower (DESIGN.md §4a)
  const int L = large_k ? KCW : KC;  // entries of one per-pair list
  dbuf<float> last(static_cast<size_t>(nq * cand_w / L), s);
  gather_probe_candidates(s, cs.data(), cp.data(), pb.slot_of.data(), add.data(), scale, INFINITY, nq,
                          static_cast<int>(n_probes), KCW, gs.data(), gp.data(), L, last.data());
  const int kc2 = static_cast<int>(std::min<int64_t>(cand_w, large_k ? large_kc : std::max(32, 2 * k)));
  dbuf<float> ms(static_cast<size_t>(nq) * kc2, s);
  dbuf<uint32_t> mp(static_cast<size_t>(nq) * kc2, s);
  select_k(s, gs.data(), gp.data(), IDX_U32, nq, cand_w, cand_w, kc2, ms.data(), mp.data(), IDX_U32, true);
  if (large_k) {
    // a row hidden by the bitset filter scores +inf in the store scan but keeps its position, and the segmented select returns
    // it whenever a pair holds fewer than kc2 kept rows: empty such slots before the exact re-score computes its true distance
    count_launch();
    drop_nonfinite_kernel<<<blocks_for(nq * kc2, 256), 256, 0, s>>>(ms.data(), mp.data(), nq * kc2);
    B2_CUDA(cudaGetLastError());
  }
  rescore_topk(s, q, nq, idx.dim, idx.data.data(), idx.dim, idx.dim, qn.data(), idx.xn.data(), fine, mp.data(), kc2,
               idx.ids.data(), k, out_idx, out_dist, INT64_MAX);

  // ---- 5. certificate (certify_kernel): the queries whose k-th exact distance is not safely below every row the bf16
  // candidates left out are searched again with exact scores and their rows written back
  dbuf<int> flags(static_cast<size_t>(nq) + 1, s);
  B2_CUDA(cudaMemsetAsync(flags.data() + nq, 0, sizeof(int), s));
  count_launch();
  certify_kernel<<<blocks_for(nq * 32, 256), 256, 0, s>>>(out_dist, k, int(fine), ms.data(), kc2, last.data(), KCW / L,
                                                         probes.data(), pb.slot_of.data(), static_cast<int>(n_probes),
                                                         add.data(), qn.data(), idx.rn_max.data(), idx.cn.data(), make_budget(idx, scale),
                                                         nq, flags.data());
  B2_CUDA(cudaGetLastError());
  if (dump) {
    count_launch();
    candidate_budget_kernel<<<blocks_for(nq * kc2, 256), 256, 0, s>>>(mp.data(), idx.ids.data(), idx.lists.d_offsets.data(), idx.n_lists,
                                                                      probes.data(), pb.slot_of.data(), static_cast<int>(n_probes), kc2,
                                                                      add.data(), qn.data(), idx.rn_max.data(), idx.cn.data(),
                                                                      make_budget(idx, scale), nq * kc2, dump->ids, dump->bound);
    B2_CUDA(cudaGetLastError());
    B2_CUDA(cudaMemcpyAsync(dump->dist, ms.data(), sizeof(float) * nq * kc2, cudaMemcpyDeviceToDevice, s));
    B2_CUDA(cudaStreamSynchronize(s));
    return;
  }
  if (!large_k) {
    count_launch();
    exact_fallback_kernel<<<static_cast<unsigned>(std::min<int64_t>(nq, 1024)), kFbThreads, 0, s>>>(
      flags.data(), probes.data(), static_cast<int>(n_probes), idx.lists.d_offsets.data(), q, idx.dim, idx.data.data(), qn.data(),
      idx.xn.data(), idx.ids.data(), int(fine), keep_bits, n_bits, k, nq, out_idx, out_dist);
    B2_CUDA(cudaGetLastError());
    postprocess_distances(s, out_dist, nq * k, idx.metric);
    set_last_flagged_async(flags.data() + nq, s);
    return;
  }
  // k > 64: the flagged queries are answered again by exact_probed_search over the lists they probed
  postprocess_distances(s, out_dist, nq * k, idx.metric);
  rerun_flagged(s, flags.data(), nq, k, out_idx, out_dist, [&](const int64_t* rows, int64_t n, int64_t* fi, float* fd) {
    dbuf<float> fq(static_cast<size_t>(n) * idx.dim, s);
    dbuf<uint32_t> fp(static_cast<size_t>(n) * n_probes, s);
    copy_rows(s, q, rows, fq.data(), nullptr, n, idx.dim);
    copy_rows(s, probes.data(), rows, fp.data(), nullptr, n, int64_t(n_probes));
    exact_probed_search(res, idx, fq.data(), n, fp.data(), n_probes, keep_bits, n_bits, k, fi, fd);
  });
}

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

cuvsError_t cuvsIvfFlatIndexParamsCreate(cuvsIvfFlatIndexParams_t* params)
{
  return guarded([=] {
    B2_EXPECTS(params != nullptr, "params is null");
    // defaults: c/src/neighbors/ivf_flat.cpp:265-277
    *params = new cuvsIvfFlatIndexParams{L2Expanded, 2.0f, true, 1024, 20, 0.5, false, false};
  });
}
cuvsError_t cuvsIvfFlatIndexParamsDestroy(cuvsIvfFlatIndexParams_t params) { return guarded([=] { delete params; }); }

cuvsError_t cuvsIvfFlatSearchParamsCreate(cuvsIvfFlatSearchParams_t* params)
{
  return guarded([=] {
    B2_EXPECTS(params != nullptr, "params is null");
    *params = new cuvsIvfFlatSearchParams{20};
  });
}
cuvsError_t cuvsIvfFlatSearchParamsDestroy(cuvsIvfFlatSearchParams_t params) { return guarded([=] { delete params; }); }

cuvsError_t cuvsIvfFlatIndexCreate(cuvsIvfFlatIndex_t* index)
{
  return guarded([=] {
    B2_EXPECTS(index != nullptr, "index is null");
    *index = new cuvsIvfFlatIndex{};
  });
}
cuvsError_t cuvsIvfFlatIndexDestroy(cuvsIvfFlatIndex_t index)
{
  return guarded([=] {
    if (!index) return;
    drop_index<ivf_flat_index>(index);
    delete index;
  });
}

cuvsError_t cuvsIvfFlatIndexGetNLists(cuvsIvfFlatIndex_t index, int64_t* n_lists)
{
  return guarded([=] { *n_lists = index_of<ivf_flat_index>(index).n_lists; });
}
cuvsError_t cuvsIvfFlatIndexGetDim(cuvsIvfFlatIndex_t index, int64_t* dim) { return guarded([=] { *dim = index_of<ivf_flat_index>(index).dim; }); }
cuvsError_t cuvsIvfFlatIndexGetCenters(cuvsIvfFlatIndex_t index, DLManagedTensor* centers)
{
  return guarded([=] {
    auto& idx        = index_of<ivf_flat_index>(index);
    int64_t shape[2] = {idx.n_lists, idx.dim};
    dl_fill_view(centers, idx.centers.data(), idx.device, DLDataType{kDLFloat, 32, 1}, 2, shape);
  });
}

cuvsError_t cuvsB200IvfFlatGetListSizes(cuvsIvfFlatIndex_t index, DLManagedTensor* list_sizes)
{
  return guarded([=] {
    auto& idx        = index_of<ivf_flat_index>(index);
    int64_t shape[1] = {idx.n_lists};
    dl_fill_view(list_sizes, idx.lists.d_sizes.data(), idx.device, DLDataType{kDLUInt, 32, 1}, 1, shape);
  });
}
cuvsError_t cuvsB200IvfFlatGetListIndices(cuvsIvfFlatIndex_t index, uint32_t label, DLManagedTensor* ids)
{
  return guarded([=] {
    auto& idx = index_of<ivf_flat_index>(index);
    B2_EXPECTS(label < idx.n_lists, "label %u out of range", label);
    int64_t shape[1] = {idx.lists.h_sizes[label]};
    dl_fill_view(ids, idx.ids.data() + idx.lists.h_offsets[label], idx.device, DLDataType{kDLInt, 64, 1}, 1, shape);
  });
}
cuvsError_t cuvsB200IvfFlatSetCenters(cuvsResources_t res, cuvsIvfFlatIndex_t index, DLManagedTensor* centers)
{
  return guarded([=] {
    auto r    = as_res(res);
    auto& idx = index_of<ivf_flat_index>(index);
    B2_EXPECTS(centers != nullptr, "centers is null");
    const DLTensor& c = centers->dl_tensor;
    B2_EXPECTS(dl_is(c, kDLFloat, 32) && c.ndim == 2 && c.shape[0] == idx.n_lists && c.shape[1] == idx.dim && dl_is_c_contiguous(c),
               "centers must be float32 [n_lists, dim]");
    B2_EXPECTS(idx.lists.size == 0, "centres can only be replaced while the index is empty");
    B2_CUDA(cudaMemcpyAsync(idx.centers.data(), dl_ptr<float>(c), sizeof(float) * idx.n_lists * idx.dim, cudaMemcpyDefault, r->stream));
    refresh_centers_tc(r, idx);
  });
}
cuvsError_t cuvsB200IvfFlatGetSize(cuvsIvfFlatIndex_t index, int64_t* size) { return guarded([=] { *size = index_of<ivf_flat_index>(index).lists.size; }); }

cuvsError_t cuvsB200IvfFlatCandidates(cuvsResources_t res, cuvsIvfFlatIndex_t index, uint32_t n_probes, int k, DLManagedTensor* queries,
                                      DLManagedTensor* cand_ids, DLManagedTensor* cand_dist, DLManagedTensor* bound)
{
  return guarded([=] {
    auto r    = as_res(res);
    auto& idx = index_of<ivf_flat_index>(index);
    B2_EXPECTS(queries && cand_ids && cand_dist && bound, "null argument");
    const DLTensor& q  = queries->dl_tensor;
    const DLTensor& ci = cand_ids->dl_tensor;
    const DLTensor& cd = cand_dist->dl_tensor;
    const DLTensor& b  = bound->dl_tensor;
    B2_EXPECTS(dl_is(q, kDLFloat, 32) && dl_is_device(q) && dl_is_c_contiguous(q) && q.ndim == 2 && q.shape[1] == idx.dim, "bad queries");
    B2_EXPECTS(k >= 1 && k <= 64, "k must be in [1, 64]");
    const int64_t nq = q.shape[0];
    const int kc2    = std::max(32, 2 * k);
    B2_EXPECTS(dl_is(ci, kDLInt, 64) && dl_is(cd, kDLFloat, 32) && dl_is(b, kDLFloat, 32) && dl_is_device(ci) && dl_is_device(cd) &&
                 dl_is_device(b) && ci.ndim == 2 && cd.ndim == 2 && ci.shape[0] == nq && cd.shape[0] == nq && ci.shape[1] == kc2 &&
                 cd.shape[1] == kc2 && b.ndim == 2 && b.shape[0] == nq && b.shape[1] == kc2 && dl_is_c_contiguous(ci) &&
                 dl_is_c_contiguous(cd) && dl_is_c_contiguous(b),
               "cand_ids / cand_dist / bound must be [nq, max(32, 2k)] int64 / float32 / float32, on the device");
    B2_EXPECTS(static_cast<int64_t>(std::min(n_probes, idx.n_lists)) * 2 * (k + k / 2 <= 16 ? 16 : 32) >= kc2, "n_probes too small for kc2");
    dbuf<int64_t> ni(static_cast<size_t>(nq) * k, r->stream);
    dbuf<float> nd(static_cast<size_t>(nq) * k, r->stream);
    const dl_view nt(ni.data(), q.device, DLDataType{kDLInt, 64, 1}, nq, k), dt(nd.data(), q.device, DLDataType{kDLFloat, 32, 1}, nq, k);
    flat_candidates c{dl_ptr<int64_t>(ci), dl_ptr<float>(cd), dl_ptr<float>(b)};
    ivf_flat_search(r, idx, n_probes, q, nt.t(), dt.t(), nullptr, 0, &c);
  });
}

cuvsError_t cuvsIvfFlatBuild(cuvsResources_t res, cuvsIvfFlatIndexParams_t params, DLManagedTensor* dataset, cuvsIvfFlatIndex_t index)
{
  return guarded([=] {
    auto r = as_res(res);
    B2_EXPECTS(params && dataset && index, "null argument");
    const DLTensor& ds = dataset->dl_tensor;
    B2_EXPECTS(dl_is_dataset_dtype(ds), "Unsupported dataset DLtensor dtype: %d and bits: %d", ds.dtype.code, ds.dtype.bits);
    drop_index<ivf_flat_index>(index);
    // int8 / uint8 datasets in L2 or inner product keep their type; float16 ones, and 8-bit ones for cosine, are widened to fp32
    // rows (c/src/neighbors/ivf_flat.cpp dtype switch)
    if (row_type_for(ds.dtype, params->metric) != row_type::f32) {
      set_index(index, ivf_flat_build(r, *params, ds), ds.dtype);
    } else {
      f32_matrix w;
      widen_to_f32(r, ds, w);
      set_index(index, ivf_flat_build(r, *params, w.t), ds.dtype);
    }
  });
}

cuvsError_t cuvsIvfFlatSearch(cuvsResources_t res, cuvsIvfFlatSearchParams_t params, cuvsIvfFlatIndex_t index,
                              DLManagedTensor* queries_t, DLManagedTensor* neighbors_t, DLManagedTensor* distances_t, cuvsFilter filter)
{
  return guarded([=] {
    auto r = as_res(res);
    B2_EXPECTS(params && queries_t && neighbors_t && distances_t, "null argument");
    auto& idx = index_of<ivf_flat_index>(index);
    const DLTensor& queries   = queries_t->dl_tensor;
    const DLTensor& neighbors = neighbors_t->dl_tensor;
    const DLTensor& distances = distances_t->dl_tensor;
    check_search_tensors(queries, neighbors, distances, idx.dim, false);
    B2_EXPECTS(queries.dtype.code == index->dtype.code && queries.dtype.bits == index->dtype.bits, "type mismatch between index and queries");
    B2_EXPECTS(dl_is_c_contiguous(queries), "queries must be row-major contiguous");
    const filter_view filt = read_prefilter(filter, false, "ivf_flat search: only bitset pre-filters are supported (as in the reference)");
    f32_rows qv;
    widen_to_f32(r, queries, qv);
    ivf_flat_search(r, idx, params->n_probes, qv.t, neighbors, distances, filt.bits, filt.n_samples);
  });
}

cuvsError_t cuvsIvfFlatExtend(cuvsResources_t res, DLManagedTensor* new_vectors, DLManagedTensor* new_indices, cuvsIvfFlatIndex_t index)
{
  return guarded([=] {
    auto r    = as_res(res);
    auto& idx = index_of<ivf_flat_index>(index);
    B2_EXPECTS(new_vectors != nullptr, "new_vectors is null");
    B2_EXPECTS(dl_is_dataset_dtype(new_vectors->dl_tensor), "Unsupported new_vectors DLtensor dtype: %d and bits: %d",
               new_vectors->dl_tensor.dtype.code, new_vectors->dl_tensor.dtype.bits);
    f32_rows wv;
    if (idx.type != row_type::f32) {  // 8-bit lists take rows of their own type
      const DLTensor& nv = new_vectors->dl_tensor;
      B2_EXPECTS(nv.dtype.code == index->dtype.code && nv.dtype.bits == 8, "type mismatch between index and new_vectors");
      B2_EXPECTS(nv.ndim == 2 && dl_is_c_contiguous(nv), "matrix must be a row-major 2-D tensor");
      wv.t = nv;
    } else {
      widen_to_f32(r, new_vectors->dl_tensor, wv);
    }
    const DLTensor& v = wv.t;
    B2_EXPECTS(v.ndim == 2 && v.shape[1] == idx.dim && dl_is_c_contiguous(v), "new_vectors must be [n, dim] row-major");
    dbuf<int64_t> ids_buf;
    // reference: new ids continue after the current size when none are given
    ivf_flat_extend(r, idx, v, device_ids(r, new_indices, v.shape[0], ids_buf), idx.lists.size);
  });
}

// cuVS index file, serialization version 4 (cpp/src/neighbors/ivf_flat/ivf_flat_serialize.cuh:25-84; per-list records
// cpp/src/neighbors/ivf_list.cuh:108-133): the 4-byte dtype tag of the index's type ("<f4\0", "<e2\0", "|i1\0", "|u1\0": the
// kind and size the reader dispatches on, c/src/neighbors/ivf_flat.cpp:307-325), then NPY records (npy_io.hpp) —
//   version i4 = 4, size i8, dim u4, n_lists u4, metric i4, adaptive_centers u1, conservative_memory_allocation u1,
//   centers f4 [n_lists, dim], has_norms u1 (+ center_norms f4 [n_lists] for L2), list_sizes u4 [n_lists], then per list:
//   capacity u4 = size rounded up to 32 and (capacity > 0) data [capacity, dim] of the index's type ('<f4', '<f2', '|i1',
//   '|u1') in the reference's interleaved layout (groups of 32 rows, element (r, k) at (r/32)*32*dim + (k/veclen)*32*veclen +
//   (r%32)*veclen + k%veclen, veclen = 16 / sizeof(T) when dim is a multiple of it, else 1: ivf_flat.hpp:184-201, 284-293) and
//   indices i8 [capacity] (-1 = kInvalidRecord on the padding rows).
namespace {

inline int flat_veclen(int dim, int size) { return dim % (16 / size) == 0 ? 16 / size : 1; }
inline int64_t interleaved_at(int64_t r, int k, int dim, int vl) { return (r / 32) * 32 * dim + (k / vl) * 32 * vl + (r % 32) * vl + k % vl; }

// fp32 storage value <-> file element of `size` bytes of type t (the values are the type's: the conversions are exact)
void put_element(DLDataType t, float v, uint8_t* out)
{
  if (t.bits == 32) std::memcpy(out, &v, 4);
  else if (t.bits == 16) { const __half h = __float2half_rn(v); std::memcpy(out, &h, 2); }
  else *out = static_cast<uint8_t>(static_cast<int>(v));
}
float get_element(DLDataType t, const uint8_t* in)
{
  if (t.bits == 32) { float v; std::memcpy(&v, in, 4); return v; }
  if (t.bits == 16) { __half h; std::memcpy(&h, in, 2); return __half2float(h); }
  return t.code == kDLInt ? static_cast<float>(static_cast<int8_t>(*in)) : static_cast<float>(*in);
}

}  // namespace

cuvsError_t cuvsIvfFlatSerialize(cuvsResources_t res, const char* filename, cuvsIvfFlatIndex_t index)
{
  return guarded([=] {
    auto r    = as_res(res);
    auto& idx = index_of<ivf_flat_index>(index);
    std::ofstream os(filename, std::ios::out | std::ios::binary);
    B2_EXPECTS(bool(os), "Cannot open file %s", filename);
    const npy::file_dtype& ft = npy::file_dtype_for(index->dtype);
    os.write(ft.tag, 4);  // three characters and the terminating zero
    npy::write_scalar<int32_t>(os, 4);
    npy::write_scalar<int64_t>(os, idx.lists.size);
    npy::write_scalar<uint32_t>(os, static_cast<uint32_t>(idx.dim));
    npy::write_scalar<uint32_t>(os, idx.n_lists);
    npy::write_scalar<int32_t>(os, static_cast<int32_t>(idx.metric));
    npy::write_scalar<bool>(os, idx.adaptive_centers);
    npy::write_scalar<bool>(os, false);
    std::vector<float> c(static_cast<size_t>(idx.n_lists) * idx.dim);
    B2_CUDA(cudaMemcpyAsync(c.data(), idx.centers.data(), c.size() * sizeof(float), cudaMemcpyDeviceToHost, r->stream));
    B2_CUDA(cudaStreamSynchronize(r->stream));
    npy::write_array<float>(os, c.data(), {static_cast<int64_t>(idx.n_lists), idx.dim});
    const bool has_norms = is_l2(idx.metric);
    npy::write_scalar<bool>(os, has_norms);
    if (has_norms) {
      std::vector<float> cn(idx.n_lists);
      for (uint32_t l = 0; l < idx.n_lists; ++l) {
        float acc = 0.f;
        for (int j = 0; j < idx.dim; ++j) acc = fmaf(c[static_cast<size_t>(l) * idx.dim + j], c[static_cast<size_t>(l) * idx.dim + j], acc);
        cn[l] = acc;
      }
      npy::write_array<float>(os, cn.data(), {static_cast<int64_t>(idx.n_lists)});
    }
    std::vector<uint32_t> sizes(idx.n_lists);
    for (uint32_t l = 0; l < idx.n_lists; ++l) sizes[l] = static_cast<uint32_t>(idx.lists.h_sizes[l]);
    npy::write_array<uint32_t>(os, sizes.data(), {static_cast<int64_t>(idx.n_lists)});
    const bool native = idx.type != row_type::f32;
    const int dim = idx.dim, es = ft.size, vl = flat_veclen(dim, es);
    std::vector<float> rows;
    std::vector<uint8_t> rows8, inter;
    std::vector<int64_t> ids;
    for (uint32_t l = 0; l < idx.n_lists; ++l) {
      const int64_t sz = idx.lists.h_sizes[l], cap = (sz + 31) / 32 * 32, row0 = idx.lists.h_offsets[l];
      npy::write_scalar<uint32_t>(os, static_cast<uint32_t>(cap));
      if (!cap) continue;
      ids.assign(static_cast<size_t>(cap), int64_t(-1));
      inter.assign(static_cast<size_t>(cap) * dim * es, 0);
      B2_CUDA(cudaMemcpyAsync(ids.data(), idx.ids.data() + row0, static_cast<size_t>(sz) * sizeof(int64_t), cudaMemcpyDeviceToHost, r->stream));
      if (native) {
        rows8.resize(static_cast<size_t>(sz) * idx.Kp8);
        B2_CUDA(cudaMemcpyAsync(rows8.data(), idx.rows8.data() + row0 * idx.Kp8, rows8.size(), cudaMemcpyDeviceToHost, r->stream));
      } else {
        rows.resize(static_cast<size_t>(sz) * dim);
        B2_CUDA(cudaMemcpyAsync(rows.data(), idx.data.data() + row0 * dim, rows.size() * sizeof(float), cudaMemcpyDeviceToHost, r->stream));
      }
      B2_CUDA(cudaStreamSynchronize(r->stream));
      for (int64_t rr = 0; rr < sz; ++rr)
        for (int k = 0; k < dim; ++k) {
          uint8_t* o = inter.data() + interleaved_at(rr, k, dim, vl) * es;
          if (native) *o = rows8[static_cast<size_t>(rr) * idx.Kp8 + k];
          else put_element(index->dtype, rows[static_cast<size_t>(rr) * dim + k], o);
        }
      npy::write_header(os, ft.descr, {cap, dim});
      os.write(reinterpret_cast<const char*>(inter.data()), static_cast<std::streamsize>(inter.size()));
      npy::write_array<int64_t>(os, ids.data(), {cap});
    }
    B2_EXPECTS(bool(os), "Error writing %s", filename);
  });
}

cuvsError_t cuvsIvfFlatDeserialize(cuvsResources_t res, const char* filename, cuvsIvfFlatIndex_t index)
{
  return guarded([=] {
    auto r = as_res(res);
    B2_EXPECTS(index && filename, "null argument");
    std::ifstream is(filename, std::ios::in | std::ios::binary);
    B2_EXPECTS(bool(is), "Cannot open file %s", filename);
    char tag[4]{};
    B2_EXPECTS(bool(is.read(tag, 4)), "ivf_flat::deserialize: failed to read dtype prefix");
    const npy::file_dtype* ft = npy::file_dtype_named(std::string(tag, 3));
    B2_EXPECTS(ft != nullptr, "ivf_flat::deserialize: unsupported dtype prefix '%.3s' in the index file", tag);
    const DLDataType dtype = ft->dl;
    const int ver = npy::read_scalar<int32_t>(is, filename);
    B2_EXPECTS(ver == 4, "serialization version mismatch, expected %d, got %d ", 4, ver);
    const int64_t n_rows = npy::read_scalar<int64_t>(is, filename);
    auto idx      = std::make_unique<ivf_flat_index>();
    idx->device   = r->device;
    idx->dim      = static_cast<int>(npy::read_scalar<uint32_t>(is, filename));
    idx->n_lists  = npy::read_scalar<uint32_t>(is, filename);
    idx->metric   = static_cast<cuvsDistanceType>(npy::read_scalar<int32_t>(is, filename));
    idx->adaptive_centers = npy::read_scalar<uint8_t>(is, filename) != 0;
    idx->type     = row_type_for(dtype, idx->metric);
    idx->Kp8      = tc_pad_k_i8(idx->dim);
    (void)npy::read_scalar<uint8_t>(is, filename);  // conservative_memory_allocation: an allocation policy, nothing to restore
    std::vector<float> c(static_cast<size_t>(idx->n_lists) * idx->dim);
    npy::read_array<float>(is, c.data(), static_cast<int64_t>(c.size()), filename);
    if (npy::read_scalar<uint8_t>(is, filename) != 0) {
      std::vector<float> cn(idx->n_lists);  // recomputed on load (refresh_centers_tc)
      npy::read_array<float>(is, cn.data(), idx->n_lists, filename);
    }
    std::vector<uint32_t> sizes32(idx->n_lists);
    npy::read_array<uint32_t>(is, sizes32.data(), idx->n_lists, filename);
    std::vector<int64_t> sizes(sizes32.begin(), sizes32.end());
    idx->centers.alloc(c.size());
    B2_CUDA(cudaMemcpyAsync(idx->centers.data(), c.data(), c.size() * sizeof(float), cudaMemcpyHostToDevice, r->stream));
    B2_CUDA(cudaStreamSynchronize(r->stream));
    refresh_centers_tc(r, *idx);
    idx->lists.set_sizes(r->stream, sizes);
    B2_EXPECTS(idx->lists.size == n_rows, "ivf_flat::deserialize: list sizes sum to %lld, header says %lld rows", (long long)idx->lists.size,
               (long long)n_rows);
    const bool native = idx->type != row_type::f32;
    if (native) alloc_list_storage(r->stream, idx->lists, idx->Kp8, idx->rows8, idx->ids);
    else alloc_list_storage(r->stream, idx->lists, idx->dim, idx->data, idx->ids);
    const int es = dtype.bits / 8, dim = idx->dim, vl = flat_veclen(dim, es);
    std::vector<float> rows;
    std::vector<uint8_t> rows8, inter;
    std::vector<int64_t> ids;
    for (uint32_t l = 0; l < idx->n_lists; ++l) {
      const int64_t cap = npy::read_scalar<uint32_t>(is, filename);
      const int64_t sz  = sizes[l], row0 = idx->lists.h_offsets[l];
      B2_EXPECTS(cap >= sz, "ivf_flat::deserialize: list %u stores %lld rows, list_sizes says %lld", l, (long long)cap, (long long)sz);
      if (!cap) continue;
      const npy::header h = npy::read_header(is, filename);
      B2_EXPECTS(npy::file_dtype_named(h.descr) == ft && !h.fortran && h.count() == cap * dim,
                 "ivf_flat::deserialize: list %u holds %lld elements of '%s', the file's type '%.3s' needs %lld", l, (long long)h.count(),
                 h.descr.c_str(), tag, (long long)(cap * dim));
      inter.resize(static_cast<size_t>(cap) * dim * es);
      is.read(reinterpret_cast<char*>(inter.data()), static_cast<std::streamsize>(inter.size()));
      B2_EXPECTS(bool(is), "%s: truncated file", filename);
      ids.resize(static_cast<size_t>(cap));
      npy::read_array<int64_t>(is, ids.data(), cap, filename);
      if (!sz) continue;
      if (native) {
        rows8.assign(static_cast<size_t>(sz) * idx->Kp8, 0);
        for (int64_t rr = 0; rr < sz; ++rr)
          for (int k = 0; k < dim; ++k) rows8[static_cast<size_t>(rr) * idx->Kp8 + k] = inter[interleaved_at(rr, k, dim, vl)];
        B2_CUDA(cudaMemcpyAsync(idx->rows8.data() + row0 * idx->Kp8, rows8.data(), rows8.size(), cudaMemcpyHostToDevice, r->stream));
      } else {
        rows.resize(static_cast<size_t>(sz) * dim);
        for (int64_t rr = 0; rr < sz; ++rr)
          for (int k = 0; k < dim; ++k)
            rows[static_cast<size_t>(rr) * dim + k] = get_element(dtype, inter.data() + interleaved_at(rr, k, dim, vl) * es);
        B2_CUDA(cudaMemcpyAsync(idx->data.data() + row0 * dim, rows.data(), rows.size() * sizeof(float), cudaMemcpyHostToDevice, r->stream));
      }
      B2_CUDA(cudaMemcpyAsync(idx->ids.data() + row0, ids.data(), static_cast<size_t>(sz) * sizeof(int64_t), cudaMemcpyHostToDevice, r->stream));
      B2_CUDA(cudaStreamSynchronize(r->stream));
    }
    refresh_rows(r, *idx);
    set_index(index, idx.release(), dtype);
  });
}

}  // extern "C"
