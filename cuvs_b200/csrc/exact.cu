// Exact fp32 kernels (oracle arithmetic): norms, dense distance tiles, candidate re-scoring.
// See exact.cuh.  Reference semantics restated:
//   expanded L2 + clamps      cpp/src/distance/detail/distance_ops/l2_exp.cuh:100-118
//   unexpanded / IP / cosine  cpp/tests/neighbors/naive_knn.cuh:34-86
//   post-selection sqrt       cpp/src/neighbors/detail/knn_brute_force.cuh:468-479
#include "common.hpp"
#include "exact.cuh"
#include "exact_device.cuh"
#include "timing.hpp"

#include <cfloat>
#include <type_traits>
#include <vector>

namespace b200 {
namespace {

template <typename T>
__global__ void row_norms_kernel(const T* __restrict__ x, int64_t n, int d, int64_t ld, float* __restrict__ out)
{
  int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const T* r = x + i * ld;
  float acc  = 0.f;
  if constexpr (!std::is_same_v<T, float>) {
    for (int k = 0; k < d; ++k) { const float v = widen(r[k]); acc = fmaf(v, v, acc); }
  } else if ((d & 3) == 0 && (ld & 3) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0) {
    const float4* r4 = reinterpret_cast<const float4*>(r);
    for (int k = 0; k < d / 4; ++k) {
      float4 v = r4[k];
      acc      = fmaf(v.x, v.x, acc);
      acc      = fmaf(v.y, v.y, acc);
      acc      = fmaf(v.z, v.z, acc);
      acc      = fmaf(v.w, v.w, acc);
    }
  } else {
    for (int k = 0; k < d; ++k) acc = fmaf(r[k], r[k], acc);
  }
  out[i] = acc;
}

__global__ void rsqrt_rows_kernel(const float* xn, float* out, int64_t n)
{
  int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i < n) out[i] = xn[i] > 0.f ? 1.0f / sqrtf(xn[i]) : 0.f;
}

__global__ void scale_rows_kernel(float* __restrict__ x, int64_t n, int d, int64_t ld, const float* __restrict__ scale)
{
  int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (t >= n * d) return;
  const int64_t r = t / d;
  const int c     = static_cast<int>(t % d);
  x[r * ld + c] *= scale[r];
}

__device__ __forceinline__ bool keep_sample(const filter_view& f, int64_t q, int64_t j)
{
  if (f.kind == 0) return true;
  int64_t bit = f.kind == 1 ? j : q * f.n_samples + j;
  return (f.bits[bit >> 5] >> (bit & 31)) & 1u;
}

constexpr int TM = 64, TN = 64, TK = 16;

// 64x64 output tile per CTA, 256 threads, 4x4 micro-tile per thread; every output accumulates over
// k = 0..d-1 in order (one fmaf per k), which is the oracle's order.
template <bool SqDiff, typename T>
__global__ void __launch_bounds__(256) exact_tile_kernel(const float* __restrict__ q, int64_t nq, int64_t ldq,
                                                           const T* __restrict__ x, int64_t n, int64_t ldx, int d,
                                                           const float* __restrict__ qn, const float* __restrict__ xn,
                                                           int metric, float* __restrict__ out, int64_t ldo,
                                                           filter_view filt, int64_t q_row0, bool self_clamp)
{
  __shared__ float As[TK][TM + 1];
  __shared__ float Bs[TK][TN + 1];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int64_t row0 = static_cast<int64_t>(blockIdx.y) * TM, col0 = static_cast<int64_t>(blockIdx.x) * TN;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < d; k0 += TK) {
    // 64 rows x 16 k = 1024 elements per operand, 4 per thread
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      int idx = tid + e * 256;
      int r = idx >> 4, kk = idx & 15;
      int64_t gr = row0 + r, gc = col0 + r;
      As[kk][r] = (gr < nq && k0 + kk < d) ? q[gr * ldq + k0 + kk] : 0.f;
      Bs[kk][r] = (gc < n && k0 + kk < d) ? widen(x[gc * ldx + k0 + kk]) : 0.f;
    }
    __syncthreads();
    const int kmax = min(TK, d - k0);
    for (int kk = 0; kk < kmax; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if constexpr (SqDiff) {
            float t   = a[i] - b[j];
            acc[i][j] = fmaf(t, t, acc[i][j]);
          } else {
            acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
          }
        }
    }
    __syncthreads();
  }
  const bool select_min = metric != InnerProduct;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int64_t gr = row0 + ty * 4 + i;
    if (gr >= nq) continue;
    float qnv = qn ? qn[gr] : 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int64_t gc = col0 + tx * 4 + j;
      if (gc >= n) continue;
      float v = finish_distance(acc[i][j], qnv, xn ? xn[gc] : 0.f, metric, self_clamp);
      if (!keep_sample(filt, q_row0 + gr, gc)) v = select_min ? FLT_MAX : -FLT_MAX;
      out[gr * ldo + gc] = v;
    }
  }
}

constexpr int kMaxCand      = 256;   // one warp per query
constexpr int kMaxCandBlock = 2048;  // one CTA per query

// one warp per query
template <typename T>
__global__ void __launch_bounds__(128) rescore_kernel(const float* __restrict__ q, int64_t nq, int64_t ldq,
                                                       const T* __restrict__ x, int64_t ldx, int d,
                                                       const float* __restrict__ qn, const float* __restrict__ xn,
                                                       int metric, const uint32_t* __restrict__ cand_pos, int kc,
                                                       const int64_t* __restrict__ src_ids, int k,
                                                       int64_t* __restrict__ out_idx, float* __restrict__ out_dist,
                                                       int64_t pad_id, bool self_clamp)
{
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warps = blockDim.x >> 5, wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* sd       = reinterpret_cast<float*>(smem_raw) + static_cast<size_t>(wid) * kc;
  int64_t* si     = reinterpret_cast<int64_t*>(reinterpret_cast<float*>(smem_raw) + static_cast<size_t>(warps) * kc) +
                static_cast<size_t>(wid) * kc;
  const int64_t qi = static_cast<int64_t>(blockIdx.x) * warps + wid;
  if (qi >= nq) return;
  const bool select_min = metric != InnerProduct;
  const float* qr       = q + qi * ldq;
  const float qnv       = qn ? qn[qi] : 0.f;
  bool vec4             = false;
  if constexpr (std::is_same_v<T, float>) vec4 = exact_vec4(q, ldq, x, ldx, d);

  for (int c = lane; c < kc; c += 32) {
    uint32_t pos = cand_pos[qi * kc + c];
    float dist   = select_min ? FLT_MAX : -FLT_MAX;
    int64_t id   = INT64_MAX;
    if (pos != 0xffffffffu) {
      const float acc = exact_accumulate(qr, x + static_cast<int64_t>(pos) * ldx, d, vec4, metric);
      dist            = finish_distance(acc, qnv, xn ? xn[pos] : 0.f, metric, self_clamp);
      id   = src_ids ? src_ids[pos] : static_cast<int64_t>(pos);
    }
    sd[c] = dist;
    si[c] = id;
  }
  __syncwarp();
  // rank by (distance, id, slot): unique ranks even among empty slots
  for (int c = lane; c < kc; c += 32) {
    float dv = sd[c];
    int64_t iv = si[c];
    int rank = 0;
    for (int o = 0; o < kc; ++o) {
      float d2 = sd[o];
      int64_t i2 = si[o];
      bool better = (d2 != dv) ? (select_min ? d2 < dv : d2 > dv) : ((i2 != iv) ? (i2 < iv) : (o < c));
      rank += better ? 1 : 0;
    }
    if (rank < k) {
      bool valid = iv != INT64_MAX;
      out_idx[qi * k + rank]  = valid ? iv : pad_id;
      out_dist[qi * k + rank] = dv;
    }
  }
  for (int j = kc + lane; j < k; j += 32) {  // k > kc: pad
    out_idx[qi * k + j]  = pad_id;
    out_dist[qi * k + j] = select_min ? FLT_MAX : -FLT_MAX;
  }
}

// More candidates than one warp's shared memory holds (refine with 257..2048 candidates): one CTA per query.  Every candidate
// is scored by one thread with exact_accumulate, as in rescore_kernel, then the kc entries are sorted by rescore_kernel's
// ranking rule, (distance, id, slot), with a bitonic sort over kpow2 entries; the padding entries (slot >= kc) rank last.
template <typename T>
__global__ void __launch_bounds__(256) rescore_block_kernel(const float* __restrict__ q, int64_t ldq, const T* __restrict__ x,
                                                             int64_t ldx, int d, const float* __restrict__ qn,
                                                             const float* __restrict__ xn, int metric,
                                                             const uint32_t* __restrict__ cand_pos, int kc, int kpow2,
                                                             const int64_t* __restrict__ src_ids, int k,
                                                             int64_t* __restrict__ out_idx, float* __restrict__ out_dist, int64_t pad_id,
                                                             bool self_clamp)
{
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int64_t* si = reinterpret_cast<int64_t*>(smem_raw);
  float* sd   = reinterpret_cast<float*>(si + kpow2);
  int* sc     = reinterpret_cast<int*>(sd + kpow2);
  const int64_t qi      = blockIdx.x;
  const bool select_min = metric != InnerProduct;
  const float* qr       = q + qi * ldq;
  const float qnv       = qn ? qn[qi] : 0.f;
  bool vec4             = false;
  if constexpr (std::is_same_v<T, float>) vec4 = exact_vec4(q, ldq, x, ldx, d);
  for (int c = threadIdx.x; c < kpow2; c += blockDim.x) {
    float dist = select_min ? FLT_MAX : -FLT_MAX;
    int64_t id = INT64_MAX;
    const uint32_t pos = c < kc ? cand_pos[qi * kc + c] : 0xffffffffu;
    if (pos != 0xffffffffu) {
      const float acc = exact_accumulate(qr, x + static_cast<int64_t>(pos) * ldx, d, vec4, metric);
      dist            = finish_distance(acc, qnv, xn ? xn[pos] : 0.f, metric, self_clamp);
      id   = src_ids ? src_ids[pos] : static_cast<int64_t>(pos);
    }
    sd[c] = dist;
    si[c] = id;
    sc[c] = c;
  }
  __syncthreads();
  // a before b in the ranking (slots are unique, so this is a strict total order)
  block_bitonic_sort(sd, si, sc, kpow2, [&](int a, int b) {
    const bool pa = sc[a] >= kc, pb = sc[b] >= kc;
    if (pa != pb) return pb;
    if (sd[a] != sd[b]) return select_min ? sd[a] < sd[b] : sd[a] > sd[b];
    return si[a] != si[b] ? si[a] < si[b] : sc[a] < sc[b];
  });
  for (int j = threadIdx.x; j < k; j += blockDim.x) {
    const int64_t iv = si[j];
    out_idx[qi * k + j]  = iv != INT64_MAX ? iv : pad_id;
    out_dist[qi * k + j] = sd[j];
  }
}

__global__ void postprocess_kernel(float* dist, int64_t count, int metric)
{
  int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= count) return;
  float v = dist[i];
  if (metric == L2SqrtExpanded || metric == L2SqrtUnexpanded) {
    if (v != FLT_MAX) dist[i] = sqrtf(fmaxf(v, 0.f));
  }
}

// dst[dst_row(i)] = src[src_row(i)] for rows of `width` elements; a null row map is the identity
template <typename T>
__global__ void copy_rows_kernel(const T* __restrict__ src, const int64_t* __restrict__ src_rows, T* __restrict__ dst,
                                 const int64_t* __restrict__ dst_rows, int64_t n, int64_t width)
{
  int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (t >= n * width) return;
  const int64_t i = t / width, j = t % width;
  dst[(dst_rows ? dst_rows[i] : i) * width + j] = src[(src_rows ? src_rows[i] : i) * width + j];
}

// floor[q] = min over the query's lists of the list's last (= worst, lists are sorted best-first) entry; a list that is not
// full ends in +inf and constrains nothing.  Every row the scan rejected — by a list's own k'-th entry or by the bound shared
// between the splits, which is some full list's k'-th entry at an earlier time and only ever decreases — scores above it.
__global__ void list_floor_kernel(const float* __restrict__ cs, int64_t nq, int64_t row_stride, int KC, float* __restrict__ out)
{
  const int64_t q = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
  const int lane  = threadIdx.x & 31;
  if (q >= nq) return;
  float m = INFINITY;
  for (int64_t l = lane; l * KC < row_stride; l += 32) m = fminf(m, cs[q * row_stride + l * KC + KC - 1]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) out[q] = m;
}

// The certificate (DESIGN.md §3), one warp per query: flags[q] = 1 (flags[nq] counts them) unless the exact k-th distance
// out_dist[q, k-1] (selection form, before postprocess_distances) beats the worst approximate score A of the rows outside the
// candidates by more than eps_rel * (eq |q|^2 + ec).  Such rows exist when the candidate list is full and score worse than its
// worst entry; with a floor (raw engine units, +inf: none), the bound of the rows that never entered a list, also worse than it.
// kExactInts (8-bit scans): while m = |q|^2 + max|x|^2 < 2^23, every value the scan keys, the re-score and this kernel form is an
// integer below 2^24 in magnitude (norms and partial sums <= m, distances <= 2m), so all of them are exact and eps is 0.
template <bool kExactInts>
__global__ void certify_kernel(const float* __restrict__ cand_score, const uint32_t* __restrict__ cand_pos, int kc,
                                  const float* __restrict__ approx_floor, const float* __restrict__ qn,
                                  const float* __restrict__ out_dist, int k, approx_map amap, bool select_min, int64_t nq,
                                  int* __restrict__ flags)
{
  const int64_t qi = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
  const int lane   = threadIdx.x & 31;
  if (qi >= nq) return;
  const float qnv    = qn[qi];
  float worst_approx = select_min ? -FLT_MAX : FLT_MAX;
  int n_valid        = 0;
  for (int c = lane; c < kc; c += 32) {
    if (cand_pos[qi * kc + c] == 0xffffffffu) continue;
    ++n_valid;
    float a      = amap.sa * cand_score[qi * kc + c] + amap.sb * qnv + amap.sc;
    worst_approx = select_min ? fmaxf(worst_approx, a) : fminf(worst_approx, a);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    n_valid += __shfl_xor_sync(0xffffffffu, n_valid, o);
    float t = __shfl_xor_sync(0xffffffffu, worst_approx, o);
    worst_approx = select_min ? fmaxf(worst_approx, t) : fminf(worst_approx, t);
  }
  if (lane != 0) return;
  const float kth = out_dist[qi * k + k - 1];
  int flag        = 0;
  bool outside    = n_valid == kc;  // candidate list is full: rows outside it exist (dropped by the merge to kc)
  if (approx_floor != nullptr) {
    const float fl = approx_floor[qi];
    if (fl < FLT_MAX) {
      const float a = amap.sa * fl + amap.sb * qnv + amap.sc;
      worst_approx  = !outside ? a : (select_min ? fminf(worst_approx, a) : fmaxf(worst_approx, a));
      outside       = true;
    }
  }
  if (outside) {
    const float mag = amap.eq * qnv + amap.ec;
    float eps       = amap.eps_rel * mag;
    if (kExactInts && mag < 8388608.0f) eps = 0.f;
    bool ok   = select_min ? (kth < worst_approx - eps) : (kth > worst_approx + eps);
    flag      = ok ? 0 : 1;
  }
  flags[qi] = flag;
  if (flag) atomicAdd(flags + nq, 1);
}

}  // namespace

template <typename T>
void row_norms(cudaStream_t stream, const T* x, int64_t n, int d, int64_t ld, float* out)
{
  if (n == 0) return;
  count_launch();
  row_norms_kernel<<<static_cast<unsigned>((n + 127) / 128), 128, 0, stream>>>(x, n, d, ld, out);
  B2_CUDA(cudaGetLastError());
}

void rsqrt_rows(cudaStream_t stream, const float* xn, int64_t n, float* out)
{
  if (n == 0) return;
  count_launch();
  rsqrt_rows_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(xn, out, n);
  B2_CUDA(cudaGetLastError());
}

void normalize_rows(cudaStream_t stream, float* x, int64_t n, int d, int64_t ld)
{
  if (n == 0) return;
  dbuf<float> inv(static_cast<size_t>(n), stream);
  row_norms(stream, x, n, d, ld, inv.data());
  rsqrt_rows(stream, inv.data(), n, inv.data());
  count_launch();
  scale_rows_kernel<<<static_cast<unsigned>((n * d + 255) / 256), 256, 0, stream>>>(x, n, d, ld, inv.data());
  B2_CUDA(cudaGetLastError());
}

template <typename T>
void exact_distance_tile(cudaStream_t stream, const float* q, int64_t nq, int64_t ldq, const T* x, int64_t n,
                         int64_t ldx, int d, const float* qn, const float* xn, cuvsDistanceType metric, float* out,
                         int64_t ldo, filter_view filt, int64_t q_row0, bool self_clamp)
{
  if (nq == 0 || n == 0) return;
  dim3 grid(static_cast<unsigned>((n + TN - 1) / TN), static_cast<unsigned>((nq + TM - 1) / TM));
  B2_EXPECTS(grid.y <= 65535, "exact_distance_tile: too many query rows per call");
  const bool sq = (metric == L2Unexpanded || metric == L2SqrtUnexpanded);
  count_launch();
  timed_section ts("exact_tile", stream);
  if (sq)
    exact_tile_kernel<true, T><<<grid, 256, 0, stream>>>(q, nq, ldq, x, n, ldx, d, qn, xn, int(metric), out, ldo, filt, q_row0,
                                                                         self_clamp);
  else
    exact_tile_kernel<false, T><<<grid, 256, 0, stream>>>(q, nq, ldq, x, n, ldx, d, qn, xn, int(metric), out, ldo, filt, q_row0,
                                                                         self_clamp);
  B2_CUDA(cudaGetLastError());
}

template <typename T>
void rescore_topk(cudaStream_t stream, const float* q, int64_t nq, int64_t ldq, const T* x, int64_t ldx, int d,
                  const float* qn, const float* xn, cuvsDistanceType metric, const uint32_t* cand_pos, int kc,
                  const int64_t* src_ids, int k, int64_t* out_idx, float* out_dist, int64_t pad_id, bool self_clamp)
{
  if (nq == 0) return;
  if (kc > kMaxCand) {
    B2_EXPECTS(kc <= kMaxCandBlock && k <= kc, "rescore_topk: candidate count %d out of range", kc);
    int kpow2 = 1;
    while (kpow2 < kc) kpow2 <<= 1;
    const size_t smem = static_cast<size_t>(kpow2) * (sizeof(int64_t) + sizeof(float) + sizeof(int));
    count_launch();
    rescore_block_kernel<T><<<static_cast<unsigned>(nq), 256, smem, stream>>>(q, ldq, x, ldx, d, qn, xn, int(metric), cand_pos, kc, kpow2,
                                                                          src_ids, k, out_idx, out_dist, pad_id, self_clamp);
    B2_CUDA(cudaGetLastError());
    return;
  }
  B2_EXPECTS(kc >= 1 && kc <= kMaxCand, "rescore_topk: candidate count %d out of range", kc);
  const int warps = 4;
  size_t smem     = static_cast<size_t>(warps) * kc * (sizeof(float) + sizeof(int64_t));
  count_launch();
  rescore_kernel<T><<<static_cast<unsigned>((nq + warps - 1) / warps), warps * 32, smem, stream>>>(
    q, nq, ldq, x, ldx, d, qn, xn, int(metric), cand_pos, kc, src_ids, k, out_idx, out_dist, pad_id, self_clamp);
  B2_CUDA(cudaGetLastError());
}

#define B2_EXACT_ROW_TYPE(T)                                                                                            \
  template void row_norms<T>(cudaStream_t, const T*, int64_t, int, int64_t, float*);                                  \
  template void exact_distance_tile<T>(cudaStream_t, const float*, int64_t, int64_t, const T*, int64_t, int64_t, int,    \
                                       const float*, const float*, cuvsDistanceType, float*, int64_t, filter_view, int64_t, bool); \
  template void rescore_topk<T>(cudaStream_t, const float*, int64_t, int64_t, const T*, int64_t, int, const float*,     \
                                const float*, cuvsDistanceType, const uint32_t*, int, const int64_t*, int, int64_t*, float*, \
                                int64_t, bool);
B2_EXACT_ROW_TYPE(float)
B2_EXACT_ROW_TYPE(__half)
B2_EXACT_ROW_TYPE(int8_t)
B2_EXACT_ROW_TYPE(uint8_t)
#undef B2_EXACT_ROW_TYPE

template <typename T>
void copy_rows(cudaStream_t s, const T* src, const int64_t* src_rows, T* dst, const int64_t* dst_rows, int64_t n, int64_t width)
{
  if (n == 0) return;
  count_launch();
  copy_rows_kernel<T><<<blocks_for(n * width, 256), 256, 0, s>>>(src, src_rows, dst, dst_rows, n, width);
  B2_CUDA(cudaGetLastError());
}
template void copy_rows<float>(cudaStream_t, const float*, const int64_t*, float*, const int64_t*, int64_t, int64_t);
template void copy_rows<int64_t>(cudaStream_t, const int64_t*, const int64_t*, int64_t*, const int64_t*, int64_t, int64_t);
template void copy_rows<uint32_t>(cudaStream_t, const uint32_t*, const int64_t*, uint32_t*, const int64_t*, int64_t, int64_t);

void rerun_flagged(cudaStream_t s, const int* flags, int64_t nq, int k, int64_t* out_idx, float* out_dist,
                   const std::function<void(const int64_t* rows, int64_t n, int64_t* idx, float* dist)>& answer)
{
  int n_flagged = 0;
  B2_CUDA(cudaMemcpyAsync(&n_flagged, flags + nq, sizeof(int), cudaMemcpyDeviceToHost, s));
  B2_CUDA(cudaStreamSynchronize(s));
  set_last_flagged(n_flagged);
  if (n_flagged == 0) return;
  std::vector<int> hflags(static_cast<size_t>(nq));
  B2_CUDA(cudaMemcpyAsync(hflags.data(), flags, sizeof(int) * nq, cudaMemcpyDeviceToHost, s));
  B2_CUDA(cudaStreamSynchronize(s));
  std::vector<int64_t> hrows;
  hrows.reserve(static_cast<size_t>(n_flagged));
  for (int64_t i = 0; i < nq; ++i)
    if (hflags[i]) hrows.push_back(i);
  dbuf<int64_t> rows(static_cast<size_t>(n_flagged), s);
  B2_CUDA(cudaMemcpyAsync(rows.data(), hrows.data(), sizeof(int64_t) * n_flagged, cudaMemcpyHostToDevice, s));
  dbuf<int64_t> fi(static_cast<size_t>(n_flagged) * k, s);
  dbuf<float> fd(static_cast<size_t>(n_flagged) * k, s);
  answer(rows.data(), n_flagged, fi.data(), fd.data());
  copy_rows(s, fi.data(), nullptr, out_idx, rows.data(), n_flagged, k);
  copy_rows(s, fd.data(), nullptr, out_dist, rows.data(), n_flagged, k);
  B2_CUDA(cudaStreamSynchronize(s));  // hrows is host memory read by the copy above
}

void list_floors(cudaStream_t s, const float* cs, int64_t nq, int64_t row_stride, int KC, float* out)
{
  if (nq == 0) return;
  count_launch();
  list_floor_kernel<<<blocks_for(nq * 32, 256), 256, 0, s>>>(cs, nq, row_stride, KC, out);
  B2_CUDA(cudaGetLastError());
}

void certify_candidates(cudaStream_t s, const float* cand_score, const uint32_t* cand_pos, int kc, const float* floor,
                        const float* qn, const float* out_dist, int k, const approx_map& amap, bool select_min, bool exact_ints,
                        int64_t nq, int* flags)
{
  B2_CUDA(cudaMemsetAsync(flags + nq, 0, sizeof(int), s));
  if (nq == 0) return;
  count_launch();
  auto kernel = exact_ints ? certify_kernel<true> : certify_kernel<false>;
  kernel<<<blocks_for(nq * 32, 256), 256, 0, s>>>(cand_score, cand_pos, kc, floor, qn, out_dist, k, amap, select_min, nq, flags);
  B2_CUDA(cudaGetLastError());
}

void postprocess_distances(cudaStream_t stream, float* dist, int64_t count, cuvsDistanceType metric)
{
  if (count == 0) return;
  if (metric != L2SqrtExpanded && metric != L2SqrtUnexpanded) return;
  count_launch();
  postprocess_kernel<<<static_cast<unsigned>((count + 255) / 256), 256, 0, stream>>>(dist, count, int(metric));
  B2_CUDA(cudaGetLastError());
}

}  // namespace b200
