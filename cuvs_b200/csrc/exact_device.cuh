// Device side of the exact fp32 layer (exact.cuh).  Every kernel that must return oracle/oracle.c's bits scores a candidate
// with exact_accumulate and finish_distance, so the re-score and the exact fallbacks cannot drift apart.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstdint>

#include <cuvs/distance/distance.h>

namespace b200 {

/** The distance in selection form from exact_accumulate's sum.  Expanded L2 is clamped at 0 and, with `self_clamp` (searches:
 *  l2_exp.cuh's self-neighbour rule), zeroed below 1e-3 between rows of equal norm; k-means assignment, like
 *  oracle_kmeans_assign, clamps at 0 only. */
__device__ __forceinline__ float finish_distance(float acc, float qn, float xn, int metric, bool self_clamp = true)
{
  switch (metric) {
    case L2Expanded:
    case L2SqrtExpanded: {
      float val = fmaf(-2.0f, acc, qn + xn);
      if (!(val > 0.0f)) val = 0.0f;
      if (self_clamp && val * val < 1e-6f && qn == xn) val = 0.0f;
      return val;
    }
    case CosineExpanded: return 1.0f - acc / (sqrtf(qn) * sqrtf(xn));
    default: return acc;  // InnerProduct, L2Unexpanded (acc already holds the sum of squares)
  }
}

/** Whether exact_accumulate may read the rows of q [., ldq] and x [., ldx] as float4: d, ldq and ldx multiples of 4 and both
 *  bases 16-byte aligned.  Either form accumulates in the same order, so the choice never changes a bit of the result. */
__device__ __forceinline__ bool exact_vec4(const float* q, int64_t ldq, const float* x, int64_t ldx, int d)
{
  return ((d & 3) == 0) && ((ldx & 3) == 0) && ((ldq & 3) == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0) &&
         ((reinterpret_cast<uintptr_t>(q) & 15) == 0);
}

/** The oracle's sum over the components of qr and xr, one fmaf each in ascending order: squared differences for the unexpanded
 *  L2 metrics, products otherwise.  finish_distance(sum, |q|^2, |x|^2, metric) is then the distance in selection form. */
__device__ __forceinline__ float exact_accumulate(const float* __restrict__ qr, const float* __restrict__ xr, int d, bool vec4,
                                                  int metric)
{
  const bool sqdiff = (metric == L2Unexpanded || metric == L2SqrtUnexpanded);
  float acc         = 0.f;
  if (vec4) {
    const float4* x4 = reinterpret_cast<const float4*>(xr);
    const float4* q4 = reinterpret_cast<const float4*>(qr);
    for (int kk = 0; kk < d / 4; ++kk) {
      float4 a = q4[kk], b = x4[kk];
      if (sqdiff) {
        float t;
        t = a.x - b.x; acc = fmaf(t, t, acc);
        t = a.y - b.y; acc = fmaf(t, t, acc);
        t = a.z - b.z; acc = fmaf(t, t, acc);
        t = a.w - b.w; acc = fmaf(t, t, acc);
      } else {
        acc = fmaf(a.x, b.x, acc);
        acc = fmaf(a.y, b.y, acc);
        acc = fmaf(a.z, b.z, acc);
        acc = fmaf(a.w, b.w, acc);
      }
    }
  } else {
    for (int kk = 0; kk < d; ++kk) {
      if (sqdiff) { float t = qr[kk] - xr[kk]; acc = fmaf(t, t, acc); }
      else acc = fmaf(qr[kk], xr[kk], acc);
    }
  }
  return acc;
}

/** A row element as fp32: every float16, int8 and uint8 value is exactly representable, so the narrow row types give the
 *  same sums as their widened fp32 copies. */
__device__ __forceinline__ float widen(float v) { return v; }
__device__ __forceinline__ float widen(__half v) { return __half2float(v); }
__device__ __forceinline__ float widen(int8_t v) { return static_cast<float>(v); }
__device__ __forceinline__ float widen(uint8_t v) { return static_cast<float>(v); }

/** exact_accumulate over rows stored as float16, int8 or uint8: each element widened on load, same order and fmaf as above. */
template <typename T>
__device__ __forceinline__ float exact_accumulate(const float* __restrict__ qr, const T* __restrict__ xr, int d, bool, int metric)
{
  const bool sqdiff = (metric == L2Unexpanded || metric == L2SqrtUnexpanded);
  float acc         = 0.f;
  for (int kk = 0; kk < d; ++kk) {
    const float x = widen(xr[kk]);
    if (sqdiff) { float t = qr[kk] - x; acc = fmaf(t, t, acc); }
    else acc = fmaf(qr[kk], x, acc);
  }
  return acc;
}

/** Bitonic sort, by the whole block, of the n (a power of two) entries (sd, si, and slot when not null) in shared memory:
 *  entry i goes before entry j when before(i, j), a strict total order.  Ends with __syncthreads(). */
template <typename Before>
__device__ __forceinline__ void block_bitonic_sort(float* sd, int64_t* si, int* slot, int n, Before before)
{
  for (int size = 2; size <= n; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = threadIdx.x; i < (n >> 1); i += blockDim.x) {
        const int lo = (i / stride) * (stride << 1) + (i % stride), hi = lo + stride;
        const bool up = (lo & size) == 0;
        if (before(hi, lo) == up) {
          const float td = sd[lo]; sd[lo] = sd[hi]; sd[hi] = td;
          const int64_t ti = si[lo]; si[lo] = si[hi]; si[hi] = ti;
          if (slot) { const int tc = slot[lo]; slot[lo] = slot[hi]; slot[hi] = tc; }
        }
      }
      __syncthreads();
    }
  }
}

}  // namespace b200
