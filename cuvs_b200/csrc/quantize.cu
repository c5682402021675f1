// Scalar and binary quantizers: cuvsScalarQuantizer* and cuvsBinaryQuantizer* behind the C boundary.
//
// Reference path: cpp/src/preprocessing/quantize/detail/scalar.cuh:33-123 (a quantile range found by sorting a row sample,
// then an elementwise map to int8) and detail/binary.cuh:38-389 (per-column thresholds: zero, the mean, or the median of a
// row sample found by transposing and sorting every column; then one bit per column), C wrappers
// c/src/preprocessing/quantize/{scalar,binary}.cpp.  Here:
//   - the transforms are streaming kernels at HBM speed: 16-byte loads, bits packed LSB first from lane groups, the
//     threshold row in shared memory; the inverse is a 256-entry table built once per call;
//   - the quantile and the medians are one exact radix select on order-preserving keys (8 bits per pass, per-column
//     histograms in shared memory), in place on a row-major sample: no sort, no transpose, no second copy;
//   - the column mean is a two-pass float64 reduction in a fixed order, the same for host and device inputs;
//   - sample rows are drawn on the host from a fixed seed and gathered from host or device memory, so both give one quantizer.
// Host inputs are streamed through bounded device buffers; nothing runs on the CPU but the row draw.  DESIGN.md "Quantizers".
#include "common.hpp"
#include "hash.cuh"
#include "timing.hpp"

#include <cuvs/preprocessing/quantize/binary.h>
#include <cuvs/preprocessing/quantize/scalar.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <type_traits>
#include <vector>

namespace b200 {
namespace {

constexpr size_t kHostChunkBytes = size_t(64) << 20;  // a host input's rows are staged through buffers of about this size
constexpr size_t kSampleBytes    = size_t(1) << 30;   // bound of a median sample's column chunk on the device
constexpr uint64_t kScalarSeed   = 137;
constexpr uint64_t kBinarySeed   = 29837;
constexpr int64_t kScalarSampleValues = 1000000;
constexpr int kThreads = 256;

// --------------------------------------------------------------------------------------------------------- element types
enum class ftype { f32 = 0, f16 = 1, f64 = 2 };

DLDataType dtype_of(ftype t)
{
  return {kDLFloat, static_cast<uint8_t>(t == ftype::f32 ? 32 : (t == ftype::f16 ? 16 : 64)), 1};
}
ftype ftype_of(const DLTensor& t, const char* what)
{
  if (dl_is(t, kDLFloat, 32)) return ftype::f32;
  if (dl_is(t, kDLFloat, 16)) return ftype::f16;
  if (dl_is(t, kDLFloat, 64)) return ftype::f64;
  B2_FAIL("%s must be float32, float16 or float64 (got dtype code %d, bits %d, lanes %d)", what, int(t.dtype.code),
          int(t.dtype.bits), int(t.dtype.lanes));
}
/** f(T{}) with T the element type of `t`: float, __half or double. */
template <typename F>
decltype(auto) with_ftype(ftype t, F&& f)
{
  switch (t) {
    case ftype::f16: return f(__half{});
    case ftype::f64: return f(double{});
    default: return f(float{});
  }
}

/** A quantizer's input or output: 2-D, C-contiguous, in device (true) or host (false) memory. */
bool check_matrix(const DLManagedTensor* m, const char* what)
{
  B2_EXPECTS(m != nullptr, "%s is null", what);
  const DLTensor& t = m->dl_tensor;
  B2_EXPECTS(t.ndim == 2, "%s must be a 2-D tensor (got %d dimensions)", what, int(t.ndim));
  B2_EXPECTS(dl_is_c_contiguous(t), "%s must be C-contiguous (row-major without strides)", what);
  B2_EXPECTS(t.shape[0] >= 0 && t.shape[1] >= 0, "%s has a negative extent", what);
  switch (t.device.device_type) {
    case kDLCUDA:
    case kDLCUDAManaged: return true;
    case kDLCPU:
    case kDLCUDAHost: return false;
    default: B2_FAIL("%s must be in host or CUDA device memory (got device type %d)", what, int(t.device.device_type));
  }
}
void check_same_memory(bool in_dev, bool out_dev)
{
  B2_EXPECTS(in_dev == out_dev, "the output must be in the same kind of memory as the input (input in %s memory, output in %s memory)",
             in_dev ? "device" : "host", out_dev ? "device" : "host");
}

// value compared in T's order (half through float: exact)
__device__ __forceinline__ float cmpv(float v) { return v; }
__device__ __forceinline__ float cmpv(__half v) { return __half2float(v); }
__device__ __forceinline__ double cmpv(double v) { return v; }
// correctly rounded double -> T
__device__ __forceinline__ void from_double(double v, float& o) { o = __double2float_rn(v); }
__device__ __forceinline__ void from_double(double v, __half& o) { o = __double2half(v); }
__device__ __forceinline__ void from_double(double v, double& o) { o = v; }
template <typename T>
__device__ __forceinline__ T to_t(double v)
{
  T o;
  from_double(v, o);
  return o;
}

// order-preserving unsigned keys: key(a) < key(b) iff a < b (with -0 below +0 and NaNs outside the infinities)
template <typename T>
struct radix_key;
template <>
struct radix_key<float> {
  using K = uint32_t;
  static constexpr int kBits = 32;
  __device__ static K key(float v) { const K b = __float_as_uint(v); return b ^ ((b >> 31) ? 0xffffffffu : 0x80000000u); }
  __device__ static float value(K k) { return __uint_as_float(k ^ ((k >> 31) ? 0x80000000u : 0xffffffffu)); }
};
template <>
struct radix_key<__half> {
  using K = uint16_t;
  static constexpr int kBits = 16;
  __device__ static K key(__half v)
  {
    const K b = __half_as_ushort(v);
    return static_cast<K>(b ^ ((b >> 15) ? 0xffffu : 0x8000u));
  }
  __device__ static __half value(K k) { return __ushort_as_half(static_cast<K>(k ^ ((k >> 15) ? 0x8000u : 0xffffu))); }
};
template <>
struct radix_key<double> {
  using K = uint64_t;
  static constexpr int kBits = 64;
  __device__ static K key(double v)
  {
    const K b = static_cast<K>(__double_as_longlong(v));
    return b ^ ((b >> 63) ? ~K(0) : (K(1) << 63));
  }
  __device__ static double value(K k) { return __longlong_as_double(static_cast<long long>(k ^ ((k >> 63) ? (K(1) << 63) : ~K(0)))); }
};

// ------------------------------------------------------------------------------------------------------------ row sample
/** `count` distinct row ids of [0, n), ascending, drawn with Floyd's algorithm from a counter-based generator seeded with
 *  `seed`; every row when count >= n.  The same on every machine. */
std::vector<int64_t> sample_rows(int64_t n, int64_t count, uint64_t seed)
{
  std::vector<int64_t> ids;
  if (count >= n) {
    ids.resize(static_cast<size_t>(n));
    for (int64_t i = 0; i < n; ++i) ids[i] = i;
    return ids;
  }
  std::vector<uint64_t> taken(static_cast<size_t>((n + 63) / 64), 0);
  for (int64_t j = n - count; j < n; ++j) {
    const uint64_t z = mix64(seed * 0x9e3779b97f4a7c15ull + static_cast<uint64_t>(j));
    int64_t t        = static_cast<int64_t>((static_cast<unsigned __int128>(z) * static_cast<uint64_t>(j + 1)) >> 64);
    if (taken[t >> 6] >> (t & 63) & 1) t = j;
    taken[t >> 6] |= uint64_t(1) << (t & 63);
  }
  ids.reserve(static_cast<size_t>(count));
  for (int64_t w = 0; w < static_cast<int64_t>(taken.size()); ++w)
    for (uint64_t b = taken[w]; b; b &= b - 1) ids.push_back(w * 64 + __builtin_ctzll(b));
  return ids;
}

template <typename T>
__global__ void gather_kernel(const T* __restrict__ x, int64_t d, const int64_t* __restrict__ ids, int64_t rows, int64_t c0, int64_t w,
                              T* __restrict__ out)
{
  const int64_t total = rows * w;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / w, c = i - r * w;
    out[i] = x[ids[r] * d + c0 + c];
  }
}

/** sample[i, :] = x[ids[i], c0 : c0 + w] on the device, from device or host rows (host rows are gathered in bounded pieces). */
template <typename T>
void gather_rows(resources* r, const T* x, bool dev, int64_t d, const std::vector<int64_t>& ids, const int64_t* dids, int64_t c0,
                 int64_t w, T* sample)
{
  const int64_t rows = static_cast<int64_t>(ids.size());
  if (dev) {
    count_launch();
    gather_kernel<T><<<static_cast<unsigned>(std::min<int64_t>(blocks_for(rows * w, kThreads), 4096)), kThreads, 0, r->stream>>>(
      x, d, dids, rows, c0, w, sample);
    B2_CUDA(cudaGetLastError());
    return;
  }
  const int64_t piece = std::max<int64_t>(1, static_cast<int64_t>(kHostChunkBytes / (sizeof(T) * w)));
  std::vector<T> stage(static_cast<size_t>(std::min(rows, piece) * w));
  for (int64_t i0 = 0; i0 < rows; i0 += piece) {
    const int64_t m = std::min(piece, rows - i0);
    for (int64_t i = 0; i < m; ++i) std::memcpy(&stage[i * w], x + ids[i0 + i] * d + c0, sizeof(T) * w);
    // from pageable memory the copy returns once `stage` has been read, so the next piece may overwrite it
    B2_CUDA(cudaMemcpyAsync(sample + i0 * w, stage.data(), sizeof(T) * m * w, cudaMemcpyHostToDevice, r->stream));
  }
}

// -------------------------------------------------------------------------------------------------- exact order statistic
constexpr int kSelTile = 32;                // columns per block
constexpr int kSelPitch = 257;              // per-column histogram stride in shared memory (257: columns on distinct banks)

template <typename T>
__global__ void __launch_bounds__(kThreads) radix_hist_kernel(const T* __restrict__ data, int64_t rows, int cols, int64_t ld,
                                                              int64_t cstride, int shift, const typename radix_key<T>::K* __restrict__ prefix,
                                                              int64_t rows_per_split, unsigned long long* __restrict__ hist)
{
  using RK = radix_key<T>;
  using K  = typename RK::K;
  __shared__ uint32_t h[kSelTile * kSelPitch];
  const int c0 = blockIdx.x * kSelTile;
  const int W  = min(kSelTile, cols - c0);
  int Wp       = 1;
  while (Wp < W) Wp <<= 1;
  for (int i = threadIdx.x; i < W * kSelPitch; i += blockDim.x) h[i] = 0;
  __syncthreads();
  const int c       = threadIdx.x & (Wp - 1);
  const int64_t r0  = blockIdx.y * rows_per_split;
  const int64_t r1  = min(rows, r0 + rows_per_split);
  const int hs      = shift + 8;  // key bits above this pass are fixed by the prefix
  if (c < W) {
    const K want      = prefix[c0 + c];
    const T* col      = data + (c0 + c) * cstride;
    const int64_t step = blockDim.x / Wp;
    for (int64_t r = r0 + threadIdx.x / Wp; r < r1; r += step) {
      const K k = RK::key(col[r * ld]);
      if (hs >= RK::kBits || (k >> hs) == (want >> hs)) atomicAdd(&h[c * kSelPitch + ((k >> shift) & 255)], 1u);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < W * 256; i += blockDim.x) {
    const uint32_t v = h[(i >> 8) * kSelPitch + (i & 255)];
    if (v) atomicAdd(&hist[static_cast<int64_t>(c0 + (i >> 8)) * 256 + (i & 255)], static_cast<unsigned long long>(v));
  }
}

/** Per column: the bin holding the rank-th smallest key among those matching the prefix; fixes that byte of the prefix,
 *  makes the rank relative to the bin, and clears the histogram for the next pass. */
template <typename K>
__global__ void radix_pick_kernel(int cols, int shift, unsigned long long* __restrict__ hist, K* __restrict__ prefix,
                                  unsigned long long* __restrict__ rank)
{
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  unsigned long long* hc = hist + static_cast<int64_t>(c) * 256;
  const unsigned long long k = rank[c];
  unsigned long long cum     = 0;
  int b                      = 0;
  for (; b < 255; ++b) {
    if (cum + hc[b] > k) break;
    cum += hc[b];
  }
  rank[c]   = k - cum;
  prefix[c] = static_cast<K>(prefix[c] | (static_cast<K>(b) << shift));
  for (int i = 0; i < 256; ++i) hc[i] = 0;
}

template <typename T>
__global__ void radix_emit_kernel(int cols, const typename radix_key<T>::K* __restrict__ prefix, T* __restrict__ out)
{
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < cols) out[c] = radix_key<T>::value(prefix[c]);
}

/**
 * out[c] = the ranks[c]-th smallest (0-based) of column c's `rows` values, exactly, where column c's value in row i is
 * data[i * ld + c * cstride].  A radix select: one pass per key byte, most significant first; each pass histograms, per
 * column, the byte of the keys whose higher bytes equal the column's prefix so far.  cstride 1 gives the columns of a
 * row-major matrix; cstride 0 gives `cols` ranks of one column.  The data are only read.
 */
template <typename T>
void select_ranks(resources* r, const T* data, int64_t rows, int cols, int64_t ld, int64_t cstride, const std::vector<int64_t>& ranks, T* out)
{
  using K  = typename radix_key<T>::K;
  auto s   = r->stream;
  dbuf<unsigned long long> hist(static_cast<size_t>(cols) * 256, s), rank(static_cast<size_t>(cols), s);
  dbuf<K> prefix(static_cast<size_t>(cols), s);
  std::vector<unsigned long long> rk(ranks.begin(), ranks.end());
  B2_CUDA(cudaMemcpyAsync(rank.data(), rk.data(), sizeof(unsigned long long) * cols, cudaMemcpyHostToDevice, s));
  B2_CUDA(cudaMemsetAsync(prefix.data(), 0, sizeof(K) * cols, s));
  B2_CUDA(cudaMemsetAsync(hist.data(), 0, sizeof(unsigned long long) * 256 * cols, s));
  const int tiles        = (cols + kSelTile - 1) / kSelTile;
  const int64_t want     = std::max<int64_t>(1, (4 * static_cast<int64_t>(r->sm_count > 0 ? r->sm_count : 132)) / tiles);
  const int64_t per      = std::max<int64_t>(1024, (rows + want - 1) / want);
  const int64_t splits   = (rows + per - 1) / per;
  B2_EXPECTS(splits < 65536, "order statistic: %lld rows are more than one pass can split", (long long)rows);
  for (int shift = radix_key<T>::kBits - 8; shift >= 0; shift -= 8) {
    count_launch(2);
    radix_hist_kernel<T><<<dim3(tiles, static_cast<unsigned>(splits)), kThreads, 0, s>>>(data, rows, cols, ld, cstride, shift, prefix.data(),
                                                                                         per, hist.data());
    radix_pick_kernel<K><<<blocks_for(cols, 128), 128, 0, s>>>(cols, shift, hist.data(), prefix.data(), rank.data());
  }
  count_launch();
  radix_emit_kernel<T><<<blocks_for(cols, 128), 128, 0, s>>>(cols, prefix.data(), out);
  B2_CUDA(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------ host rows, streamed
/** launch(in, out, rows) over all `n` rows: once on device pointers, or, for host data, chunk by chunk through bounded
 *  device buffers (in, kernel, out), returning once the host output is written. */
template <typename Launch>
void over_rows(resources* r, bool dev, const void* in, size_t in_row, void* out, size_t out_row, int64_t n, Launch&& launch)
{
  if (n == 0) return;
  if (dev) {
    launch(in, out, n);
    return;
  }
  auto s              = r->stream;
  const int64_t chunk = std::min<int64_t>(n, std::max<int64_t>(1, static_cast<int64_t>(kHostChunkBytes / std::max(in_row, out_row))));
  dbuf<char> din(static_cast<size_t>(chunk) * in_row, s), dout(static_cast<size_t>(chunk) * out_row, s);
  for (int64_t r0 = 0; r0 < n; r0 += chunk) {
    const int64_t m = std::min(chunk, n - r0);
    B2_CUDA(cudaMemcpyAsync(din.data(), static_cast<const char*>(in) + r0 * in_row, m * in_row, cudaMemcpyHostToDevice, s));
    launch(din.data(), dout.data(), m);
    B2_CUDA(cudaMemcpyAsync(static_cast<char*>(out) + r0 * out_row, dout.data(), m * out_row, cudaMemcpyDeviceToHost, s));
  }
  B2_CUDA(cudaStreamSynchronize(s));
}

unsigned stream_grid(resources* r, int64_t work_items, int per_block)
{
  const int64_t cap = 8 * static_cast<int64_t>(r->sm_count > 0 ? r->sm_count : 132);
  return static_cast<unsigned>(std::max<int64_t>(1, std::min(cap, (work_items + per_block - 1) / per_block)));
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// --------------------------------------------------------------------------------------------------------- bit packing
constexpr size_t kThrSmemBytes = 48 * 1024;  // threshold rows up to this size are kept in shared memory

/**
 * out[row, j / 8] bit j % 8 = x[row, j] > t[j] (t = 0 without thresholds); one warp per row.  Each lane holds V = 16 / sizeof(T)
 * consecutive columns (one 16-byte load when the row pitch and base allow it), so a byte of output spans G = 8 / V lanes and
 * is OR-ed together with G - 1 shuffles, least significant column first.  Bytes past ceil(d / 8) up to out_cols are zeroed.
 */
template <typename T, bool kThr>
__global__ void __launch_bounds__(kThreads) pack_bits_kernel(const T* __restrict__ x, int64_t n, int64_t d, const T* __restrict__ thr_g,
                                                             bool thr_smem, bool vec, uint8_t* __restrict__ out, int64_t out_cols)
{
  constexpr int V = 16 / static_cast<int>(sizeof(T));
  constexpr int G = 8 / V;
  extern __shared__ __align__(16) unsigned char smem[];
  const T* thr = thr_g;
  if (kThr && thr_smem) {
    T* st = reinterpret_cast<T*>(smem);
    for (int64_t j = threadIdx.x; j < d; j += blockDim.x) st[j] = thr_g[j];
    __syncthreads();
    thr = st;
  }
  const int lane       = threadIdx.x & 31;
  const int64_t nbytes = (d + 7) / 8;
  const int64_t warps  = static_cast<int64_t>(gridDim.x) * (blockDim.x >> 5);
  for (int64_t row = blockIdx.x * static_cast<int64_t>(blockDim.x >> 5) + (threadIdx.x >> 5); row < n; row += warps) {
    const T* xr   = x + row * d;
    uint8_t* orow = out + row * out_cols;
#pragma unroll 2
    for (int64_t c0 = 0; c0 < d; c0 += 32 * V) {
      const int64_t c = c0 + lane * V;
      alignas(16) T v[V];
      if (vec) {
        if (c < d) *reinterpret_cast<uint4*>(v) = __ldcs(reinterpret_cast<const uint4*>(xr + c));
      } else {
#pragma unroll
        for (int j = 0; j < V; ++j)
          if (c + j < d) v[j] = xr[c + j];
      }
      unsigned bits = 0;
#pragma unroll
      for (int j = 0; j < V; ++j) {
        if (c + j < d) {
          const auto t = kThr ? cmpv(thr[c + j]) : decltype(cmpv(v[j]))(0);
          if (cmpv(v[j]) > t) bits |= 1u << j;
        }
      }
      bits <<= V * (lane % G);
#pragma unroll
      for (int o = 1; o < G; o <<= 1) bits |= __shfl_xor_sync(0xffffffffu, bits, o);
      const int64_t b = c0 / 8 + lane / G;
      if (lane % G == 0 && b < nbytes) orow[b] = static_cast<uint8_t>(bits);
    }
    for (int64_t b = nbytes + lane; b < out_cols; b += 32) orow[b] = 0;
  }
}

template <typename T>
void pack_bits(resources* r, const T* x, int64_t n, int64_t d, const T* thr, uint8_t* out, int64_t out_cols)
{
  const bool vec      = (d * sizeof(T)) % 16 == 0 && aligned16(x);
  const bool thr_smem = thr != nullptr && d * sizeof(T) <= kThrSmemBytes;
  const size_t smem   = thr_smem ? d * sizeof(T) : 0;
  const unsigned grid = stream_grid(r, n, kThreads / 32);
  count_launch();
  if (thr)
    pack_bits_kernel<T, true><<<grid, kThreads, smem, r->stream>>>(x, n, d, thr, thr_smem, vec, out, out_cols);
  else
    pack_bits_kernel<T, false><<<grid, kThreads, 0, r->stream>>>(x, n, d, nullptr, false, vec, out, out_cols);
  B2_CUDA(cudaGetLastError());
}

// ----------------------------------------------------------------------------------------------------- scalar quantize
/** -128 at or below lo (and NaN), 127 at or above hi, else lroundf(float(scale * x + offset)) with the multiply and the add
 *  rounded separately. */
template <typename T>
__device__ __forceinline__ int8_t quantize_one(T xv, T lo, T hi, double scale, double offset)
{
  const auto x = cmpv(xv);
  if (!(x > cmpv(lo))) return -128;
  if (x >= cmpv(hi)) return 127;
  const double y = __dadd_rn(__dmul_rn(scale, static_cast<double>(x)), offset);
  return static_cast<int8_t>(lroundf(__double2float_rn(y)));
}

template <typename T>
__global__ void __launch_bounds__(kThreads) scalar_quantize_kernel(const T* __restrict__ x, int64_t count, T lo, T hi, double scale,
                                                                   double offset, bool vec, int8_t* __restrict__ out)
{
  constexpr int kLoads = static_cast<int>(sizeof(T));  // 16 elements = sizeof(T) 16-byte loads
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  const int64_t tid    = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t nvec   = vec ? count / 16 : 0;
  for (int64_t i = tid; i < nvec; i += stride) {
    alignas(16) T v[16];
    const uint4* src = reinterpret_cast<const uint4*>(x + i * 16);
#pragma unroll
    for (int k = 0; k < kLoads; ++k) reinterpret_cast<uint4*>(v)[k] = __ldcs(src + k);
    alignas(16) int8_t q[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) q[j] = quantize_one(v[j], lo, hi, scale, offset);
    __stcs(reinterpret_cast<uint4*>(out) + i, *reinterpret_cast<const uint4*>(q));
  }
  for (int64_t e = nvec * 16 + tid; e < count; e += stride) out[e] = quantize_one(x[e], lo, hi, scale, offset);
}

/** The table of the 256 codes' values, indexed by the code's byte: T((double(c) - offset) / scale), IEEE-rounded. */
template <typename T>
__global__ void inverse_table_kernel(double scale, double offset, T* __restrict__ table)
{
  const int byte = threadIdx.x;
  const double c = static_cast<double>(static_cast<int8_t>(static_cast<uint8_t>(byte)));
  table[byte]    = to_t<T>(__ddiv_rn(__dsub_rn(c, offset), scale));
}

template <int N>
struct code_vec;  // N codes in one load
template <>
struct code_vec<2> { using type = uint16_t; };
template <>
struct code_vec<4> { using type = uint32_t; };
template <>
struct code_vec<8> { using type = uint2; };

/** out[e] = table[codes[e]]; each step of a thread turns V = 16 / sizeof(T) codes into one 16-byte store, so a warp's loads and
 *  stores are both contiguous. */
template <typename T>
__global__ void __launch_bounds__(kThreads) inverse_lookup_kernel(const uint8_t* __restrict__ codes, int64_t count, const T* __restrict__ table_g,
                                                                  bool vec, T* __restrict__ out)
{
  constexpr int V = 16 / static_cast<int>(sizeof(T));
  using CV        = typename code_vec<V>::type;
  __shared__ T table[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) table[i] = table_g[i];
  __syncthreads();
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  const int64_t tid    = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t nvec   = vec ? count / V : 0;
#pragma unroll 4
  for (int64_t i = tid; i < nvec; i += stride) {
    alignas(8) uint8_t c[V];
    *reinterpret_cast<CV*>(c) = __ldcs(reinterpret_cast<const CV*>(codes) + i);
    alignas(16) T v[V];
#pragma unroll
    for (int j = 0; j < V; ++j) v[j] = table[c[j]];
    __stcs(reinterpret_cast<uint4*>(out) + i, *reinterpret_cast<const uint4*>(v));
  }
  for (int64_t e = nvec * V + tid; e < count; e += stride) out[e] = table[codes[e]];
}

// --------------------------------------------------------------------------------------------------------- column means
constexpr int kMeanThreads   = 128;
constexpr int64_t kMeanSplit = 1024;  // row blocks of the first pass (partial sums: kMeanSplit x d doubles)

/** partial[rb, c] = the sum, in row order, of x[r, c] over the rows of row block rb (rows_per_block rows from row 0 of x). */
template <typename T>
__global__ void __launch_bounds__(kMeanThreads) column_partial_kernel(const T* __restrict__ x, int64_t rows, int64_t d, int64_t rows_per_block,
                                                                      double* __restrict__ partial)
{
  const int64_t c = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (c >= d) return;
  const int64_t r0 = blockIdx.y * rows_per_block;
  const int64_t r1 = min(rows, r0 + rows_per_block);
  double acc       = 0.0;
#pragma unroll 8
  for (int64_t r = r0; r < r1; ++r) acc += static_cast<double>(cmpv(x[r * d + c]));
  partial[blockIdx.y * d + c] = acc;
}

template <typename T>
__global__ void column_mean_kernel(const double* __restrict__ partial, int64_t blocks, int64_t d, int64_t n, T* __restrict__ out)
{
  const int64_t c = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (c >= d) return;
  double acc = 0.0;
  for (int64_t b = 0; b < blocks; ++b) acc += partial[b * d + c];
  out[c] = to_t<T>(__ddiv_rn(acc, static_cast<double>(n)));
}

/** out[c] = T(sum_r x[r, c] / n): float64 sums over fixed row blocks, added in block order; host rows are streamed in
 *  whole row blocks, so host and device inputs give the same bits. */
template <typename T>
void column_means(resources* r, const T* x, bool dev, int64_t n, int64_t d, T* out)
{
  auto s                 = r->stream;
  const int64_t per      = (n + kMeanSplit - 1) / kMeanSplit;
  const int64_t blocks   = (n + per - 1) / per;
  dbuf<double> partial(static_cast<size_t>(blocks * d), s);
  const unsigned gx      = blocks_for(d, kMeanThreads);
  const int64_t row_size = d * static_cast<int64_t>(sizeof(T));
  // host rows: chunks of whole row blocks (at least one)
  const int64_t chunk_blocks = dev ? blocks : std::max<int64_t>(1, static_cast<int64_t>(kHostChunkBytes) / std::max<int64_t>(1, per * row_size));
  dbuf<T> staged;
  if (!dev) staged.alloc(static_cast<size_t>(std::min(blocks, chunk_blocks) * per * d), s);
  for (int64_t b0 = 0; b0 < blocks; b0 += chunk_blocks) {
    const int64_t nb   = std::min(chunk_blocks, blocks - b0);
    const int64_t r0   = b0 * per;
    const int64_t rows = std::min(n - r0, nb * per);
    const T* src       = x + r0 * d;
    if (!dev) {
      B2_CUDA(cudaMemcpyAsync(staged.data(), src, rows * row_size, cudaMemcpyHostToDevice, s));
      src = staged.data();
    }
    count_launch();
    column_partial_kernel<T><<<dim3(gx, static_cast<unsigned>(nb)), kMeanThreads, 0, s>>>(src, rows, d, per, partial.data() + b0 * d);
  }
  count_launch();
  column_mean_kernel<T><<<gx, kMeanThreads, 0, s>>>(partial.data(), blocks, d, n, out);
  B2_CUDA(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------------ binary quantizer
struct binary_quantizer {
  ftype type = ftype::f32;
  int threshold = ZERO;
  int64_t dim   = 0;
  owned<unsigned char> thr;  // dim values of `type` (MEAN, SAMPLING_MEDIAN)
};

/** The sample size of SAMPLING_MEDIAN: floor(n * ratio) (a float32 product), rounded up to even, at least 2, minus one;
 *  an odd count no larger than n. */
int64_t median_sample_size(int64_t n, float ratio)
{
  const int64_t m = static_cast<int64_t>(static_cast<float>(n) * ratio);
  int64_t s       = std::max<int64_t>((m + 1) / 2 * 2, 2) - 1;
  if (s > n) s = (n % 2) ? n : n - 1;
  return s;
}

void binary_train(resources* r, const cuvsBinaryQuantizerParams& p, DLManagedTensor* dataset, cuvsBinaryQuantizer_t handle)
{
  B2_EXPECTS(handle != nullptr, "quantizer is null");
  const bool dev    = check_matrix(dataset, "dataset");
  const DLTensor& t = dataset->dl_tensor;
  const ftype ft    = ftype_of(t, "dataset");
  const int64_t n = t.shape[0], d = t.shape[1];
  B2_EXPECTS(n >= 1 && d >= 1, "dataset must have at least one row and one column (got %lld x %lld)", (long long)n, (long long)d);
  B2_EXPECTS(p.threshold == ZERO || p.threshold == MEAN || p.threshold == SAMPLING_MEDIAN,
             "threshold must be ZERO, MEAN or SAMPLING_MEDIAN (got %d)", int(p.threshold));
  if (p.threshold == SAMPLING_MEDIAN)
    B2_EXPECTS(p.sampling_ratio > 0.0f && p.sampling_ratio <= 1.0f, "sampling_ratio must lie in (0, 1] (got %g)", double(p.sampling_ratio));
  auto q       = std::make_unique<binary_quantizer>();
  q->type      = ft;
  q->threshold = p.threshold;
  q->dim       = d;
  if (p.threshold != ZERO) {
    with_ftype(ft, [&](auto tag) {
      using T = decltype(tag);
      q->thr.alloc(sizeof(T) * d);
      T* thr    = reinterpret_cast<T*>(q->thr.data());
      const T* x = dl_ptr<const T>(t);
      if (p.threshold == MEAN) {
        column_means<T>(r, x, dev, n, d, thr);
        return;
      }
      const int64_t s = median_sample_size(n, p.sampling_ratio);
      const auto ids  = sample_rows(n, s, kBinarySeed);
      dbuf<int64_t> dids;
      if (dev) {
        dids.alloc(ids.size(), r->stream);
        B2_CUDA(cudaMemcpyAsync(dids.data(), ids.data(), sizeof(int64_t) * ids.size(), cudaMemcpyHostToDevice, r->stream));
      }
      const int64_t chunk = std::min<int64_t>(d, std::max<int64_t>(1, static_cast<int64_t>(kSampleBytes / (sizeof(T) * s))));
      dbuf<T> sample(static_cast<size_t>(s * chunk), r->stream);
      const std::vector<int64_t> ranks(static_cast<size_t>(chunk), (s - 1) / 2);
      for (int64_t c0 = 0; c0 < d; c0 += chunk) {
        const int64_t w = std::min(chunk, d - c0);
        gather_rows<T>(r, x, dev, d, ids, dids.data(), c0, w, sample.data());
        select_ranks<T>(r, sample.data(), s, static_cast<int>(w), w, 1, ranks, thr + c0);
      }
    });
  }
  set_index(handle, q.release(), dtype_of(ft));
}

void binary_transform(resources* r, const binary_quantizer* q, DLManagedTensor* dataset, DLManagedTensor* out)
{
  const bool dev     = check_matrix(dataset, "dataset");
  const bool out_dev = check_matrix(out, "output");
  const DLTensor& t  = dataset->dl_tensor;
  const DLTensor& o  = out->dl_tensor;
  const ftype ft     = ftype_of(t, "dataset");
  const int64_t n = t.shape[0], d = t.shape[1];
  const int64_t nbytes = (d + 7) / 8;
  B2_EXPECTS(dl_is(o, kDLUInt, 8), "output must be uint8 (got dtype code %d, bits %d)", int(o.dtype.code), int(o.dtype.bits));
  B2_EXPECTS(o.shape[0] >= n && o.shape[1] >= nbytes, "output must have at least %lld rows and %lld columns (got %lld x %lld)",
             (long long)n, (long long)nbytes, (long long)o.shape[0], (long long)o.shape[1]);
  check_same_memory(dev, out_dev);
  const void* thr = nullptr;
  if (q) {
    B2_EXPECTS(q->type == ft, "dataset is %s but the quantizer was trained on %s",
               ft == ftype::f32 ? "float32" : (ft == ftype::f16 ? "float16" : "float64"),
               q->type == ftype::f32 ? "float32" : (q->type == ftype::f16 ? "float16" : "float64"));
    if (q->threshold != ZERO) {
      B2_EXPECTS(d == q->dim, "dataset has %lld columns but the quantizer has %lld thresholds", (long long)d, (long long)q->dim);
      thr = q->thr.data();
    }
  }
  const int64_t out_cols = o.shape[1];
  with_ftype(ft, [&](auto tag) {
    using T = decltype(tag);
    over_rows(r, dev, t.data, sizeof(T) * d, o.data, static_cast<size_t>(out_cols), n, [&](const void* in, void* dst, int64_t rows) {
      pack_bits<T>(r, static_cast<const T*>(in), rows, d, static_cast<const T*>(thr), static_cast<uint8_t*>(dst), out_cols);
    });
  });
}

// ------------------------------------------------------------------------------------------------------ scalar quantizer
void scalar_train(resources* r, const cuvsScalarQuantizerParams& p, DLManagedTensor* dataset, cuvsScalarQuantizer* q)
{
  B2_EXPECTS(q != nullptr, "quantizer is null");
  B2_EXPECTS(p.quantile > 0.0f && p.quantile <= 1.0f, "quantile must lie in (0, 1] (got %g)", double(p.quantile));
  const bool dev    = check_matrix(dataset, "dataset");
  const DLTensor& t = dataset->dl_tensor;
  const ftype ft    = ftype_of(t, "dataset");
  const int64_t n = t.shape[0], d = t.shape[1];
  B2_EXPECTS(n >= 1 && d >= 1, "dataset must have at least one row and one column (got %lld x %lld)", (long long)n, (long long)d);
  const int64_t R   = std::min<int64_t>(n, std::max<int64_t>(1, kScalarSampleValues / d));
  const int64_t S   = R * d;
  const int64_t pmax = static_cast<int64_t>(std::ceil((0.5 + 0.5 * static_cast<double>(p.quantile)) * static_cast<double>(S))) - 1;
  const int64_t pmin = S - 1 - pmax;
  with_ftype(ft, [&](auto tag) {
    using T        = decltype(tag);
    const T* x     = dl_ptr<const T>(t);
    const auto ids = sample_rows(n, R, kScalarSeed);
    dbuf<int64_t> dids;
    if (dev) {
      dids.alloc(ids.size(), r->stream);
      B2_CUDA(cudaMemcpyAsync(dids.data(), ids.data(), sizeof(int64_t) * ids.size(), cudaMemcpyHostToDevice, r->stream));
    }
    dbuf<T> sample(static_cast<size_t>(S), r->stream), mm(2, r->stream);
    gather_rows<T>(r, x, dev, d, ids, dids.data(), 0, d, sample.data());
    select_ranks<T>(r, sample.data(), S, 2, 1, 0, {pmin, pmax}, mm.data());
    T h[2];
    B2_CUDA(cudaMemcpyAsync(h, mm.data(), sizeof(h), cudaMemcpyDeviceToHost, r->stream));
    B2_CUDA(cudaStreamSynchronize(r->stream));
    if constexpr (std::is_same_v<T, __half>) {
      q->min_ = static_cast<double>(__half2float(h[0]));
      q->max_ = static_cast<double>(__half2float(h[1]));
    } else {
      q->min_ = static_cast<double>(h[0]);
      q->max_ = static_cast<double>(h[1]);
    }
  });
}

/** lo = T(min_), hi = T(max_), widened to double; scale = 255 / (hi - lo) when hi > lo, else 1; offset = -128 - lo * scale. */
template <typename T>
void scalar_map(const cuvsScalarQuantizer* q, T& lo, T& hi, double& scale, double& offset)
{
  double l, h;
  if constexpr (std::is_same_v<T, __half>) {
    lo = __double2half(q->min_);
    hi = __double2half(q->max_);
    l  = __half2float(lo);
    h  = __half2float(hi);
  } else {
    lo = static_cast<T>(q->min_);
    hi = static_cast<T>(q->max_);
    l  = lo;
    h  = hi;
  }
  scale  = h > l ? 255.0 / (h - l) : 1.0;
  const double prod = l * scale;  // rounded before the subtraction: no fused multiply-add
  offset = -128.0 - prod;
}

void scalar_transform(resources* r, const cuvsScalarQuantizer* q, DLManagedTensor* dataset, DLManagedTensor* out)
{
  B2_EXPECTS(q != nullptr, "quantizer is null");
  const bool dev     = check_matrix(dataset, "dataset");
  const bool out_dev = check_matrix(out, "output");
  const DLTensor& t  = dataset->dl_tensor;
  const DLTensor& o  = out->dl_tensor;
  const ftype ft     = ftype_of(t, "dataset");
  B2_EXPECTS(dl_is(o, kDLInt, 8), "output must be int8 (got dtype code %d, bits %d)", int(o.dtype.code), int(o.dtype.bits));
  B2_EXPECTS(o.shape[0] == t.shape[0] && o.shape[1] == t.shape[1], "output must have the dataset's shape %lld x %lld (got %lld x %lld)",
             (long long)t.shape[0], (long long)t.shape[1], (long long)o.shape[0], (long long)o.shape[1]);
  check_same_memory(dev, out_dev);
  const int64_t n = t.shape[0], d = t.shape[1];
  with_ftype(ft, [&](auto tag) {
    using T = decltype(tag);
    T lo, hi;
    double scale, offset;
    scalar_map<T>(q, lo, hi, scale, offset);
    over_rows(r, dev, t.data, sizeof(T) * d, o.data, static_cast<size_t>(d), n, [&](const void* in, void* dst, int64_t rows) {
      const bool vec = aligned16(in) && aligned16(dst);
      count_launch();
      scalar_quantize_kernel<T><<<stream_grid(r, rows * d, kThreads * 16), kThreads, 0, r->stream>>>(
        static_cast<const T*>(in), rows * d, lo, hi, scale, offset, vec, static_cast<int8_t*>(dst));
      B2_CUDA(cudaGetLastError());
    });
  });
}

void scalar_inverse(resources* r, const cuvsScalarQuantizer* q, DLManagedTensor* dataset, DLManagedTensor* out)
{
  B2_EXPECTS(q != nullptr, "quantizer is null");
  const bool dev     = check_matrix(dataset, "dataset");
  const bool out_dev = check_matrix(out, "output");
  const DLTensor& t  = dataset->dl_tensor;
  const DLTensor& o  = out->dl_tensor;
  B2_EXPECTS(dl_is(t, kDLInt, 8), "dataset must be int8 codes (got dtype code %d, bits %d)", int(t.dtype.code), int(t.dtype.bits));
  const ftype ft = ftype_of(o, "output");
  B2_EXPECTS(o.shape[0] == t.shape[0] && o.shape[1] == t.shape[1], "output must have the dataset's shape %lld x %lld (got %lld x %lld)",
             (long long)t.shape[0], (long long)t.shape[1], (long long)o.shape[0], (long long)o.shape[1]);
  check_same_memory(dev, out_dev);
  const int64_t n = t.shape[0], d = t.shape[1];
  with_ftype(ft, [&](auto tag) {
    using T = decltype(tag);
    T lo, hi;
    double scale, offset;
    scalar_map<T>(q, lo, hi, scale, offset);
    dbuf<T> table(256, r->stream);
    count_launch();
    inverse_table_kernel<T><<<1, 256, 0, r->stream>>>(scale, offset, table.data());
    over_rows(r, dev, t.data, static_cast<size_t>(d), o.data, sizeof(T) * d, n, [&](const void* in, void* dst, int64_t rows) {
      const bool vec = aligned16(in) && aligned16(dst);
      count_launch();
      inverse_lookup_kernel<T><<<stream_grid(r, rows * d, kThreads * (16 / static_cast<int>(sizeof(T)))), kThreads, 0, r->stream>>>(
        static_cast<const uint8_t*>(in), rows * d, table.data(), vec, static_cast<T*>(dst));
      B2_CUDA(cudaGetLastError());
    });
  });
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

cuvsError_t cuvsScalarQuantizerParamsCreate(cuvsScalarQuantizerParams_t* params)
{
  return guarded([=] {
    B2_EXPECTS(params != nullptr, "params is null");
    *params = new cuvsScalarQuantizerParams{0.99f};
  });
}
cuvsError_t cuvsScalarQuantizerParamsDestroy(cuvsScalarQuantizerParams_t params) { return guarded([=] { delete params; }); }

cuvsError_t cuvsScalarQuantizerCreate(cuvsScalarQuantizer_t* quantizer)
{
  return guarded([=] {
    B2_EXPECTS(quantizer != nullptr, "quantizer is null");
    *quantizer = new cuvsScalarQuantizer{0.0, 0.0};
  });
}
cuvsError_t cuvsScalarQuantizerDestroy(cuvsScalarQuantizer_t quantizer) { return guarded([=] { delete quantizer; }); }

cuvsError_t cuvsScalarQuantizerTrain(cuvsResources_t res, cuvsScalarQuantizerParams_t params, DLManagedTensor* dataset,
                                     cuvsScalarQuantizer_t quantizer)
{
  return guarded([=] {
    B2_EXPECTS(params != nullptr, "params is null");
    scalar_train(as_res(res), *params, dataset, quantizer);
  });
}
cuvsError_t cuvsScalarQuantizerTransform(cuvsResources_t res, cuvsScalarQuantizer_t quantizer, DLManagedTensor* dataset, DLManagedTensor* out)
{
  return guarded([=] { scalar_transform(as_res(res), quantizer, dataset, out); });
}
cuvsError_t cuvsScalarQuantizerInverseTransform(cuvsResources_t res, cuvsScalarQuantizer_t quantizer, DLManagedTensor* dataset,
                                                DLManagedTensor* out)
{
  return guarded([=] { scalar_inverse(as_res(res), quantizer, dataset, out); });
}

cuvsError_t cuvsBinaryQuantizerParamsCreate(cuvsBinaryQuantizerParams_t* params)
{
  return guarded([=] {
    B2_EXPECTS(params != nullptr, "params is null");
    // defaults of c/src/preprocessing/quantize/binary.cpp:95-101
    *params = new cuvsBinaryQuantizerParams{MEAN, 0.1f};
  });
}
cuvsError_t cuvsBinaryQuantizerParamsDestroy(cuvsBinaryQuantizerParams_t params) { return guarded([=] { delete params; }); }

cuvsError_t cuvsBinaryQuantizerCreate(cuvsBinaryQuantizer_t* quantizer)
{
  return guarded([=] {
    B2_EXPECTS(quantizer != nullptr, "quantizer is null");
    *quantizer = new cuvsBinaryQuantizer{0, {kDLFloat, 32, 1}};
  });
}
cuvsError_t cuvsBinaryQuantizerDestroy(cuvsBinaryQuantizer_t quantizer)
{
  return guarded([=] {
    if (quantizer == nullptr) return;
    drop_index<binary_quantizer>(quantizer);  // the thresholds go with the handle
    delete quantizer;
  });
}

cuvsError_t cuvsBinaryQuantizerTrain(cuvsResources_t res, cuvsBinaryQuantizerParams_t params, DLManagedTensor* dataset,
                                     cuvsBinaryQuantizer_t quantizer)
{
  return guarded([=] {
    B2_EXPECTS(params != nullptr, "params is null");
    binary_train(as_res(res), *params, dataset, quantizer);
  });
}
cuvsError_t cuvsBinaryQuantizerTransform(cuvsResources_t res, DLManagedTensor* dataset, DLManagedTensor* out)
{
  return guarded([=] { binary_transform(as_res(res), nullptr, dataset, out); });
}
cuvsError_t cuvsBinaryQuantizerTransformWithParams(cuvsResources_t res, cuvsBinaryQuantizer_t quantizer, DLManagedTensor* dataset,
                                                   DLManagedTensor* out)
{
  return guarded([=] {
    B2_EXPECTS(quantizer != nullptr && quantizer->addr != 0, "the binary quantizer is not trained");
    binary_transform(as_res(res), &index_of<binary_quantizer>(quantizer), dataset, out);
  });
}

}  // extern "C"
