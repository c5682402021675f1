// NN-descent (cuvsNNDescentBuild and CAGRA's build_algo = NN_DESCENT): an approximate kNN graph of all rows, built and
// refined entirely on the device.
//
// Reference: cpp/src/neighbors/detail/nn_descent.cuh (GNND), C wrapper c/src/neighbors/nn_descent.cpp.  The reference keeps
// its sample lists and reverse graph in pinned host memory and builds them on the host; here every step is a kernel and
// only the per-iteration update count crosses to the host.  The semantics are deterministic (the same graph bits on every
// run, whatever the thread scheduling); DESIGN.md "NN-descent" states them and tests/nn_descent_ref.py restates them in numpy.
//
// State: per row u a list L(u) of Ki keys, sorted ascending, key = (ordered dist << 32) | id, with two flag bits in the id
// word: kNew (not yet sampled as new) and kFresh (entered during the current iteration; counted, then cleared).
// Per iteration t:
//   sample_kernel      new(u): first S new entries (marked old), old(u): first S entries old at the start
//   reverse            Rnew(v) / Rold(v): the S sources u with the smallest (hash(t, u, v), u), grouped by target
//   join_kernel        one warpgroup per row: N = new ∪ Rnew, O = (old ∪ Rold) \ N, the N x (N ∪ O) distance block
//                      (wgmma on fp16 / 8-bit rows), one
//                      proposal per candidate (its best partner), rejected early against the target's live worst entry
//   merge_kernel       one CTA per target: top-Ki of the list and its proposals, duplicates removed
//   fresh_count_kernel the number of ids that entered a list
// Then every list is re-scored exactly (rescore_topk) and the best `degree` entries kept.
#include "exact.cuh"
#include "hash.cuh"
#include "nn_descent.cuh"
#include "ptx_sm90.cuh"
#include "timing.hpp"

#include <cuda_fp16.h>

#include <cub/device/device_scan.cuh>

#include <cuvs/neighbors/nn_descent.h>

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <memory>
#include <type_traits>

namespace b200 {
namespace {

constexpr int kS               = 32;   // samples per list
constexpr int kMaxKi           = 1024; // list length: merge keeps two lists of Ki keys in shared memory
constexpr int kJoinThreads     = 128;  // one thread per candidate slot: N in [0, 64), O in [64, 128)
constexpr int kDimChunk        = 32;   // columns staged per step of the join
constexpr uint32_t kInvalid    = 0xffffffffu;
constexpr uint32_t kNew        = 1u << 31;
constexpr uint32_t kFresh      = 1u << 30;
constexpr uint32_t kIdMask     = kFresh - 1;
constexpr uint64_t kKeyMask    = ~static_cast<uint64_t>(kNew | kFresh);
constexpr uint64_t kNoKey      = ~0ull;
constexpr uint64_t kInitSeed   = 0x6e6e2d696e697400ull;
constexpr uint64_t kRevSeed    = 0x6e6e2d7265760000ull;
enum dist_kind { kL2 = 0, kIP = 1, kCos = 2, kHam = 3 };  // kHam: bitwise Hamming over 8-bit rows

__device__ __forceinline__ uint32_t ord_f(float f)
{
  const uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ uint64_t make_key(float d, uint32_t id) { return (static_cast<uint64_t>(ord_f(d)) << 32) | id; }

// ---- the one distance function: d(a, b) of the unordered pair, in selection form, the same bits wherever it is evaluated
template <typename T> struct acc_of { using type = float; };
template <> struct acc_of<int8_t> { using type = int; };
template <> struct acc_of<uint8_t> { using type = int; };
__device__ __forceinline__ float as_acc(float v, float) { return v; }
__device__ __forceinline__ float as_acc(__half v, float) { return __half2float(v); }
__device__ __forceinline__ int as_acc(int8_t v, int) { return v; }
__device__ __forceinline__ int as_acc(uint8_t v, int) { return v; }
template <typename T> __device__ __forceinline__ typename acc_of<T>::type load_acc(T v) { return as_acc(v, typename acc_of<T>::type{}); }

__device__ __forceinline__ void accumulate(float& acc, float a, float b, bool l2)
{
  if (l2) {
    const float t = __fsub_rn(a, b);
    acc           = fmaf(t, t, acc);
  } else {
    acc = fmaf(a, b, acc);
  }
}
__device__ __forceinline__ void accumulate(int& acc, int a, int b, bool l2)
{
  if (l2) {
    const int t = a - b;
    acc += t * t;
  } else {
    acc += a * b;
  }
}
// cosine: 1 - dot * (inv_a * inv_b), symmetric in a and b; unit rows pass no inverse norms
template <typename A>
__device__ __forceinline__ float finish(A acc, int kind, const float* inv, uint32_t a, uint32_t b)
{
  const float v = static_cast<float>(acc);
  if (kind == kL2) return v;
  if (kind == kIP) return -v;
  const float s = inv ? __fmul_rn(inv[a], inv[b]) : 1.0f;
  return __fsub_rn(1.0f, __fmul_rn(v, s));
}

template <typename T>
__device__ __forceinline__ float pair_dist(const T* __restrict__ x, int64_t ld, int d, int kind, const float* inv, uint32_t a, uint32_t b)
{
  const T* ra = x + a * ld;
  const T* rb = x + b * ld;
  typename acc_of<T>::type acc = 0;
  for (int k = 0; k < d; ++k) accumulate(acc, load_acc(ra[k]), load_acc(rb[k]), kind == kL2);
  return finish(acc, kind, inv, a, b);
}

__device__ __forceinline__ uint32_t lanemask_lt() { return (1u << (threadIdx.x & 31)) - 1u; }

// ascending bitonic sort of n (a power of two) keys in shared memory by the whole block; ends synchronised
__device__ void block_sort_keys(uint64_t* k, int n)
{
  for (int size = 2; size <= n; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = threadIdx.x; i < (n >> 1); i += blockDim.x) {
        const int lo = (i / stride) * (stride << 1) + (i % stride), hi = lo + stride;
        const bool up = (lo & size) == 0;
        const uint64_t a = k[lo], b = k[hi];
        if ((a > b) == up) { k[lo] = b; k[hi] = a; }
      }
      __syncthreads();
    }
  }
}

// ascending bitonic sort of one key per lane (32 keys) across the warp
__device__ __forceinline__ uint64_t warp_sort_key(uint64_t v)
{
  const int lane = threadIdx.x & 31;
  for (int size = 2; size <= 32; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      const uint64_t o  = __shfl_xor_sync(0xffffffffu, v, stride);
      const bool up     = (lane & size) == 0 || size == 32;
      const bool low    = (lane & stride) == 0;
      v = (low == up) ? min(v, o) : max(v, o);
    }
  }
  return v;
}

// number of entries of the ascending array a[0, len) (flag bits masked off) below key
__device__ __forceinline__ int count_below(const uint64_t* a, int len, uint64_t key)
{
  int lo = 0, hi = len;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if ((a[mid] & kKeyMask) < key) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// ---- the tensor-core form of d for fp16 and 8-bit join rows: from the Gram entry g = <a, b> of a wgmma block (fp32
// accumulate of exact fp16 products, or exact s32) and per-row squared norms; every term is symmetric in a and b, and a
// Gram entry depends only on the two rows, so d has the same bits at any block position and in either operand order.
// Hamming: g = popc(a AND b) from the binary wgmma and per-row popcounts in place of the norms,
// popc(a XOR b) = popc(a) + popc(b) - 2 popc(a AND b), an exact integer.
__device__ __forceinline__ float tc_finish(float g, int kind, const float* nrm, const int*, const float*, uint32_t a, uint32_t b)
{
  if (kind == kL2) return fmaf(-2.0f, g, __fadd_rn(nrm[a], nrm[b]));
  if (kind == kIP) return -g;
  return __fsub_rn(1.0f, g);  // unit rows
}
__device__ __forceinline__ float tc_finish(int g, int kind, const float*, const int* nrm, const float* inv, uint32_t a, uint32_t b)
{
  if (kind == kL2) return static_cast<float>(static_cast<int64_t>(nrm[a]) + nrm[b] - 2 * static_cast<int64_t>(g));
  if (kind == kIP) return -static_cast<float>(g);
  if (kind == kHam) return static_cast<float>(nrm[a] + nrm[b] - 2 * g);
  return __fsub_rn(1.0f, __fmul_rn(static_cast<float>(g), __fmul_rn(inv[a], inv[b])));
}

template <typename T> struct tc_acc { using type = float; };
template <> struct tc_acc<int8_t> { using type = int; };
template <> struct tc_acc<uint8_t> { using type = int; };

constexpr int kTcTileBytes = 128 * 128;  // 128 rows x 128 bytes (64 fp16 or 128 8-bit columns), SWIZZLE_128B

// Stages k-block kb of the rows ids[0, 128) (kInvalid: a zero row; columns past d are zero) as a K-major SWIZZLE_128B tile:
// the 16-byte chunk c of row r sits at chunk c ^ (r % 8) of the row's 128 bytes.
template <typename T>
__device__ __forceinline__ void stage_kblock(unsigned char* tile, const T* __restrict__ x, int64_t ld, int d, int kb, const uint32_t* ids)
{
  using R          = typename std::conditional<sizeof(T) == 2, uint16_t, uint8_t>::type;
  constexpr int per = 16 / static_cast<int>(sizeof(T));
  const R* xr      = reinterpret_cast<const R*>(x);
  for (int q = threadIdx.x; q < 128 * 8; q += blockDim.x) {
    const int r = q >> 3, c = q & 7;
    const uint32_t id = ids[r];
    const int col0    = kb * 8 * per + c * per;
    alignas(16) R e[per];
#pragma unroll
    for (int i = 0; i < per; ++i) e[i] = (id != kInvalid && col0 + i < d) ? xr[static_cast<int64_t>(id) * ld + col0 + i] : R(0);
    *reinterpret_cast<uint4*>(tile + r * 128 + ((c ^ (r & 7)) << 4)) = *reinterpret_cast<const uint4*>(e);
  }
}

// G[64 x 128] = rows [0, 64) x rows [0, 128) of ids over all d columns: m64n128k16 fp16 with fp32 accumulate, or m64n128k32
// s8 / u8 with s32, or (ham, 8-bit rows) m64n128k256 b1 AND-popcount with s32.  Issued by the whole warpgroup (the CTA); `g`
// holds ptx::wgmma_bf16<128>'s fragment layout.
template <typename T>
__device__ __forceinline__ void gram_block(unsigned char* tile, const T* __restrict__ x, int64_t ld, int d, const uint32_t* ids, float (&g)[64],
                                           bool ham)
{
  const int nkb     = static_cast<int>((static_cast<int64_t>(d) * sizeof(T) + 127) / 128);
  const uint32_t lo = ptx::smem_desc_lo(ptx::smem_u32(tile));
  for (int kb = 0; kb < nkb; ++kb) {
    stage_kblock(tile, x, ld, d, kb, ids);
    ptx::fence_proxy_async();
    __syncthreads();
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {  // +2 per 32-byte K step (k16 fp16, k32 8-bit, k256 bits)
      const uint64_t dsc = ptx::desc(lo + k * 2, ptx::kDescHiSw128);
      if constexpr (std::is_same<T, __half>::value) ptx::wgmma_f16_128(g, dsc, dsc, (kb | k) != 0 ? 1u : 0u);
      else if (ham) ptx::wgmma_b1_128(reinterpret_cast<uint32_t(&)[64]>(g), dsc, dsc, (kb | k) != 0 ? 1u : 0u);
      else ptx::wgmma_i8_128<std::is_same<T, uint8_t>::value>(reinterpret_cast<uint32_t(&)[64]>(g), dsc, dsc, (kb | k) != 0 ? 1u : 0u);
    }
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    __syncthreads();
  }
}

template <typename G> __device__ __forceinline__ G gram_at(const float (&g)[64], int i) { return reinterpret_cast<const G(&)[64]>(g)[i]; }

// ---------------------------------------------------------------------------------------------------------------- init
// One CTA per row: warp 0 draws the ids (candidate j of row u is mix64(seed ^ (u << 32 | j)) mod (n - 1), an index into the
// rows other than u; repeats are skipped until Ki ids are distinct), then the block scores and sorts them.
__device__ __forceinline__ void draw_ids(uint32_t u, int64_t n, int Ki, uint32_t* ids)
{
  const int lane = threadIdx.x;
  int cnt = 0;
  for (uint64_t j0 = 0; cnt < Ki; j0 += 32) {
    const uint64_t h = mix64(kInitSeed ^ ((static_cast<uint64_t>(u) << 32) | (j0 + lane)));
    const uint32_t c = static_cast<uint32_t>(h % static_cast<uint64_t>(n - 1));
    const uint32_t id = c + (c >= u ? 1u : 0u);
    bool dup = false;
    for (int e = 0; e < cnt; ++e) dup |= ids[e] == id;
    const uint32_t peers = __match_any_sync(0xffffffffu, id);
    const bool ok       = !dup && (__ffs(peers) - 1) == lane;
    const uint32_t b    = __ballot_sync(0xffffffffu, ok);
    const int rank      = __popc(b & lanemask_lt());
    if (ok && cnt + rank < Ki) ids[cnt + rank] = id;
    cnt = min(Ki, cnt + __popc(b));
    __syncwarp();
  }
}

// fp32 join rows: the list's distances with pair_dist
template <typename T>
__global__ void __launch_bounds__(128) init_kernel(const T* __restrict__ x, int64_t ld, int d, int kind, const float* __restrict__ inv, int64_t n,
                                                   int Ki, int KiP, uint64_t* __restrict__ L)
{
  extern __shared__ __align__(16) uint64_t init_smem[];
  uint64_t* keys = init_smem;                                   // [KiP]
  uint32_t* ids  = reinterpret_cast<uint32_t*>(keys + KiP);     // [Ki]
  const uint32_t u = blockIdx.x;
  if (threadIdx.x < 32) draw_ids(u, n, Ki, ids);
  __syncthreads();
  for (int e = threadIdx.x; e < KiP; e += blockDim.x) {
    if (e < Ki) {
      const uint32_t id = ids[e];
      keys[e] = make_key(pair_dist(x, ld, d, kind, inv, u, id), id);
    } else {
      keys[e] = kNoKey;
    }
  }
  __syncthreads();
  block_sort_keys(keys, KiP);
  for (int e = threadIdx.x; e < Ki; e += blockDim.x) L[static_cast<int64_t>(u) * Ki + e] = keys[e] | kNew;
}

// fp16 and 8-bit join rows: the list's distances from Gram blocks as the join forms them, u as row 0 and 127 ids per block
template <typename T>
__global__ void __launch_bounds__(128) init_tc_kernel(const T* __restrict__ x, int64_t ld, int d, int kind, const float* __restrict__ nrm_f,
                                                      const int* __restrict__ nrm_i, const float* __restrict__ inv, int64_t n, int Ki, int KiP,
                                                      uint64_t* __restrict__ L)
{
  using G = typename tc_acc<T>::type;
  __shared__ __align__(1024) unsigned char tile[kTcTileBytes];
  __shared__ uint32_t rows[128];
  extern __shared__ __align__(16) uint64_t init_smem[];
  uint64_t* keys = init_smem;                                   // [KiP]
  uint32_t* ids  = reinterpret_cast<uint32_t*>(keys + KiP);     // [Ki]
  const uint32_t u = blockIdx.x;
  const int t = threadIdx.x, lane = t & 31;
  if (t < 32) draw_ids(u, n, Ki, ids);
  for (int e = t; e < KiP; e += blockDim.x) keys[e] = kNoKey;
  __syncthreads();
  for (int e0 = 0; e0 < Ki; e0 += 127) {
    rows[t] = t == 0 ? u : (e0 + t - 1 < Ki ? ids[e0 + t - 1] : kInvalid);
    __syncthreads();
    float g[64];
    gram_block(tile, x, ld, d, rows, g, kind == kHam);
    if (t < 4) {  // row 0 of the block: warp 0, lanes 0..3
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int c = 8 * j + 2 * lane + h, e = e0 + c - 1;
          if (c >= 1 && e < Ki) keys[e] = make_key(tc_finish(gram_at<G>(g, 4 * j + h), kind, nrm_f, nrm_i, inv, u, ids[e]), ids[e]);
        }
    }
    __syncthreads();
  }
  block_sort_keys(keys, KiP);
  for (int e = t; e < Ki; e += blockDim.x) L[static_cast<int64_t>(u) * Ki + e] = keys[e] | kNew;
}

// -------------------------------------------------------------------------------------------------------------- sample
// One warp per row: new(u) = the first S new entries in list order, which are then marked old; old(u) = the first S
// entries that were old when the iteration started.
__global__ void sample_kernel(uint64_t* __restrict__ L, int64_t n, int Ki, uint32_t* __restrict__ nw, uint32_t* __restrict__ nw_cnt,
                              uint32_t* __restrict__ od, uint32_t* __restrict__ od_cnt)
{
  const int64_t u = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
  const int lane  = threadIdx.x & 31;
  if (u >= n) return;
  uint64_t* row = L + u * Ki;
  int nn = 0, no = 0;
  for (int c0 = 0; c0 < Ki && (nn < kS || no < kS); c0 += 32) {
    const int e     = c0 + lane;
    const bool ok   = e < Ki;
    const uint64_t k = ok ? row[e] : 0;
    const bool is_new = ok && (static_cast<uint32_t>(k) & kNew);
    const bool is_old = ok && !is_new;
    const uint32_t bn = __ballot_sync(0xffffffffu, is_new), bo = __ballot_sync(0xffffffffu, is_old);
    const int rn = nn + __popc(bn & lanemask_lt()), ro = no + __popc(bo & lanemask_lt());
    if (is_new && rn < kS) {
      nw[u * kS + rn] = static_cast<uint32_t>(k) & kIdMask;
      row[e]          = k & ~static_cast<uint64_t>(kNew);
    }
    if (is_old && ro < kS) od[u * kS + ro] = static_cast<uint32_t>(k) & kIdMask;
    nn = min(kS, nn + __popc(bn));
    no = min(kS, no + __popc(bo));
  }
  if (lane == 0) { nw_cnt[u] = nn; od_cnt[u] = no; }
}

// ------------------------------------------------------------------------------------------------------------ grouping
// (target, key) pairs grouped by target: off[n + 1] = exclusive prefix of the counts, out[off[t], off[t + 1]) the keys of t in
// no particular order (every consumer is order-independent).
__global__ void group_count_kernel(const uint32_t* __restrict__ tgt, const unsigned long long* __restrict__ m_dev, int64_t m_cap,
                                   uint32_t* __restrict__ cnt)
{
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t m = m_dev ? static_cast<int64_t>(*m_dev) : m_cap;
  if (i >= m) return;
  const uint32_t t = tgt[i];
  if (t != kInvalid) atomicAdd(cnt + t, 1u);
}
__global__ void group_scatter_kernel(const uint32_t* __restrict__ tgt, const uint64_t* __restrict__ key, const unsigned long long* __restrict__ m_dev,
                                     int64_t m_cap, const uint32_t* __restrict__ off, uint32_t* __restrict__ fill, uint64_t* __restrict__ out)
{
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t m = m_dev ? static_cast<int64_t>(*m_dev) : m_cap;
  if (i >= m) return;
  const uint32_t t = tgt[i];
  if (t != kInvalid) out[off[t] + atomicAdd(fill + t, 1u)] = key[i];
}

struct grouping {
  dbuf<uint32_t> cnt, off;
  dbuf<unsigned char> tmp;
  size_t tmp_bytes = 0;
  void run(cudaStream_t s, const uint32_t* tgt, const uint64_t* key, const unsigned long long* m_dev, int64_t m_cap, int64_t n, uint64_t* out)
  {
    if (cnt.size() < static_cast<size_t>(n + 1)) {
      cnt.alloc(static_cast<size_t>(n + 1), s);
      off.alloc(static_cast<size_t>(n + 1), s);
      size_t need = 0;
      B2_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, need, cnt.data(), off.data(), static_cast<int>(n + 1), s));
      tmp.alloc(std::max<size_t>(need, 1), s);
      tmp_bytes = need;
    }
    B2_CUDA(cudaMemsetAsync(cnt.data(), 0, sizeof(uint32_t) * (n + 1), s));
    count_launch(2);
    group_count_kernel<<<blocks_for(std::max<int64_t>(m_cap, 1), 256), 256, 0, s>>>(tgt, m_dev, m_cap, cnt.data());
    size_t bytes = tmp_bytes;
    B2_CUDA(cub::DeviceScan::ExclusiveSum(tmp.data(), bytes, cnt.data(), off.data(), static_cast<int>(n + 1), s));
    B2_CUDA(cudaMemsetAsync(cnt.data(), 0, sizeof(uint32_t) * (n + 1), s));
    group_scatter_kernel<<<blocks_for(std::max<int64_t>(m_cap, 1), 256), 256, 0, s>>>(tgt, key, m_dev, m_cap, off.data(), cnt.data(), out);
    B2_CUDA(cudaGetLastError());
  }
};

// ------------------------------------------------------------------------------------------------------------- reverse
// For v in list(u): the pair (v, (hash(t, u, v) << 32) | u).
__global__ void reverse_pairs_kernel(const uint32_t* __restrict__ list, const uint32_t* __restrict__ cnt, int64_t n, uint64_t it_hash,
                                     uint32_t* __restrict__ tgt, uint64_t* __restrict__ key)
{
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n * kS) return;
  const int64_t u = i / kS;
  const int s     = static_cast<int>(i % kS);
  if (s >= static_cast<int>(cnt[u])) { tgt[i] = kInvalid; return; }
  const uint32_t v = list[i];
  const uint64_t h = mix64(it_hash ^ ((static_cast<uint64_t>(u) << 32) | v));
  tgt[i] = v;
  key[i] = (h & 0xffffffff00000000ull) | static_cast<uint64_t>(u);
}

// One warp per target v: the S smallest keys of its group, kept sorted across the lanes while the group streams through.
__global__ void reverse_select_kernel(const uint64_t* __restrict__ grouped, const uint32_t* __restrict__ off, int64_t n, uint32_t* __restrict__ out,
                                      uint32_t* __restrict__ out_cnt)
{
  const int64_t v = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
  const int lane  = threadIdx.x & 31;
  if (v >= n) return;
  const uint32_t b = off[v], e = off[v + 1];
  uint64_t best = kNoKey;  // lane i: the i-th smallest so far
  for (uint32_t c = b; c < e; c += 32) {
    uint64_t k = c + lane < e ? grouped[c + lane] : kNoKey;
    k          = warp_sort_key(k);
    // the 32 smallest of two ascending runs: min of one run and the other reversed is bitonic, then sorted
    const uint64_t rev = __shfl_sync(0xffffffffu, k, 31 - lane);
    best               = warp_sort_key(min(best, rev));
  }
  const bool ok = best != kNoKey;
  if (ok) out[v * kS + lane] = static_cast<uint32_t>(best);
  const int c = __popc(__ballot_sync(0xffffffffu, ok));
  if (lane == 0) out_cnt[v] = c;
}

// ---------------------------------------------------------------------------------------------------------------- join
struct join_lists {
  const uint32_t *nw, *nw_cnt, *rn, *rn_cnt, *od, *od_cnt, *ro, *ro_cnt;
};

// One CTA per row u.  Slots: [0, 32) new(u), [32, 64) Rnew(u), [64, 96) old(u), [96, 128) Rold(u); N keeps the first
// occurrence of each id of slots [0, 64), O the ids of [64, 128) not in N, first occurrence.  fp16 and 8-bit rows: the
// 64 x 128 matrix d(N_i, (N ∪ O)_j) comes from a wgmma Gram block (gram_block, tc_finish).  fp32 rows: the candidate rows are
// staged kDimChunk columns at a time and each thread accumulates an 8 x 8 block over the columns in ascending order, so
// every entry has pair_dist's bits.  Then a ∈ N proposes its best
// partner by (d, id) over (N ∪ O) \ {a}, a ∈ O its best partner over N; a proposal is kept only when it beats the target's
// live worst entry (its list can only improve, so the final top-Ki is unchanged).
template <typename T>
__global__ void __launch_bounds__(kJoinThreads) join_kernel(const T* __restrict__ x, int64_t ld, int d, int kind, const float* __restrict__ inv,
                                                            const float* __restrict__ nrm_f, const int* __restrict__ nrm_i, join_lists jl,
                                                            int64_t u0, const uint64_t* __restrict__ L, int Ki, uint32_t* __restrict__ p_tgt,
                                                            uint64_t* __restrict__ p_key, unsigned long long* __restrict__ p_count)
{
  constexpr bool TC        = !std::is_same<T, float>::value;
  constexpr int kTileBytes = TC ? kTcTileBytes : kDimChunk * (kJoinThreads + 4) * static_cast<int>(sizeof(T));
  constexpr int kDBytes    = 64 * (kJoinThreads + 1) * 4;
  __shared__ __align__(1024) unsigned char smem[kTileBytes > kDBytes ? kTileBytes : kDBytes];
  __shared__ uint32_t slot[kJoinThreads], cand[kJoinThreads];
  __shared__ int wcnt[4];
  T (*tile)[kJoinThreads + 4] = reinterpret_cast<T (*)[kJoinThreads + 4]>(smem);
  float (*D)[kJoinThreads + 1] = reinterpret_cast<float (*)[kJoinThreads + 1]>(smem);
  const int64_t u = u0 + blockIdx.x;
  const int t = threadIdx.x, part = t >> 5, lane = t & 31;
  {
    const uint32_t* list = part == 0 ? jl.nw : part == 1 ? jl.rn : part == 2 ? jl.od : jl.ro;
    const uint32_t* cnt  = part == 0 ? jl.nw_cnt : part == 1 ? jl.rn_cnt : part == 2 ? jl.od_cnt : jl.ro_cnt;
    slot[t] = lane < static_cast<int>(cnt[u]) ? list[u * kS + lane] : kInvalid;
  }
  __syncthreads();
  const uint32_t my = slot[t];
  bool keep = my != kInvalid;
  for (int j = 0; keep && j < (t < 64 ? t : 64); ++j) keep = slot[j] != my;
  for (int j = 64; keep && t >= 64 && j < t; ++j) keep = slot[j] != my;
  const uint32_t bal = __ballot_sync(0xffffffffu, keep);
  if (lane == 0) wcnt[part] = __popc(bal);
  __syncthreads();
  const int nN = wcnt[0] + wcnt[1], nO = wcnt[2] + wcnt[3];
  if (keep) cand[(t < 64 ? 0 : 64) + ((part & 1) ? wcnt[part - 1] : 0) + __popc(bal & lanemask_lt())] = my;
  if (nN == 0) return;
  __syncthreads();
  const bool valid_row = t < 64 ? t < nN : t - 64 < nO;
  const uint32_t row_id = valid_row ? cand[t] : 0;
  if constexpr (TC) {
    // rows [0, 64) of the block are N, rows [64, 128) O: the wgmma block is N x (N ∪ O)
    __shared__ uint32_t ids[kJoinThreads];
    ids[t] = valid_row ? row_id : kInvalid;
    __syncthreads();
    using G = typename tc_acc<T>::type;
    float g[64];
    gram_block(smem, x, ld, d, ids, g, kind == kHam);
    // (the tile is dead: D reuses its shared memory)
    const int r0 = 16 * part + (lane >> 2);
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int h = 0; h < 4; ++h) {
        const int gi = r0 + 8 * (h >> 1), gj = 8 * j + 2 * (lane & 3) + (h & 1);
        const bool ok = gi < nN && (gj < 64 ? gj < nN : gj - 64 < nO);
        D[gi][gj] = ok ? tc_finish(gram_at<G>(g, 4 * j + h), kind, nrm_f, nrm_i, inv, cand[gi], cand[gj]) : 0.f;
      }
  } else {
    const int ib = t & 7, jb = t >> 3;
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = 0;
    for (int k0 = 0; k0 < d; k0 += kDimChunk) {
      const int kmax = min(kDimChunk, d - k0);
      for (int r = part; r < kJoinThreads; r += 4) {
        const bool ok = r < 64 ? r < nN : r - 64 < nO;
        if (lane < kmax) tile[lane][r] = ok ? x[static_cast<int64_t>(cand[r]) * ld + k0 + lane] : T(0);
      }
      __syncthreads();
      for (int k = 0; k < kmax; ++k) {
        float a[8], b[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) a[i] = load_acc(tile[k][ib * 8 + i]);
#pragma unroll
        for (int j = 0; j < 8; ++j) b[j] = load_acc(tile[k][jb * 8 + j]);
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) accumulate(acc[i][j], a[i], b[j], kind == kL2);
      }
      __syncthreads();
    }
    // (the tile is dead: D reuses its shared memory)
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int gi = ib * 8 + i;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int gj = jb * 8 + j;
        const bool ok = gi < nN && (gj < 64 ? gj < nN : gj - 64 < nO);
        D[gi][gj] = ok ? finish(acc[i][j], kind, inv, cand[gi], cand[gj]) : 0.f;
      }
    }
  }
  __syncthreads();
  uint64_t best = kNoKey;
  if (t < nN) {
    for (int c = 0; c < nN; ++c)
      if (c != t) best = min(best, make_key(D[t][c], cand[c]));
    for (int c = 0; c < nO; ++c) best = min(best, make_key(D[t][64 + c], cand[64 + c]));
  } else if (t >= 64 && t - 64 < nO) {
    for (int i = 0; i < nN; ++i) best = min(best, make_key(D[i][t], cand[i]));
  }
  bool emit = false;
  if (best != kNoKey) emit = best < (L[static_cast<int64_t>(row_id) * Ki + Ki - 1] & kKeyMask);
  const uint32_t eb = __ballot_sync(0xffffffffu, emit);
  unsigned long long base = 0;
  if (lane == 0 && eb) base = atomicAdd(p_count, static_cast<unsigned long long>(__popc(eb)));
  base = __shfl_sync(0xffffffffu, base, 0);
  if (emit) {
    const unsigned long long at = base + __popc(eb & lanemask_lt());
    p_tgt[at] = row_id;
    p_key[at] = best;
  }
}

// --------------------------------------------------------------------------------------------------------------- merge
// One CTA per target a with proposals: L(a) becomes the top-Ki of L(a) and the proposals, duplicate ids removed (a duplicate
// has the same key, since d is a function of the pair).  Proposals stream through 128 at a time: those at or beyond the live
// worst entry are dropped, the rest sorted, deduplicated against each other and the list, and merged by rank.  An entry
// already in the list keeps its flags; an entering one is new and fresh.
__global__ void __launch_bounds__(128) merge_kernel(uint64_t* __restrict__ L, int Ki, const uint64_t* __restrict__ grouped, const uint32_t* __restrict__ off)
{
  extern __shared__ __align__(16) uint64_t merge_smem[];
  uint64_t* lk   = merge_smem;   // [Ki]
  uint64_t* nk   = lk + Ki;      // [Ki]
  uint64_t* pk   = nk + Ki;      // [128]
  uint64_t* surv = pk + 128;     // [128]
  __shared__ int wc[4];
  const int64_t a = blockIdx.x;
  const uint32_t b = off[a], e = off[a + 1];
  if (b == e) return;
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  uint64_t* row = L + a * Ki;
  for (int i = t; i < Ki; i += 128) lk[i] = row[i];
  __syncthreads();
  for (uint32_t c0 = b; c0 < e; c0 += 128) {
    uint64_t p = c0 + t < e ? grouped[c0 + t] : kNoKey;
    if (p >= (lk[Ki - 1] & kKeyMask)) p = kNoKey;
    pk[t] = p;
    __syncthreads();
    block_sort_keys(pk, 128);
    p = pk[t];
    bool ok = p != kNoKey && (t == 0 || pk[t - 1] != p);
    if (ok) {
      const int at = count_below(lk, Ki, p);
      ok = at == Ki || (lk[at] & kKeyMask) != p;
    }
    const uint32_t bal = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) wc[w] = __popc(bal);
    __syncthreads();
    int base = 0;
    for (int q = 0; q < w; ++q) base += wc[q];
    const int m = wc[0] + wc[1] + wc[2] + wc[3];
    if (ok) surv[base + __popc(bal & lanemask_lt())] = p;
    __syncthreads();
    if (m == 0) continue;
    for (int i = t; i < Ki; i += 128) {
      const int pos = i + count_below(surv, m, lk[i] & kKeyMask);
      if (pos < Ki) nk[pos] = lk[i];
    }
    for (int j = t; j < m; j += 128) {
      const int pos = j + count_below(lk, Ki, surv[j]);
      if (pos < Ki) nk[pos] = surv[j] | kNew | kFresh;
    }
    __syncthreads();
    for (int i = t; i < Ki; i += 128) lk[i] = nk[i];
    __syncthreads();
  }
  for (int i = t; i < Ki; i += 128) row[i] = lk[i];
}

// updates: the entries that entered a list during the iteration; their fresh bit is cleared
__global__ void fresh_count_kernel(uint64_t* __restrict__ L, int64_t count, unsigned long long* __restrict__ updates)
{
  unsigned long long c = 0;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < count; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const uint64_t k = L[i];
    if (static_cast<uint32_t>(k) & kFresh) {
      L[i] = k & ~static_cast<uint64_t>(kFresh);
      ++c;
    }
  }
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(updates, c);
}

// ------------------------------------------------------------------------------------------------------ row preparation
// sum of squares of a row in its join type, ascending (fmaf over fp16 values, exact int over 8-bit ones)
template <typename T>
__global__ void sq_norm_kernel(const T* __restrict__ x, int64_t n, int d, int64_t ld, typename acc_of<T>::type* __restrict__ out)
{
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  typename acc_of<T>::type acc = 0;
  for (int k = 0; k < d; ++k) {
    const auto v = load_acc(x[i * ld + k]);
    accumulate(acc, v, v, false);
  }
  out[i] = acc;
}

// bits set in each 8-bit row (the Hamming join's per-row term)
template <typename T>
__global__ void popc_rows_kernel(const T* __restrict__ x, int64_t n, int d, int64_t ld, int* __restrict__ out)
{
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  int acc = 0;
  for (int k = 0; k < d; ++k) acc += __popc(static_cast<uint8_t>(x[i * ld + k]));
  out[i] = acc;
}

// per-column sums over fixed row blocks in fp64 (partial[blk, d]), then summed in block order: the same mean on every run
constexpr int kMeanRows = 4096;
__global__ void col_sum_kernel(const float* __restrict__ x, int64_t n, int d, int64_t ld, double* __restrict__ partial)
{
  const int64_t r0 = static_cast<int64_t>(blockIdx.x) * kMeanRows, r1 = min(n, r0 + kMeanRows);
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    double s = 0;
    for (int64_t r = r0; r < r1; ++r) s += x[r * ld + c];
    partial[static_cast<int64_t>(blockIdx.x) * d + c] = s;
  }
}
__global__ void col_shift_kernel(const double* __restrict__ partial, int blocks, int64_t n, int d, float* __restrict__ shift)
{
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= d) return;
  double s = 0;
  for (int b = 0; b < blocks; ++b) s += partial[static_cast<int64_t>(b) * d + c];
  shift[c] = static_cast<float>(rint(s / static_cast<double>(n)));
}

// fp16 rows for the join: (x - shift[c]) * scale[row], each optional, computed in fp32 and rounded once
template <typename T>
__global__ void to_half_kernel(const T* __restrict__ x, int64_t n, int d, int64_t ld, const float* __restrict__ shift, const float* __restrict__ scale,
                               __half* __restrict__ out)
{
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n * d) return;
  const int64_t r = i / d;
  const int c     = static_cast<int>(i % d);
  float v = static_cast<float>(load_acc(x[r * ld + c]));
  if (shift) v = __fsub_rn(v, shift[c]);
  if (scale) v = __fmul_rn(v, scale[r]);
  out[i] = __float2half_rn(v);
}

// ------------------------------------------------------------------------------------------------------------ re-score
// the batch's rows widened to the fp32 query block of rescore_topk
template <typename T>
__global__ void widen_rows_kernel(const T* __restrict__ x, int64_t ld, int d, int64_t count, float* __restrict__ out)
{
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= count * d) return;
  out[i] = static_cast<float>(load_acc(x[(i / d) * ld + i % d]));
}

__global__ void list_ids_kernel(const uint64_t* __restrict__ L, int64_t count, uint32_t* __restrict__ ids)
{
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i < count) ids[i] = static_cast<uint32_t>(L[i]) & kIdMask;
}

__global__ void narrow_ids_kernel(const int64_t* __restrict__ in, int64_t count, uint32_t* __restrict__ out)
{
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i < count) out[i] = static_cast<uint32_t>(in[i]);
}

const char* metric_name(cuvsDistanceType m)
{
  switch (m) {
    case L2Expanded: return "L2Expanded";
    case L2SqrtExpanded: return "L2SqrtExpanded";
    case CosineExpanded: return "CosineExpanded";
    case L1: return "L1";
    case L2Unexpanded: return "L2Unexpanded";
    case L2SqrtUnexpanded: return "L2SqrtUnexpanded";
    case InnerProduct: return "InnerProduct";
    case Linf: return "Linf";
    case Canberra: return "Canberra";
    case LpUnexpanded: return "LpUnexpanded";
    case CorrelationExpanded: return "CorrelationExpanded";
    case JaccardExpanded: return "JaccardExpanded";
    case HellingerExpanded: return "HellingerExpanded";
    case Haversine: return "Haversine";
    case BrayCurtis: return "BrayCurtis";
    case JensenShannon: return "JensenShannon";
    case HammingUnexpanded: return "HammingUnexpanded";
    case KLDivergence: return "KLDivergence";
    case RusselRaoExpanded: return "RusselRaoExpanded";
    case DiceExpanded: return "DiceExpanded";
    case BitwiseHamming: return "BitwiseHamming";
    default: return "unknown";
  }
}

// the iterations, over join rows of type T (the rows as given, or their fp16 copy)
template <typename T>
void iterate(resources* r, const T* x, int64_t ld, int d, int kind, const float* inv, int64_t n, int Ki, int max_iterations, float threshold,
             uint64_t* L)
{
  auto s = r->stream;
  constexpr bool TC = !std::is_same<T, float>::value;
  const int KiP = [&] { int p = 1; while (p < Ki) p <<= 1; return p; }();
  // squared norms for the tensor-core L2 form: fp32 over the fp16 values, exact int32 over 8-bit ones; Hamming: popcounts
  dbuf<float> nrm_f;
  dbuf<int> nrm_i;
  if constexpr (sizeof(T) == 1) {
    if (kind == kHam) {
      nrm_i.alloc(static_cast<size_t>(n), s);
      count_launch();
      popc_rows_kernel<T><<<blocks_for(n, 128), 128, 0, s>>>(x, n, d, ld, nrm_i.data());
      B2_CUDA(cudaGetLastError());
    }
  }
  if (TC && kind == kL2) {
    count_launch();
    if constexpr (std::is_same<T, __half>::value) {
      nrm_f.alloc(static_cast<size_t>(n), s);
      sq_norm_kernel<T><<<blocks_for(n, 128), 128, 0, s>>>(x, n, d, ld, nrm_f.data());
    } else if constexpr (TC) {
      nrm_i.alloc(static_cast<size_t>(n), s);
      sq_norm_kernel<T><<<blocks_for(n, 128), 128, 0, s>>>(x, n, d, ld, nrm_i.data());
    }
    B2_CUDA(cudaGetLastError());
  }
  {
    timed_section ts("nn_descent_init", s);
    const size_t smem = sizeof(uint64_t) * KiP + sizeof(uint32_t) * Ki;
    count_launch();
    if constexpr (TC) {
      B2_CUDA(cudaFuncSetAttribute(init_tc_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
      init_tc_kernel<T><<<static_cast<unsigned>(n), 128, smem, s>>>(x, ld, d, kind, nrm_f.data(), nrm_i.data(), inv, n, Ki, KiP, L);
    } else {
      B2_CUDA(cudaFuncSetAttribute(init_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
      init_kernel<T><<<static_cast<unsigned>(n), 128, smem, s>>>(x, ld, d, kind, inv, n, Ki, KiP, L);
    }
    B2_CUDA(cudaGetLastError());
  }
  const size_t ns = static_cast<size_t>(n) * kS;
  dbuf<uint32_t> nw(ns, s), od(ns, s), rn(ns, s), ro(ns, s), nw_cnt(n, s), od_cnt(n, s), rn_cnt(n, s), ro_cnt(n, s);
  dbuf<uint32_t> pair_tgt(ns, s);
  dbuf<uint64_t> pair_key(ns, s), pair_grouped(ns, s);
  // proposals of one chunk of join rows (at most 128 per row); chunks keep them within a fixed budget
  const int64_t chunk = std::min<int64_t>(n, std::max<int64_t>(1, (int64_t(6) << 30) / (kJoinThreads * 20)));
  const size_t pcap   = static_cast<size_t>(chunk) * kJoinThreads;
  dbuf<uint32_t> p_tgt(pcap, s);
  dbuf<uint64_t> p_key(pcap, s), p_grouped(pcap, s);
  dbuf<unsigned long long> counters(2, s);  // [0] proposals of the chunk, [1] updates of the iteration
  grouping grp;
  const size_t merge_smem = sizeof(uint64_t) * (2 * static_cast<size_t>(Ki) + 256);
  B2_CUDA(cudaFuncSetAttribute(merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(merge_smem)));
  const double stop_at = static_cast<double>(threshold) * static_cast<double>(n) * Ki;
  for (int it = 0; it < max_iterations; ++it) {
    {
      timed_section ts("nn_descent_sample", s);
      count_launch();
      sample_kernel<<<blocks_for(n * 32, 256), 256, 0, s>>>(L, n, Ki, nw.data(), nw_cnt.data(), od.data(), od_cnt.data());
      B2_CUDA(cudaGetLastError());
    }
    {
      timed_section ts("nn_descent_reverse", s);
      const uint64_t it_hash = mix64(kRevSeed ^ static_cast<uint64_t>(it));
      for (int pass = 0; pass < 2; ++pass) {
        count_launch(2);
        reverse_pairs_kernel<<<blocks_for(static_cast<int64_t>(ns), 256), 256, 0, s>>>(pass ? od.data() : nw.data(), pass ? od_cnt.data() : nw_cnt.data(),
                                                                                       n, it_hash, pair_tgt.data(), pair_key.data());
        grp.run(s, pair_tgt.data(), pair_key.data(), nullptr, static_cast<int64_t>(ns), n, pair_grouped.data());
        reverse_select_kernel<<<blocks_for(n * 32, 256), 256, 0, s>>>(pair_grouped.data(), grp.off.data(), n, pass ? ro.data() : rn.data(),
                                                                       pass ? ro_cnt.data() : rn_cnt.data());
        B2_CUDA(cudaGetLastError());
      }
    }
    const join_lists jl{nw.data(), nw_cnt.data(), rn.data(), rn_cnt.data(), od.data(), od_cnt.data(), ro.data(), ro_cnt.data()};
    for (int64_t u0 = 0; u0 < n; u0 += chunk) {
      const int64_t nu = std::min(chunk, n - u0);
      {
        timed_section ts("nn_descent_join", s);
        B2_CUDA(cudaMemsetAsync(counters.data(), 0, sizeof(unsigned long long), s));
        count_launch();
        join_kernel<T><<<static_cast<unsigned>(nu), kJoinThreads, 0, s>>>(x, ld, d, kind, inv, nrm_f.data(), nrm_i.data(), jl, u0, L, Ki,
                                                                         p_tgt.data(), p_key.data(), counters.data());
        B2_CUDA(cudaGetLastError());
      }
      {
        timed_section ts("nn_descent_merge", s);
        grp.run(s, p_tgt.data(), p_key.data(), counters.data(), static_cast<int64_t>(pcap), n, p_grouped.data());
        count_launch();
        merge_kernel<<<static_cast<unsigned>(n), 128, merge_smem, s>>>(L, Ki, p_grouped.data(), grp.off.data());
        B2_CUDA(cudaGetLastError());
      }
    }
    unsigned long long updates = 0;
    {
      timed_section ts("nn_descent_merge", s);
      B2_CUDA(cudaMemsetAsync(counters.data() + 1, 0, sizeof(unsigned long long), s));
      count_launch();
      fresh_count_kernel<<<std::min<unsigned>(blocks_for(n * Ki, 256), 4096), 256, 0, s>>>(L, n * Ki, counters.data() + 1);
      B2_CUDA(cudaGetLastError());
      B2_CUDA(cudaMemcpyAsync(&updates, counters.data() + 1, sizeof(updates), cudaMemcpyDeviceToHost, s));
      B2_CUDA(cudaStreamSynchronize(s));
    }
    if (static_cast<double>(updates) <= stop_at) break;
  }
}

// exact re-score of every list with rescore_topk, best `degree` kept
template <typename T>
void rescore(resources* r, const T* x, int64_t ld, int d, cuvsDistanceType metric, int64_t n, int Ki, const uint64_t* L, int degree, uint32_t* graph,
             float* dist)
{
  auto s = r->stream;
  timed_section ts("nn_descent_rescore", s);
  constexpr bool f32 = std::is_same<T, float>::value;
  const bool norms   = metric == L2Expanded || metric == L2SqrtExpanded || metric == CosineExpanded;
  dbuf<float> xn;
  if (norms) {
    xn.alloc(static_cast<size_t>(n), s);
    row_norms(s, x, n, d, ld, xn.data());
  }
  // narrow rows: the batch's own rows are widened into the fp32 query block rescore_topk reads; the batch's temporaries (that
  // block, the candidate ids and the kept ids and distances) stay within about 1 GiB
  const int64_t per_row = 4 * static_cast<int64_t>(d) + 4 * static_cast<int64_t>(Ki) + 12 * static_cast<int64_t>(degree);
  const int64_t batch   = std::min<int64_t>(std::min<int64_t>(n, 1 << 20), f32 ? n : std::max<int64_t>(1, (int64_t(1) << 30) / per_row));
  dbuf<uint32_t> cand(static_cast<size_t>(batch) * Ki, s);
  dbuf<int64_t> out_idx(static_cast<size_t>(batch) * degree, s);
  dbuf<float> out_dist(static_cast<size_t>(batch) * degree, s), qf;
  if (!f32) qf.alloc(static_cast<size_t>(batch) * d, s);
  for (int64_t b0 = 0; b0 < n; b0 += batch) {
    const int64_t nb = std::min(batch, n - b0);
    count_launch();
    list_ids_kernel<<<blocks_for(nb * Ki, 256), 256, 0, s>>>(L + b0 * Ki, nb * Ki, cand.data());
    const float* q = qf.data();
    int64_t ldq    = d;
    if constexpr (f32) {
      q   = x + b0 * ld;
      ldq = ld;
    } else {
      count_launch();
      widen_rows_kernel<T><<<blocks_for(nb * d, 256), 256, 0, s>>>(x + b0 * ld, ld, d, nb, qf.data());
    }
    B2_CUDA(cudaGetLastError());
    // candidate positions are row ids: ties rank by id
    rescore_topk(s, q, nb, ldq, x, ld, d, norms ? xn.data() + b0 : nullptr, norms ? xn.data() : nullptr, metric, cand.data(), Ki, nullptr,
                 degree, out_idx.data(), out_dist.data(), -1);
    count_launch();
    narrow_ids_kernel<<<blocks_for(nb * degree, 256), 256, 0, s>>>(out_idx.data(), nb * degree, graph + b0 * degree);
    B2_CUDA(cudaGetLastError());
    if (dist) B2_CUDA(cudaMemcpyAsync(dist + b0 * degree, out_dist.data(), sizeof(float) * nb * degree, cudaMemcpyDeviceToDevice, s));
  }
  if (dist) postprocess_distances(s, dist, n * degree, metric);
}

// Hamming lists: the join's distances are exact integers and each list is sorted by (distance, id), so the output is
// every list's first `degree` entries as they stand
__global__ void list_head_kernel(const uint64_t* __restrict__ L, int64_t n, int Ki, int degree, uint32_t* __restrict__ graph, float* __restrict__ dist)
{
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n * degree) return;
  const uint64_t k = L[(i / degree) * Ki + i % degree];
  graph[i] = static_cast<uint32_t>(k) & kIdMask;
  if (dist) dist[i] = __uint_as_float(static_cast<uint32_t>(k >> 32) ^ 0x80000000u);  // ord_f of a non-negative distance
}

template <typename T>
void run_typed(resources* r, const T* x, int64_t n, int d, int64_t ld, cuvsDistanceType metric, int kind, bool half_path, int degree, int Ki,
               int max_iterations, float threshold, uint32_t* graph, float* dist)
{
  auto s = r->stream;
  dbuf<uint64_t> L(static_cast<size_t>(n) * Ki, s);
  dbuf<float> inv;
  if (kind == kCos) {
    inv.alloc(static_cast<size_t>(n), s);
    row_norms(s, x, n, d, ld, inv.data());
    rsqrt_rows(s, inv.data(), n, inv.data());
  }
  constexpr bool is_half = std::is_same<T, __half>::value;
  if (!half_path || (is_half && kind != kCos)) {
    iterate<T>(r, x, ld, d, kind, kind == kCos ? inv.data() : nullptr, n, Ki, max_iterations, threshold, L.data());
  } else {
    // fp16 join rows: L2 shifted by the rounded column means (float32 rows only), cosine scaled to unit length
    dbuf<float> shift;
    if (kind == kL2 && std::is_same<T, float>::value) {
      const int blocks = static_cast<int>((n + kMeanRows - 1) / kMeanRows);
      dbuf<double> partial(static_cast<size_t>(blocks) * d, s);
      shift.alloc(static_cast<size_t>(d), s);
      count_launch(2);
      col_sum_kernel<<<blocks, 128, 0, s>>>(reinterpret_cast<const float*>(x), n, d, ld, partial.data());
      col_shift_kernel<<<blocks_for(d, 128), 128, 0, s>>>(partial.data(), blocks, n, d, shift.data());
      B2_CUDA(cudaGetLastError());
    }
    dbuf<__half> h(static_cast<size_t>(n) * d, s);
    count_launch();
    to_half_kernel<T><<<blocks_for(n * d, 256), 256, 0, s>>>(x, n, d, ld, shift.data(), kind == kCos ? inv.data() : nullptr, h.data());
    B2_CUDA(cudaGetLastError());
    iterate<__half>(r, h.data(), d, d, kind, nullptr, n, Ki, max_iterations, threshold, L.data());
  }
  if (kind == kHam) {
    count_launch();
    list_head_kernel<<<blocks_for(n * degree, 256), 256, 0, s>>>(L.data(), n, Ki, degree, graph, dist);
    B2_CUDA(cudaGetLastError());
    return;
  }
  rescore<T>(r, x, ld, d, metric, n, Ki, L.data(), degree, graph, dist);
}

}  // namespace

void nn_descent_graph(resources* r, const void* rows, row_type rt, int64_t n, int dim, int64_t ld, cuvsDistanceType metric, int degree,
                      int intermediate, int max_iterations, float termination_threshold, int dist_comp, uint32_t* graph, float* dist)
{
  int kind = kL2;
  if (metric == InnerProduct) kind = kIP;
  else if (metric == CosineExpanded) kind = kCos;
  else if (metric == BitwiseHamming) kind = kHam;
  else B2_EXPECTS(metric == L2Expanded || metric == L2SqrtExpanded,
                  "nn-descent: metric %s (%d) is not supported; use L2Expanded, L2SqrtExpanded, InnerProduct, CosineExpanded or "
                  "BitwiseHamming (int8 / uint8 rows)",
                  metric_name(metric), static_cast<int>(metric));
  const DLDataType dt = dtype_of(rt);
  B2_EXPECTS(kind != kHam || row_bytes(rt) == 1,
             "nn-descent: BitwiseHamming distance is only supported for int8 and uint8 rows (got dtype code %d, bits %d)", dt.code, dt.bits);
  B2_EXPECTS(n >= 2 && n < (int64_t(1) << 30), "nn-descent: the dataset must have between 2 and 2^30 - 1 rows (got %lld)", (long long)n);
  B2_EXPECTS(dim >= 1, "nn-descent: the dataset has no columns");
  B2_EXPECTS(degree >= 1 && degree <= n - 1, "nn-descent: graph_degree (%d) must be in [1, n - 1 = %lld]", degree, (long long)(n - 1));
  B2_EXPECTS(dist_comp >= NND_DIST_COMP_AUTO && dist_comp <= NND_DIST_COMP_FP16, "nn-descent: unknown dist_comp_dtype %d", dist_comp);
  const int64_t ki_want = (std::max<int64_t>(intermediate, degree) + 31) / 32 * 32;
  const int Ki = static_cast<int>(std::min<int64_t>(ki_want, n - 1));
  B2_EXPECTS(Ki <= kMaxKi, "nn-descent: intermediate_graph_degree %d exceeds %d", static_cast<int>(ki_want), kMaxKi);
  B2_EXPECTS(max_iterations >= 0, "nn-descent: max_iterations must be >= 0");
  const bool f32 = rt == row_type::f32;
  B2_EXPECTS(row_bytes(rt) != 1 || dim <= 32768, "nn-descent: 8-bit rows are limited to 32768 columns (exact int32 sums), got %d", dim);
  B2_EXPECTS(f32 || dist_comp != NND_DIST_COMP_FP32, "nn-descent: dist_comp_dtype FP32 is valid for float32 data only");
  const bool half_path = f32 ? (dist_comp == NND_DIST_COMP_FP16 || (dist_comp == NND_DIST_COMP_AUTO && dim > 16)) : rt == row_type::f16;
  with_row_type(rt, [&](auto t) {
    using T = decltype(t);
    run_typed<T>(r, static_cast<const T*>(rows), n, dim, ld, metric, kind, half_path, degree, Ki, max_iterations, termination_threshold, graph,
                 dist);
  });
}

}  // namespace b200

using namespace b200;

namespace {
struct nnd_index {
  int64_t n  = 0;
  int degree = 0;
  owned<uint32_t> graph;
  owned<float> dist;  // empty when built without distances
};
// copies rows x cols elements of `es` bytes from device `src` into a row-major host or device tensor
void copy_out(resources* r, const void* src, const DLTensor& dst, int64_t rows, int64_t cols, DLDataType dt, const char* what)
{
  B2_EXPECTS(dst.dtype.code == dt.code && dst.dtype.bits == dt.bits && dst.dtype.lanes == 1, "%s has the wrong dtype", what);
  B2_EXPECTS(dst.ndim == 2 && dl_is_c_contiguous(dst), "%s must be a row-major 2-D tensor", what);
  B2_EXPECTS(dst.shape[0] == rows, "Output %s has incorrect number of rows", what);
  B2_EXPECTS(dst.shape[1] == cols, "Output %s has incorrect number of cols", what);
  B2_CUDA(cudaMemcpyAsync(dst.data, src, static_cast<size_t>(rows) * cols * (dt.bits / 8), cudaMemcpyDefault, r->stream));
  B2_CUDA(cudaStreamSynchronize(r->stream));
}
}  // namespace

extern "C" {

cuvsError_t cuvsNNDescentIndexParamsCreate(cuvsNNDescentIndexParams_t* params)
{
  return guarded([=] {
    B2_EXPECTS(params != nullptr, "params is null");
    // the reference's defaults (cpp/include/cuvs/neighbors/nn_descent.hpp index_params)
    *params = new cuvsNNDescentIndexParams{L2Expanded, 2.0f, 64, 128, 20, 0.0001f, true, NND_DIST_COMP_AUTO};
  });
}
cuvsError_t cuvsNNDescentIndexParamsDestroy(cuvsNNDescentIndexParams_t params) { return guarded([=] { delete params; }); }

cuvsError_t cuvsNNDescentIndexCreate(cuvsNNDescentIndex_t* index)
{
  return guarded([=] {
    B2_EXPECTS(index != nullptr, "index is null");
    *index = new cuvsNNDescentIndex{};
  });
}
cuvsError_t cuvsNNDescentIndexDestroy(cuvsNNDescentIndex_t index)
{
  return guarded([=] {
    if (!index) return;
    drop_index<nnd_index>(index);
    delete index;
  });
}

cuvsError_t cuvsNNDescentBuild(cuvsResources_t res, cuvsNNDescentIndexParams_t params, DLManagedTensor* dataset_t, DLManagedTensor* graph_t,
                               cuvsNNDescentIndex_t index)
{
  return guarded([=] {
    auto r = as_res(res);
    B2_EXPECTS(params && dataset_t && index, "null argument");
    const DLTensor& ds = dataset_t->dl_tensor;
    B2_EXPECTS(dl_is_dataset_dtype(ds), "Unsupported dataset DLtensor dtype: %d and bits: %d", ds.dtype.code, ds.dtype.bits);
    B2_EXPECTS(ds.ndim == 2 && dl_is_c_contiguous(ds), "dataset must be a row-major 2-D tensor");
    const int64_t n = ds.shape[0];
    const int dim   = static_cast<int>(ds.shape[1]);
    B2_EXPECTS(params->graph_degree >= 1 && params->graph_degree < static_cast<size_t>(std::max<int64_t>(n, 1)),
               "nn-descent: graph_degree (%zu) must be in [1, n - 1] for a dataset of %lld rows", params->graph_degree, (long long)n);
    auto s = r->stream;
    dbuf<unsigned char> staged;
    const void* rows = ds.data;
    if (!(dl_is_device(ds) && ds.device.device_type != kDLCUDAHost)) {
      const size_t bytes = static_cast<size_t>(n) * dim * (ds.dtype.bits / 8);
      staged.alloc(bytes, s);
      B2_CUDA(cudaMemcpyAsync(staged.data(), ds.data, bytes, cudaMemcpyDefault, s));
      rows = staged.data();
    }
    auto idx    = std::make_unique<nnd_index>();
    idx->n      = n;
    idx->degree = static_cast<int>(params->graph_degree);
    idx->graph.alloc(static_cast<size_t>(n) * idx->degree);
    if (params->return_distances) idx->dist.alloc(static_cast<size_t>(n) * idx->degree);
    nn_descent_graph(r, rows, row_type_of(ds.dtype), n, dim, dim, params->metric, idx->degree,
                     static_cast<int>(std::min<size_t>(params->intermediate_graph_degree, 1u << 30)),
                     static_cast<int>(std::min<size_t>(params->max_iterations, 1u << 30)), params->termination_threshold,
                     static_cast<int>(params->dist_comp_dtype), idx->graph.data(), idx->dist.data());
    B2_CUDA(cudaStreamSynchronize(s));
    if (graph_t) copy_out(r, idx->graph.data(), graph_t->dl_tensor, n, idx->degree, DLDataType{kDLUInt, 32, 1}, "graph");
    set_index(index, idx.release(), ds.dtype);
  });
}

cuvsError_t cuvsNNDescentIndexGetGraph(cuvsResources_t res, cuvsNNDescentIndex_t index, DLManagedTensor* graph)
{
  return guarded([=] {
    auto r   = as_res(res);
    auto& ix = index_of<nnd_index>(index);
    B2_EXPECTS(graph != nullptr, "graph is null");
    copy_out(r, ix.graph.data(), graph->dl_tensor, ix.n, ix.degree, DLDataType{kDLUInt, 32, 1}, "graph");
  });
}

cuvsError_t cuvsNNDescentIndexGetDistances(cuvsResources_t res, cuvsNNDescentIndex_t index, DLManagedTensor* distances)
{
  return guarded([=] {
    auto r   = as_res(res);
    auto& ix = index_of<nnd_index>(index);
    B2_EXPECTS(distances != nullptr, "distances is null");
    B2_EXPECTS(ix.dist.data() != nullptr, "nn-descent index doesn't contain distances - set return_distances when building");
    copy_out(r, ix.dist.data(), distances->dl_tensor, ix.n, ix.degree, DLDataType{kDLFloat, 32, 1}, "distances");
  });
}

}  // extern "C"
