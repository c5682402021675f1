// IVF-PQ fine scan for sm_90a: PQ codes streamed from HBM, decoded on the SM, contracted on wgmma, top-k' filtered
// against per-query thresholds.
//
// Replaces   cpp/src/neighbors/ivf_pq/detail/jit_lto_kernels/compute_similarity_impl.cuh:77-173
//            (+ create_lut_impl.cuh:16-79, compute_score_impl.cuh:53-79, compute_distances_impl.cuh:58-100)
// Reference formulation: one CTA per (query, probe); LUT[pq_dim][256] in shared memory; every (query, row, subspace)
// costs one shared-memory gather; the list's codes are re-read from L2/HBM by every probing query.
// Here: work item = (list, <= NQ probing queries).  Per 128-row tile of the list
//
//   warp 0      producer   one cp.async.bulk of the tile's block of the code stream (128 * pq_dim code bytes in "lane-
//                          transposed" order + 128 half-norms = 8.7 KB at pq_dim 64) into a 2..8-deep mbarrier ring;
//                          per item one TMA box with the NQ residual rows (bf16, SWIZZLE_128B)
//   warps 4-11  decode     lane l owns subspaces l and l+32: its 16 code bytes per 16 rows arrive with one 128-bit
//                          shared load; codebook words sit at [half][code][lane] (bank == lane), so a row's 64 entries are
//                          fetched with two conflict-free LDS.32 per lane and written with two STS.32 into the 128-byte-
//                          swizzled K-major operand tile (bf16 row = 256 B).
//   warps 12-19 MMA +      two warpgroups.  NQ = 64 / 128: the queries are the MMA's M side.  NQ = 64, one pass: the
//               epilogue   warpgroups take whole tiles in turn (ping-pong), D[64 queries x 128 rows] (+)= R . Y^T; NQ = 64,
//                          two passes: D[64 queries x 64 rows] (+)= R . Y_half^T per 64-row half of the tile; NQ = 128:
//                          D[64 queries x 128 rows] (+)= R_half . Y^T per 64-query half of the item (wgmma, 8 K-steps + 1 that
//                          adds -|y|^2/2: ones x three bf16 pieces); a thread's fragment is 2 query rows x 16 | 32 list rows,
//                          so each query row is tested with one max against one threshold and its hits reserve their buffer
//                          slots with one atomic.  NQ = 32 (m64 would be half empty): the rows are the M side, D[64 rows x
//                          32 queries] per half, and each element is tested against its own query's threshold.  Hits go
//                          into per-query candidate buffers; a buffer that overflows is compacted to its KC best by one
//                          warp (rank by counting) and the threshold tightened; one named barrier per tile (ping-pong: per
//                          tile of the warpgroup, over its own buffers).
//
// With few probing queries per list (50M rows / 8192 lists / 10k-query batches at 48 probes: ~59) the accumulator is 128 x 32..64
// instead of the 128 x 128 of the query-major kernel (scan_tc.cu), and HBM traffic per row is pq_dim + 4 bytes instead of a
// 2 * rot_dim + 32 byte decoded row.
#include "common.hpp"
#include "ptx_sm90.cuh"
#include "scan_pq.cuh"
#include "timing.hpp"

#include <cuda.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <mutex>

namespace b200 {
namespace {

constexpr int kDecWarps   = 8;
constexpr int kEpiWarps   = 8;                                 // two MMA + epilogue warpgroups
constexpr int kEpiThreads = 32 * kEpiWarps;
constexpr int kDecWarp0   = 4;                                 // warp 0 produces, warps 1-3 only complete its warpgroup
constexpr int kEpiWarp0   = kDecWarp0 + kDecWarps;             // 12: warpgroup aligned, as wgmma requires
constexpr int kThreads    = 32 * (kEpiWarp0 + kEpiWarps);      // 640
constexpr int kDecStages  = 2;
constexpr int kSched      = 4;   // work-item ring
constexpr int kMaxCStages = 8;
constexpr int kDecTile    = 128 * 128;  // one k-block of the decoded tile: 128 rows x 64 bf16, SWIZZLE_128B
constexpr int kExtTile    = 128 * 32;   // half-norm K extension: 128 rows x 16 bf16
constexpr int kSmemLimit  = 227 * 1024;

struct pq_args {
  const uint8_t* stream;
  const uint32_t* cb_words;
  const tc_item* items;
  const int* n_items_dev;
  int* sched;
  float* out_score;
  uint32_t* out_pos;
  int64_t out_row_stride;
  int* b_keys;
  const uint32_t* b_idx;
  const float* b_add;
  float b_scale;
  int kth;
  int n_items_host;
  int KC;
  int cap;      // candidate buffer entries per query (KC < cap <= 128)
  int cstages;  // code ring depth
  int blk;      // bytes of one tile block of the stream
};

__device__ __forceinline__ bool bar_red_or(uint32_t id, uint32_t nthreads, bool pred)
{
  uint32_t r;
  asm volatile(
    "{\n\t"
    ".reg .pred pi, po;\n\t"
    "setp.ne.u32 pi, %1, 0;\n\t"
    "bar.red.or.pred po, %2, %3, pi;\n\t"
    "selp.u32 %0, 1, 0, po;\n\t"
    "}\n"
    : "=r"(r)
    : "r"(static_cast<uint32_t>(pred)), "r"(id), "r"(nthreads)
    : "memory");
  return r != 0;
}

// monotone float -> uint32 (bigger float = bigger key); never 0 for a real float
__device__ __forceinline__ uint32_t okey(uint32_t fbits) { return (fbits & 0x80000000u) ? ~fbits : (fbits | 0x80000000u); }
__device__ __forceinline__ uint32_t okey_inv(uint32_t k) { return (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k; }

// Rows-on-M fragment (NQ = 32; see ptx::wgmma_bf16: rows r0 and r0 + 8 of the tile, query columns 8j + 2 * (lane % 4) + {0, 1})
// against the query columns' running thresholds: no two of a thread's elements share a query, so every element has its own
// threshold and every hit its own slot-reserving atomic.  Only the elements flagged in `only` are looked at; returns the
// elements whose candidate could not be stored (buffer full).
template <int NQ>
__device__ __forceinline__ uint64_t pq_filter_frag(const float (&d)[NQ / 2], uint64_t only, int lane, uint32_t pos0, uint32_t pos1,
                                                   const float* __restrict__ thr, int* cnt, unsigned long long* cand, int cap)
{
  uint64_t left = 0;
  const int cq  = 2 * (lane & 3);
  // All of the fragment's thresholds are loaded before any is tested.  Loaded one column pair at a time, each load waits
  // behind the previous pair's candidate atomics (the compiler does not move it above them), and its latency is paid once
  // per pair.  No thread changes a threshold while a tile is filtered: compaction runs between the per-tile barriers.
  float2 ths[NQ / 8];
#pragma unroll
  for (int j = 0; j < NQ / 8; ++j) ths[j] = *reinterpret_cast<const float2*>(thr + 8 * j + cq);
#pragma unroll
  for (int j = 0; j < NQ / 8; ++j) {
    const int c     = 8 * j + cq;
    const float2 th = ths[j];
    // margin over the column's threshold: a candidate iff > 0 (exact: the difference of two floats keeps its sign)
    const float m = fmaxf(fmaxf(d[4 * j] - th.x, d[4 * j + 1] - th.y), fmaxf(d[4 * j + 2] - th.x, d[4 * j + 3] - th.y));
    if (m > 0.f) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = 4 * j + e, col = c + (e & 1);
        if (((only >> i) & 1u) && d[i] - ((e & 1) ? th.y : th.x) > 0.f) {
          const uint32_t pos = (e & 2) ? pos1 : pos0;
          const int at       = atomicAdd(&cnt[col], 1);
          if (at < cap) cand[col * cap + at] = (static_cast<unsigned long long>(okey(__float_as_uint(d[i]))) << 32) | (~pos);
          else left |= 1ull << i;
        }
      }
    }
  }
  return left;
}

// Queries-on-M fragment (MMA N = 64 / 128 list rows; see ptx::wgmma_bf16: query rows q0 and q0 + 8, list rows
// 8j + 2 * (lane % 4) + {0, 1} of the warpgroup's N side) against the two query rows' thresholds th[0], th[1].  Element
// k < N / 4 of query row q0 + 8h is d[4 * (k / 2) + 2h + k % 2], list row pos0 + 8 * (k / 2) + k % 2; bit 32h + k of `only` and
// of the result stands for it.  A query row is tested with one max over its elements against one threshold (a candidate iff
// > threshold); a row with hits reserves all its buffer slots with one atomic and then stores one hit per pass (constant
// register indices only: the fragment stays in registers).  Returns the elements whose candidate could not be stored (buffer
// full).
template <int N>
__device__ __forceinline__ uint64_t pq_filter_rows(const float (&d)[N / 2], uint64_t only, int q0, uint32_t pos0,
                                                   const float (&th)[2], int* cnt, unsigned long long* cand, int cap)
{
  constexpr int NE = N / 4;
  uint64_t left    = 0;
  // four interleaved max chains per query row: short dependence chains, and few registers beside the fragment
  float mx[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] = d[4 * (k >> 1) + 2 * h + (k & 1)];
#pragma unroll
    for (int k = 4; k < NE; ++k) v[k & 3] = fmaxf(v[k & 3], d[4 * (k >> 1) + 2 * h + (k & 1)]);
    mx[h] = fmaxf(fmaxf(v[0], v[1]), fmaxf(v[2], v[3]));
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (mx[h] > th[h]) {
      uint32_t m = 0;
#pragma unroll
      for (int k = 0; k < NE; ++k) m |= (d[4 * (k >> 1) + 2 * h + (k & 1)] > th[h] ? 1u : 0u) << k;
      m &= static_cast<uint32_t>(only >> (32 * h));
      const int q = q0 + 8 * h;
      int at      = m != 0u ? atomicAdd(&cnt[q], __popc(m)) : 0;
      // one pass per hit: the hit's value is picked from the registers by a select tree on the bits of its index, so the
      // warp runs as many passes as its lane with the most hits in this row, not one per element
      while (m != 0u) {
        const int k = __ffs(m) - 1;
        m &= m - 1u;
        float v[NE / 2];
#pragma unroll
        for (int j = 0; j < NE / 2; ++j) v[j] = (k & 1) ? d[4 * j + 2 * h + 1] : d[4 * j + 2 * h];
#pragma unroll
        for (int lv = 1; (NE >> lv) > 1; ++lv)
#pragma unroll
          for (int j = 0; j < NE / 4; ++j)  // (fixed inner trip count: both loops unroll, v stays in registers)
            if (j < (NE >> (lv + 1))) v[j] = ((k >> lv) & 1) ? v[2 * j + 1] : v[2 * j];
        const uint32_t pos = pos0 + 8 * (k >> 1) + (k & 1);
        if (at < cap) cand[q * cap + at] = (static_cast<unsigned long long>(okey(__float_as_uint(v[0]))) << 32) | (~pos);
        else left |= 1ull << (32 * h + k);
        ++at;
      }
    }
  }
  return left;
}

// Selection inside one column's buffer by one warp, rank by counting: lane l holds entries l, l + 32, l + 64, l + 96 (64-bit keys
// order(t) << 32 | ~pos, unique, 0 = none; n <= 128); every entry is broadcast from shared memory and each lane counts how
// many beat its own.  rank 0 = best.  No dependent chain: n iterations of one LDS.64 + four compare-adds.  The entries are
// buf[0 .. n) followed by buf2[0 .. n2) (the two warpgroups' buffers of one column at NQ = 64 / one pass; n2 = 0 otherwise).
__device__ __forceinline__ void pq_rank_select(const unsigned long long* buf, int n, const unsigned long long* buf2, int n2, int lane,
                                               unsigned long long (&k)[4], int (&r)[4])
{
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int i = lane + 32 * e;
    k[e]        = i < n ? buf[i] : (i < n + n2 ? buf2[i - n] : 0ull);
    r[e]        = 0;
  }
  if (n + n2 <= 64) {  // (warp-uniform) the common case: buffers of <= 64 entries
#pragma unroll 4
    for (int i = 0; i < n; ++i) {
      const unsigned long long ki = buf[i];
      r[0] += ki > k[0] ? 1 : 0;
      r[1] += ki > k[1] ? 1 : 0;
    }
    for (int i = 0; i < n2; ++i) {
      const unsigned long long ki = buf2[i];
      r[0] += ki > k[0] ? 1 : 0;
      r[1] += ki > k[1] ? 1 : 0;
    }
  } else {
#pragma unroll 2
    for (int i = 0; i < n; ++i) {
      const unsigned long long ki = buf[i];
#pragma unroll
      for (int e = 0; e < 4; ++e) r[e] += ki > k[e] ? 1 : 0;
    }
    for (int i = 0; i < n2; ++i) {
      const unsigned long long ki = buf2[i];
#pragma unroll
      for (int e = 0; e < 4; ++e) r[e] += ki > k[e] ? 1 : 0;
    }
  }
}

// Ping-pong consumers (NQ = 64, one pass): each warpgroup owns whole tiles, alternately, and keeps its own thresholds,
// counters and candidate buffers.  With two residual planes (PASSES = 2) two buffer sets leave fewer than two code stages in
// shared memory at pq_dim 64 and KC = 32, so the two-pass consumers keep both warpgroups on every tile (one 64-row half each).
constexpr bool pq_pingpong(int NQ, int PASSES) { return NQ == 64 && PASSES == 1; }

template <int NQ, int NKB, int PASSES>
struct layout {
  static constexpr int n_sets     = pq_pingpong(NQ, PASSES) ? 2 : 1;  // per-warpgroup threshold / counter / buffer sets
  static constexpr int q_tile     = NQ * 128;                       // one k-block of the residual rows
  static constexpr int q_bytes    = PASSES * NKB * q_tile;
  static constexpr int dec_stage  = NKB * kDecTile + kExtTile;
  static constexpr int ones_bytes = NQ * 32;
  static constexpr int cb_bytes   = NKB * 32768;
  static constexpr int off_q      = 0;
  static constexpr int off_dec    = off_q + q_bytes;
  static constexpr int off_ones   = off_dec + kDecStages * dec_stage;
  static constexpr int off_cb     = off_ones + ones_bytes;
  static constexpr int off_thr    = off_cb + cb_bytes;
  static constexpr int off_cnt    = off_thr + n_sets * NQ * 4;
  static constexpr int off_bars   = off_cnt + n_sets * NQ * 4;
  static constexpr int n_bars     = 2 * kMaxCStages + 2 * kDecStages + 2 + 2 * kSched;
  static constexpr int off_item   = off_bars + n_bars * 8;
  static constexpr int off_cand   = (off_item + kSched * 4 + 15) / 16 * 16;   // [n_sets][NQ][cap] uint2, then the code ring
  static_assert(q_tile % 1024 == 0 && dec_stage % 1024 == 0, "operand tiles need 1024-byte alignment");
};

// One tile's MMA into the N-wide fragment d, from decode stage ds (descriptor bases d_lo / x_lo, stages `stage` apart): queries
// on M (QM) D (+)= R . Y^T, else D (+)= Y . R^T.  8 K-steps over the decoded rows and the residual rows (q_lo, k-blocks q_kb
// apart; with two passes the lo plane follows the NKB hi k-blocks), then the step that adds -|y|^2/2: the ext rows hold the
// three bf16 pieces of -hn/2 in both chunks, the ones rows three 1s in both chunks.  Waits for the result.
template <int N, bool QM, int NKB, int PASSES>
__device__ __forceinline__ void pq_tile_mma(float (&d)[N / 2], uint32_t ds, uint32_t stage, uint32_t d_lo, uint32_t x_lo, uint32_t q_lo,
                                            uint32_t q_kb, uint32_t ones_lo)
{
  ptx::wgmma_fence();
  const uint32_t a0 = d_lo + ds * stage;
#pragma unroll
  for (int kb = 0; kb < NKB; ++kb) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint64_t y  = ptx::desc(a0 + kb * (kDecTile >> 4) + k * 2, ptx::kDescHiSw128);
      const uint32_t qd = q_lo + kb * q_kb + k * 2;
      const uint64_t r  = ptx::desc(qd, ptx::kDescHiSw128);
      if (QM) ptx::wgmma_bf16<N>(d, r, y, (kb | k) != 0 ? 1u : 0u);
      else ptx::wgmma_bf16<N>(d, y, r, (kb | k) != 0 ? 1u : 0u);
      if (PASSES == 2) {
        const uint64_t rl = ptx::desc(qd + NKB * q_kb, ptx::kDescHiSw128);
        if (QM) ptx::wgmma_bf16<N>(d, rl, y, 1u);
        else ptx::wgmma_bf16<N>(d, y, rl, 1u);
      }
    }
  }
  const uint64_t xd = ptx::desc(x_lo + ds * stage, ptx::kDescHiSw32), od = ptx::desc(ones_lo, ptx::kDescHiSw32);
  if (QM) ptx::wgmma_bf16<N>(d, od, xd, 1u);
  else ptx::wgmma_bf16<N>(d, xd, od, 1u);
  ptx::wgmma_commit();
  ptx::wgmma_wait<0>();
}

// STORE (KC = 0, k > 64): no threshold filter, candidate buffers, compaction or bound.  The consumers write the score of every
// (query column, list row) of the item to out_score[out_off + col * n_tiles * 128 + row]: one dense segment per pair, its
// list's padded rows in list order (padding rows +inf).
template <int NQ, int NKB, int PASSES, bool STORE = false>
__global__ void __launch_bounds__(kThreads, 1)
pq_stream_scan_kernel(const __grid_constant__ CUtensorMap tmQ_hi, const __grid_constant__ CUtensorMap tmQ_lo, const pq_args P)
{
  using L = layout<NQ, NKB, PASSES>;
  constexpr bool kPP = pq_pingpong(NQ, PASSES) && !STORE;
  static_assert(!kPP || kDecStages == 2, "ping-pong: warpgroup w owns decode stage w and flips its phase once per owned tile");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  if (threadIdx.x == 0 && (ptx::smem_u32(smem_raw) & 1023u) != 0) __trap();
  uint8_t* sQ     = smem_raw + L::off_q;
  uint8_t* sDec   = smem_raw + L::off_dec;
  uint8_t* sOnes  = smem_raw + L::off_ones;
  uint32_t* sCb   = reinterpret_cast<uint32_t*>(smem_raw + L::off_cb);
  float* sThr     = reinterpret_cast<float*>(smem_raw + L::off_thr);
  int* sCnt       = reinterpret_cast<int*>(smem_raw + L::off_cnt);
  uint64_t* bars  = reinterpret_cast<uint64_t*>(smem_raw + L::off_bars);
  uint64_t* c_full  = bars;
  uint64_t* c_empty = c_full + kMaxCStages;
  uint64_t* d_full  = c_empty + kMaxCStages;
  uint64_t* d_empty = d_full + kDecStages;
  uint64_t* q_full  = d_empty + kDecStages;
  uint64_t* q_empty = q_full + 1;
  uint64_t* s_full  = q_empty + 1;
  uint64_t* s_empty = s_full + kSched;
  int* s_item       = reinterpret_cast<int*>(smem_raw + L::off_item);
  unsigned long long* sCand = reinterpret_cast<unsigned long long*>(smem_raw + L::off_cand);  // okey(t) << 32 | ~pos
  uint8_t* sCode  = smem_raw + L::off_cand + L::n_sets * NQ * P.cap * 8;

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const int n_items = P.n_items_dev ? *P.n_items_dev : P.n_items_host;
  const uint32_t ncs = static_cast<uint32_t>(P.cstages);

  if (warp == 0 && lane == 0) {
    ptx::prefetch_tmap(&tmQ_hi);
    if (PASSES == 2) ptx::prefetch_tmap(&tmQ_lo);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < kMaxCStages; ++s) {
      ptx::mbar_init(&c_full[s], 1);
      ptx::mbar_init(&c_empty[s], kDecWarps);
    }
    for (int s = 0; s < kDecStages; ++s) {
      ptx::mbar_init(&d_full[s], kDecWarps);
      ptx::mbar_init(&d_empty[s], kPP ? kEpiWarps / 2 : kEpiWarps);  // ping-pong: stage s is warpgroup s's
    }
    ptx::mbar_init(q_full, 1);
    ptx::mbar_init(q_empty, kEpiWarps);
    for (int s = 0; s < kSched; ++s) {
      ptx::mbar_init(&s_full[s], 1);
      ptx::mbar_init(&s_empty[s], kDecWarps + kEpiWarps);  // every consumer warp hands the slot back
    }
    ptx::fence_barrier_init();
  }
  // codebook words -> shared memory ([half][code][lane]); the constant "ones" operand of the half-norm step: every row
  // {1, 1, 1, 0, 0, 0, 0, 0} in BOTH 16-byte chunks (identical chunks: invariant under the 32-byte swizzle)
  for (int i = threadIdx.x; i < L::cb_bytes / 16; i += kThreads)
    reinterpret_cast<uint4*>(sCb)[i] = reinterpret_cast<const uint4*>(P.cb_words)[i];
  for (int i = threadIdx.x; i < L::ones_bytes / 16; i += kThreads)
    reinterpret_cast<uint4*>(sOnes)[i] = make_uint4(0x3f803f80u, 0x00003f80u, 0u, 0u);
  ptx::fence_proxy_async();
  __syncthreads();

  if (warp < kDecWarp0) {
    ptx::setmaxnreg_dec<40>();
    if (warp == 0) {
    // ------------------------------------------------------------------ producer (whole warp loops, one elected lane issues)
    uint32_t cs = 0, cph = 0, qph = 0, ss = 0, sp = 0;
    for (;;) {
      ptx::mbar_wait(&s_empty[ss], sp ^ 1);
      int it = 0;
      if (lane == 0) {
        it = atomicAdd(P.sched, 1);
        if (it >= n_items) it = -1;
        s_item[ss] = it;
        ptx::mbar_arrive(&s_full[ss]);
      }
      it = __shfl_sync(0xffffffffu, it, 0);
      if (++ss == kSched) { ss = 0; sp ^= 1; }
      if (it < 0) break;
      tc_item item = P.items[it];
      item.a_row0  = __shfl_sync(0xffffffffu, item.a_row0, 0);
      item.b_row0  = __shfl_sync(0xffffffffu, item.b_row0, 0);
      item.n_tiles = __shfl_sync(0xffffffffu, item.n_tiles, 0);
      ptx::mbar_wait(q_empty, qph ^ 1);
      if (ptx::elect_one()) {
        ptx::mbar_arrive_expect_tx(q_full, L::q_bytes);
#pragma unroll
        for (int kb = 0; kb < NKB; ++kb) {
          ptx::tma_load_2d(sQ + kb * L::q_tile, &tmQ_hi, q_full, kb * 64, static_cast<int32_t>(item.a_row0));
          if (PASSES == 2) ptx::tma_load_2d(sQ + (NKB + kb) * L::q_tile, &tmQ_lo, q_full, kb * 64, static_cast<int32_t>(item.a_row0));
        }
      }
      qph ^= 1;
      const uint8_t* src = P.stream + static_cast<int64_t>(item.b_row0 >> 7) * P.blk;
      for (uint32_t t = 0; t < item.n_tiles; ++t) {
        ptx::mbar_wait(&c_empty[cs], cph ^ 1);
        if (ptx::elect_one()) {
          ptx::mbar_arrive_expect_tx(&c_full[cs], static_cast<uint32_t>(P.blk));
          ptx::bulk_load_1d(sCode + cs * P.blk, src + static_cast<int64_t>(t) * P.blk, static_cast<uint32_t>(P.blk), &c_full[cs]);
        }
        if (++cs == ncs) { cs = 0; cph ^= 1; }
      }
    }
    }
  } else if (warp < kEpiWarp0) {
    ptx::setmaxnreg_dec<80>();
    // ------------------------------------------------------------------ decode warps: 16 rows of every tile each
    const int dw = warp - kDecWarp0;
    uint32_t offx[8];  // byte offset of this lane's word inside row x of an 8-row swizzle atom
#pragma unroll
    for (int x = 0; x < 8; ++x) offx[x] = x * 128 + ((((lane >> 2) ^ x) & 7) << 4) + ((lane & 3) << 2);
    const uint32_t cb_lane32 = ptx::smem_u32(sCb) + static_cast<uint32_t>(lane) * 4u;  // this lane's word of codebook row 0
    uint32_t cs = 0, cph = 0, ds = 0, dph = 0, ss = 0, sp = 0;
    for (;;) {
      ptx::mbar_wait(&s_full[ss], sp);
      const int it = __shfl_sync(0xffffffffu, s_item[ss], 0);  // (consumes the load before the slot is handed back)
      if (lane == 0) ptx::mbar_arrive(&s_empty[ss]);
      if (++ss == kSched) { ss = 0; sp ^= 1; }
      if (it < 0) break;
      const uint32_t n_tiles = P.items[it].n_tiles;
      for (uint32_t t = 0; t < n_tiles; ++t) {
        ptx::mbar_wait(&c_full[cs], cph);
        const uint8_t* cst = sCode + cs * P.blk;
        uint4 cw[NKB];
#pragma unroll
        for (int h = 0; h < NKB; ++h) cw[h] = *reinterpret_cast<const uint4*>(cst + dw * (NKB * 512) + h * 512 + lane * 16);
        const float hn = reinterpret_cast<const float*>(cst + NKB * 4096)[16 * dw + (lane >> 1)];
        // The ring slot is handed back only AFTER the decode below has consumed these registers.  An mbarrier arrive issued
        // right behind the loads does not wait for them: the arrive is not ordered behind outstanding LDS (the hardware only
        // scoreboards register USE), and under the tensor core's operand traffic a load can sit in the queue longer than the
        // producer needs to refill the slot from L2 — seen as one warp's 16 rows decoded from the codes of the tile that
        // occupies the slot next, with the half-norms (the tail of the block, written last) still the old ones.
        // compute-sanitizer racecheck flags exactly this pair.
        const uint32_t cs_read = cs;
        if (++cs == ncs) { cs = 0; cph ^= 1; }

        ptx::mbar_wait(&d_empty[ds], dph ^ 1);
        uint8_t* dst = sDec + ds * L::dec_stage + (2 * dw) * 1024;
#pragma unroll
        for (int h = 0; h < NKB; ++h) {
          const uint32_t w4[4] = {cw[h].x, cw[h].y, cw[h].z, cw[h].w};
          uint32_t val[16];
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            // byte extract (PRMT) + scaled add (LEA) on a 32-bit shared address: 2 integer instructions per entry instead of
            // the shift / mask-or / add-base triple the generic-pointer form compiles to (A/B at 100M: 7.88 -> 7.60 ms per batch)
            const uint32_t c = __byte_perm(w4[i >> 2], 0u, 0x4440u | static_cast<uint32_t>(i & 3));
            asm("ld.shared.u32 %0, [%1];" : "=r"(val[i]) : "r"(cb_lane32 + static_cast<uint32_t>(h) * 32768u + (c << 7)));
          }
#pragma unroll
          for (int i = 0; i < 16; ++i)
            *reinterpret_cast<uint32_t*>(dst + h * kDecTile + (i >> 3) * 1024 + offx[i & 7]) = val[i];
        }
        {
          // -hn/2 as three bf16 pieces (exact), identical in both 16-byte chunks of the row; +inf (padding) -> -inf.
          // Lane l writes chunk l % 2 of row l / 2: the warp's 32 x 16 bytes are one contiguous 512-byte span, so every
          // quarter-warp of the 128-bit store covers 128 consecutive bytes = all 32 banks once (row-major lanes, l % 16 = row,
          // put lanes 0..7 at a 32-byte stride: a 2-way conflict on every store, 4 excess wavefronts per warp and tile in ncu)
          const float hh = -0.5f * hn;
          __nv_bfloat16 p0 = __float2bfloat16_rn(hh), p1 = __float2bfloat16_rn(0.f), p2 = p1;
          if (!isinf(hh)) {
            const float r1 = hh - __bfloat162float(p0);
            p1             = __float2bfloat16_rn(r1);
            p2             = __float2bfloat16_rn(r1 - __bfloat162float(p1));
          }
          const uint32_t w0 = static_cast<uint32_t>(__bfloat16_as_ushort(p0)) | (static_cast<uint32_t>(__bfloat16_as_ushort(p1)) << 16);
          const uint32_t w1 = static_cast<uint32_t>(__bfloat16_as_ushort(p2));
          *reinterpret_cast<uint4*>(sDec + ds * L::dec_stage + NKB * kDecTile + (16 * dw) * 32 + lane * 16) =
            make_uint4(w0, w1, 0u, 0u);
        }
        // every loaded register (codes of both halves, half-norm) has fed an issued instruction by now: release the slot
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(&c_empty[cs_read]);
        ptx::fence_proxy_async();  // generic-proxy writes -> visible to the tensor core's async-proxy reads
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(&d_full[ds]);
        if (++ds == kDecStages) { ds = 0; dph ^= 1; }
      }
    }
  } else {
    ptx::setmaxnreg_inc<136>();  // 40 + 2 x 80 + 2 x 136 <= 5 x 96: only registers the other warpgroups gave back
    // ------------------------------------------------------------------ MMA + epilogue: two warpgroups
    // NQ = 64, one pass (ping-pong, kPP): warpgroup w owns every tile g (counted across items, as the decode ring counts) with
    // g % 2 == w, i.e. decode stage w, and computes D[64 queries x 128 rows] (+)= R . Y^T over the whole tile, so one
    // warpgroup's MMAs run while the other filters.  NQ = 64, two passes: one per 64-row half of the tile, D[64 queries x 64
    // rows] (+)= R . Y_half^T; NQ = 128: one per 64-query half of the item, D[64 queries x 128 rows] (+)= R_half . Y^T; NQ = 32:
    // one per 64-row half, D[64 rows x 32 queries] (+)= Y_half . R^T.  wgmma: 8 K-steps + 1 that adds -|y|^2/2.  Then the
    // fragment is tested against the running thresholds (shared memory); the hits go into per-query candidate buffers; a
    // buffer that overflows is compacted to its KC best by one warp (rank by counting) and the threshold tightened, and the
    // elements that did not fit are re-tested from the registers.
    constexpr bool kQM    = NQ >= 64;                              // queries on the MMA's M side
    constexpr bool kWhole = NQ == 128 || kPP;                      // each MMA covers all 128 rows of the tile
    constexpr int MN      = kPP ? 128 : NQ;                        // the MMA's N width
    const int ew = warp - kEpiWarp0;                                 // 0..7
    const int wg = ew >> 2;
    const int te = static_cast<int>(threadIdx.x) - 32 * kEpiWarp0;  // 0..255
    // rows-on-M: fragment rows r0 and r0 + 8 of the tile; queries-on-M: query rows q0 and q0 + 8, list rows from rb on
    const int r0 = 64 * wg + 16 * (ew & 3) + (lane >> 2);
    const int q0 = (NQ == 128 ? 64 * wg : 0) + 16 * (ew & 3) + (lane >> 2);
    const int rb = (kWhole ? 0 : 64 * wg) + 2 * (lane & 3);
    const uint32_t q_lo0   = ptx::smem_desc_lo(ptx::smem_u32(sQ)) + (NQ == 128 ? wg * 512 : 0);  // + 64 rows of 128 B
    const uint32_t d_lo0   = ptx::smem_desc_lo(ptx::smem_u32(sDec)) + (kWhole ? 0 : wg * 512);
    const uint32_t x_lo0   = ptx::smem_desc_lo(ptx::smem_u32(sDec + NKB * kDecTile)) + (kWhole ? 0 : wg * 128);  // 32 B rows
    const uint32_t ones_lo = ptx::smem_desc_lo(ptx::smem_u32(sOnes));
    const int cap = P.cap, KC = P.KC;
    const int kth = (P.kth > 0 && P.kth < KC) ? P.kth : KC;
    // this warpgroup's threshold / counter / buffer set (ping-pong: one per warpgroup) and the other warpgroup's thresholds
    float* thr_w = sThr + (kPP ? wg * NQ : 0);
    const float* thr_x = sThr + (kPP ? (wg ^ 1) * NQ : 0);
    int* cnt_w = sCnt + (kPP ? wg * NQ : 0);
    unsigned long long* cand_w = sCand + (kPP ? wg * NQ * cap : 0);
    // the barrier of the overflow loop and the warps that compact: the warpgroup's own (ping-pong), or both warpgroups.
    // (A run-time barrier id makes ptxas reserve all 16 named barriers, which is harmless at one CTA per SM.)
    const uint32_t bar_id = kPP ? 2 + wg : 1, bar_n = kPP ? 128 : kEpiThreads;
    const int cw0 = kPP ? (ew & 3) : ew, cwn = kPP ? 4 : kEpiWarps;
    uint32_t ds = kPP ? wg : 0, dph = 0, qph = 0, ss = 0, sp = 0;
    uint32_t g0 = 0;  // ping-pong: running tile number of the item's first tile

    // compaction: keep the KC best at the front, tighten the column's threshold to its kth best
    auto compact = [&](int col) {
      unsigned long long k[4];
      int r[4];
      unsigned long long* buf = cand_w + col * cap;
      const int n = min(cnt_w[col], cap);
      pq_rank_select(buf, n, nullptr, 0, lane, k, r);
      __syncwarp();
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (k[e] != 0ull && r[e] < KC) buf[r[e]] = k[e];
        if (n >= kth && k[e] != 0ull && r[e] == kth - 1) thr_w[col] = fmaxf(thr_w[col], __uint_as_float(okey_inv(static_cast<uint32_t>(k[e] >> 32))));
      }
      if (lane == 0) cnt_w[col] = min(n, KC);
      __syncwarp();
    };

    for (;;) {
      ptx::mbar_wait(&s_full[ss], sp);
      const int it = __shfl_sync(0xffffffffu, s_item[ss], 0);  // (consumes the load before the slot is handed back)
      if (lane == 0) ptx::mbar_arrive(&s_empty[ss]);
      if (++ss == kSched) { ss = 0; sp ^= 1; }
      if (it < 0) break;
      const tc_item item = P.items[it];
      if constexpr (STORE) {
        ptx::mbar_wait(q_full, qph);
        const int64_t seg = static_cast<int64_t>(item.n_tiles) * 128;  // a pair's segment: its list's padded rows
        float* out        = P.out_score + item.out_off;
        for (uint32_t t = 0; t < item.n_tiles; ++t) {
          ptx::mbar_wait(&d_full[ds], dph);
          float d[MN / 2];
          pq_tile_mma<MN, kQM, NKB, PASSES>(d, ds, L::dec_stage >> 4, d_lo0, x_lo0, q_lo0, L::q_tile >> 4, ones_lo);
          __syncwarp();
          if (lane == 0) {
            ptx::mbar_arrive(&d_empty[ds]);
            if (t + 1 == item.n_tiles) ptx::mbar_arrive(q_empty);
          }
          if (++ds == kDecStages) { ds = 0; dph ^= 1; }
          // score = -accumulator, as the filtering epilogue reports it
          if constexpr (kQM) {
            // query rows q0, q0 + 8; list rows rb + 8j + {0, 1}: one float2 per lane, a quad writes 8 consecutive rows (32 B)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int q = q0 + 8 * h;
              if (static_cast<uint32_t>(q) < item.valid_rows) {
                float* o = out + q * seg + t * 128 + rb;
#pragma unroll
                for (int j = 0; j < NQ / 8; ++j)
                  *reinterpret_cast<float2*>(o + 8 * j) = make_float2(-d[4 * j + 2 * h], -d[4 * j + 2 * h + 1]);
              }
            }
          } else {
            // list rows r0, r0 + 8; query columns 8j + 2 (lane % 4) + {0, 1}: the 8 lanes of one column write 8 consecutive rows
#pragma unroll
            for (int j = 0; j < NQ / 8; ++j)
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const int col = 8 * j + 2 * (lane & 3) + (e & 1);
                if (static_cast<uint32_t>(col) < item.valid_rows) out[col * seg + t * 128 + r0 + 8 * (e >> 1)] = -d[4 * j + e];
              }
          }
        }
        qph ^= 1;
      } else {
        // per-column state: running threshold in t = -(score) units (a row is a candidate iff t > thr), empty buffer; one set
        // per warpgroup in ping-pong
        for (int i = te; i < L::n_sets * NQ; i += kEpiThreads) {
          const int col = i % NQ;
          float thr     = INFINITY;  // columns past the item's queries never collect anything
          if (static_cast<uint32_t>(col) < item.valid_rows) {
            thr = -INFINITY;
            if (P.b_keys != nullptr) {
              const uint32_t arow = item.a_row0 + col;
              const int kb        = *reinterpret_cast<volatile int*>(P.b_keys + (P.b_idx ? P.b_idx[arow] : arow));
              const float bv      = __int_as_float(kb >= 0 ? kb : kb ^ 0x7fffffff);
              thr                 = -((bv - (P.b_add ? P.b_add[arow] : 0.f)) / P.b_scale);
            }
          }
          sThr[i] = thr;
          sCnt[i] = 0;
        }
        ptx::named_bar_sync(1, kEpiThreads);
        ptx::mbar_wait(q_full, qph);

        // ping-pong: this warpgroup's tiles of the item are t0, t0 + 2, ...; it may have none (an item of one tile)
        const uint32_t t0 = kPP ? (wg ^ (g0 & 1u)) : 0, tstep = kPP ? 2 : 1;
        if (kPP && t0 >= item.n_tiles && lane == 0) ptx::mbar_arrive(q_empty);
        for (uint32_t t = t0; t < item.n_tiles; t += tstep) {
          ptx::mbar_wait(&d_full[ds], dph);
          float d[MN / 2];
          pq_tile_mma<MN, kQM, NKB, PASSES>(d, ds, L::dec_stage >> 4, d_lo0, x_lo0, q_lo0, L::q_tile >> 4, ones_lo);
          __syncwarp();
          if (lane == 0) {
            ptx::mbar_arrive(&d_empty[ds]);
            if (t + tstep >= item.n_tiles) ptx::mbar_arrive(q_empty);  // the item's residual rows may be replaced
          }
          if (kPP) dph ^= 1;  // (the warpgroup's own stage)
          else if (++ds == kDecStages) { ds = 0; dph ^= 1; }

          const uint32_t pos0 = item.b_row0 + t * 128 + (kQM ? rb : r0);
          auto filter = [&](uint64_t only) -> uint64_t {
            if constexpr (kQM) {
              // (a warpgroup's thresholds change only in its own compaction, between its overflow barriers: read once per pass)
              float th[2] = {thr_w[q0], thr_w[q0 + 8]};
              if constexpr (kPP) {
                // The other warpgroup's buffer may hold rows of LATER tiles, which lose exact ties to this tile's rows: against
                // its threshold a row is kept iff t >= thr_x, not t > thr_x.  (Its own buffer holds only earlier rows, which
                // win ties, so t > thr_w is exact.)  thr_x can rise while this runs: a stale value only keeps more rows.
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  const float tx = thr_x[q0 + 8 * h];
                  if (tx > th[h]) th[h] = nextafterf(tx, -INFINITY);
                }
              }
              return pq_filter_rows<MN>(d, only, q0, pos0, th, cnt_w, cand_w, cap);
            } else {
              return pq_filter_frag<NQ>(d, only, lane, pos0, pos0 + 8, sThr, sCnt, sCand, cap);
            }
          };
          uint64_t left = filter(~0ull);
          // ONE barrier per tile (of the warpgroup in ping-pong, else of both) decides whether any buffer overflowed
          while (bar_red_or(bar_id, bar_n, left != 0)) {
            for (int col = cw0; col < NQ; col += cwn)
              if (cnt_w[col] > cap) compact(col);  // (warp-uniform: every lane reads the same counter)
            ptx::named_bar_sync(bar_id, bar_n);
            if (left != 0) left = filter(left);
          }
        }
        qph ^= 1;
        if constexpr (kPP) {
          g0 += item.n_tiles;
          // both warpgroups' buffers are final; the read-out ranks their union (<= 2 cap <= 128 entries, see launch())
          ptx::named_bar_sync(1, kEpiThreads);
        }

        // item done: every column's KC best -> global; publish the query's k-th best for the other items of the same query
        for (int col = ew; col < static_cast<int>(min(item.valid_rows, static_cast<uint32_t>(NQ))); col += kEpiWarps) {
          unsigned long long k[4];
          int r[4];
          const int n0 = min(sCnt[col], cap), n1 = kPP ? min(sCnt[NQ + col], cap) : 0;  // (ping-pong: the union of both sets)
          pq_rank_select(sCand + col * cap, n0, sCand + (NQ + col) * cap, n1, lane, k, r);
          const int n  = n0 + n1;
          const int nk = min(n, KC);
          const uint32_t arow = item.a_row0 + col;
          const int64_t o     = static_cast<int64_t>(item.out_off) + static_cast<int64_t>(col) * P.out_row_stride;
          auto emit = [&](unsigned long long key, int r) {
            if (key == 0ull || r >= KC) return;
            const float t = __uint_as_float(okey_inv(static_cast<uint32_t>(key >> 32)));
            if (P.out_score != nullptr) { P.out_score[o + r] = -t; P.out_pos[o + r] = ~static_cast<uint32_t>(key); }
            if (r == kth - 1 && P.b_keys != nullptr) {  // (n >= kth holds when such a rank exists)
              const float pub = __fmaf_rn(P.b_scale, -t, P.b_add ? P.b_add[arow] : 0.f);
              const int kp    = __float_as_int(pub);
              atomicMin(P.b_keys + (P.b_idx ? P.b_idx[arow] : arow), kp >= 0 ? kp : kp ^ 0x7fffffff);
            }
          };
#pragma unroll
          for (int e = 0; e < 4; ++e) emit(k[e], r[e]);
          if (P.out_score != nullptr)
            for (int slot = nk + lane; slot < KC; slot += 32) { P.out_score[o + slot] = INFINITY; P.out_pos[o + slot] = 0xffffffffu; }
        }
        ptx::named_bar_sync(1, kEpiThreads);  // the next item's column init must not overtake another warp's read-out
      }
    }
  }
}

// ------------------------------------------------------------------------------------ build-side kernels
// one CTA per 128-row tile: codes [128, pq_dim] -> lane-transposed 16-byte chunks + half norms
__global__ void __launch_bounds__(128)
pq_stream_build_kernel(const uint8_t* __restrict__ codes, const int64_t* __restrict__ ids, int64_t pad_id, int pq_dim,
                       const float* __restrict__ pq_centers, bool ip, uint8_t* __restrict__ stream)
{
  __shared__ __align__(16) uint8_t sc[128 * 64];
  const int64_t tile = blockIdx.x;
  const int r        = threadIdx.x;
  const int64_t row  = tile * 128 + r;
  const int64_t blk  = 128 * static_cast<int64_t>(pq_dim) + 512;
  const uint8_t* src = codes + row * pq_dim;
  float nrm = 0.f;
  for (int j = 0; j < pq_dim; ++j) {
    const int c = src[j];
    sc[r * pq_dim + j] = static_cast<uint8_t>(c);
    const float e0 = __bfloat162float(__float2bfloat16_rn(pq_centers[(static_cast<int64_t>(j) * 2 + 0) * 256 + c]));
    const float e1 = __bfloat162float(__float2bfloat16_rn(pq_centers[(static_cast<int64_t>(j) * 2 + 1) * 256 + c]));
    nrm = fmaf(e0, e0, nrm);
    nrm = fmaf(e1, e1, nrm);
  }
  __syncthreads();
  uint8_t* out  = stream + tile * blk;
  const int nh  = pq_dim / 32;
  for (int o = threadIdx.x; o < 8 * nh * 32; o += blockDim.x) {
    const int g = o / (nh * 32), h = (o / 32) % nh, l = o % 32;
    uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
    for (int i = 0; i < 16; ++i) w[i >> 2] |= static_cast<uint32_t>(sc[(16 * g + i) * pq_dim + 32 * h + l]) << ((i & 3) * 8);
    reinterpret_cast<uint4*>(out)[o] = make_uint4(w[0], w[1], w[2], w[3]);
  }
  reinterpret_cast<float*>(out + 128 * pq_dim)[r] = ids[row] == pad_id ? INFINITY : (ip ? 0.f : 0.5f * nrm);
}

// inverse of pq_stream_build_kernel: one CTA per tile, stream block -> codes [128, pq_dim] one code per byte
__global__ void __launch_bounds__(128) pq_stream_to_flat_kernel(const uint8_t* __restrict__ stream, int pq_dim, uint8_t* __restrict__ codes)
{
  __shared__ __align__(16) uint8_t sc[128 * 64];
  const int64_t tile = blockIdx.x;
  const int64_t blk  = 128 * static_cast<int64_t>(pq_dim) + 512;
  const uint8_t* in  = stream + tile * blk;
  const int nh       = pq_dim / 32;
  for (int o = threadIdx.x; o < 8 * nh * 32; o += blockDim.x) {
    const int g = o / (nh * 32), h = (o / 32) % nh, l = o % 32;
    const uint4 w = reinterpret_cast<const uint4*>(in)[o];
    const uint32_t w4[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int i = 0; i < 16; ++i) sc[(16 * g + i) * pq_dim + 32 * h + l] = static_cast<uint8_t>((w4[i >> 2] >> ((i & 3) * 8)) & 0xffu);
  }
  __syncthreads();
  uint4* out = reinterpret_cast<uint4*>(codes + tile * 128 * pq_dim);
  for (int o = threadIdx.x; o < 128 * pq_dim / 16; o += blockDim.x) out[o] = reinterpret_cast<const uint4*>(sc)[o];
}

// ------------------------------------------------------------------------------------ pruning-bound pre-pass
// One warp per query (grid-stride).  The query's first n_pair_probes live probes (probes are in rank order: nearest first), the
// first n_tiles tiles of each probe's list: every row scored in fp32, s = hn - r.y, by the decode warps' gather (lane l owns
// subspaces l + 32 h, 16 rows per 128-bit code load) and a shuffle reduce-scatter that leaves row 16 g + lane / 2 on the even
// lanes.  Each row's score is raised by the margin below and turned into a distance as the merge does (fmaf(scale, s, add));
// every even lane keeps its kPrimeKeep smallest, and the k-th smallest of those kept values -- if finite, at least k rows lie at or
// below it -- is raised once more and min-ed into the query's bound.  DESIGN.md §5 ("Bound pre-pass") gives the argument.
constexpr int kPrimeWarps = 8;
constexpr int kPrimeKeep  = 4;  // per even lane: 16 lanes x 4 >= 64 >= k

// One step of the reduce-scatter of 2N per-lane partial sums over lane bit 2N: the lane keeps the N rows its bit selects,
// summed with its partner's.  (selp in asm: a plain select between two elements becomes a computed index into local memory.)
template <int N>
__device__ __forceinline__ void prime_reduce_step(float (&part)[16], int lane)
{
  const uint32_t up = (lane & (2 * N)) != 0 ? 1u : 0u;
#pragma unroll
  for (int i = 0; i < N; ++i) {
    float give, keep;
    asm("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %4, 0;\n\tselp.f32 %0, %2, %3, p;\n\tselp.f32 %1, %3, %2, p;\n\t}"
        : "=f"(give), "=f"(keep) : "f"(part[i]), "f"(part[i + N]), "r"(up));
    part[i] = keep + __shfl_xor_sync(0xffffffffu, give, 2 * N);
  }
}

template <int NKB, int PASSES>
__global__ void __launch_bounds__(32 * kPrimeWarps, 3)  // (3 CTAs per SM: shared memory allows 3, see pq_bound_prime)
pq_bound_prime_kernel(const uint8_t* __restrict__ stream, const uint32_t* __restrict__ cb_words, const __nv_bfloat16* __restrict__ q_hi,
                      const __nv_bfloat16* __restrict__ q_lo, const uint32_t* __restrict__ slot_of, const uint32_t* __restrict__ pair_list,
                      const int64_t* __restrict__ list_offsets, const float* __restrict__ add, float scale, int64_t nq, int n_probes,
                      int n_pair_probes, int n_tiles, int k, int* __restrict__ b_keys)
{
  constexpr int Kp    = 64 * NKB;     // residual columns: 2 per subspace, pq_dim = 32 NKB
  constexpr int codes = 4096 * NKB;   // code bytes of a tile block, followed by the 128 half-norms
  constexpr int blk   = codes + 512;
  extern __shared__ __align__(16) uint32_t sCbw[];  // [NKB][256][32] codebook words, then ymax[Kp]
  float* sYmax = reinterpret_cast<float*>(sCbw + NKB * 8192);
  for (int i = threadIdx.x; i < NKB * 8192 / 4; i += blockDim.x)
    reinterpret_cast<uint4*>(sCbw)[i] = reinterpret_cast<const uint4*>(cb_words)[i];
  __syncthreads();
  // ymax[c] = max over codes of |entry| of column c (column 2 j + e = component e of subspace j): with it,
  // sum_j |r_j y_j| <= sum_j |r_j| ymax_j for every row of the query's lists
  // (every thread: one column, one 1/nsplit of the codes; the partial maxima meet in shared memory as non-negative floats,
  // whose bit patterns order like the floats)
  for (int c = threadIdx.x; c < Kp; c += blockDim.x) sYmax[c] = 0.f;
  __syncthreads();
  {
    constexpr int nsplit = 32 * kPrimeWarps / Kp;
    const int c = threadIdx.x % Kp, part = threadIdx.x / Kp;
    const int j = c >> 1, h = j >> 5, l = j & 31;
    float m = 0.f;
#pragma unroll 8
    for (int code = part; code < 256; code += nsplit) {
      const uint32_t w = sCbw[(h * 256 + code) * 32 + l];
      m = fmaxf(m, fabsf(__uint_as_float((c & 1) ? (w & 0xffff0000u) : (w << 16))));
    }
    atomicMax(reinterpret_cast<int*>(sYmax) + c, __float_as_int(m));
  }
  __syncthreads();

  const int lane = threadIdx.x & 31;
  const uint32_t cb_lane = ptx::smem_u32(sCbw) + static_cast<uint32_t>(lane) * 4u;
  for (int64_t q = blockIdx.x * static_cast<int64_t>(kPrimeWarps) + (threadIdx.x >> 5); q < nq; q += gridDim.x * static_cast<int64_t>(kPrimeWarps)) {
    const uint32_t* slots = slot_of + q * n_probes;
    // M = max |add| over the query's pairs: every pair converts the bound back to a threshold with its own add
    float amax = 0.f;
    for (int p = lane; p < n_probes; p += 32) {
      const uint32_t s = slots[p];
      if (s != 0xffffffffu) amax = fmaxf(amax, fabsf(add[s]));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));

    float best[kPrimeKeep];
#pragma unroll
    for (int j = 0; j < kPrimeKeep; ++j) best[j] = INFINITY;
    int taken = 0;
    for (int p = 0; p < n_probes && taken < n_pair_probes; ++p) {
      const uint32_t slot = slots[p];
      if (slot == 0xffffffffu) continue;
      ++taken;
      const float a = add[slot];
      // this lane's residual columns 64 h + 2 lane + {0, 1} (one bf16x2 word per plane), and A = sum_j |r_j| ymax_j
      float r[NKB][2][PASSES];
      float A = 0.f;
#pragma unroll
      for (int h = 0; h < NKB; ++h)
#pragma unroll
        for (int pl = 0; pl < PASSES; ++pl) {
          const __nv_bfloat16* src = pl == 0 ? q_hi : q_lo;
          const uint32_t w = *reinterpret_cast<const uint32_t*>(src + static_cast<int64_t>(slot) * Kp + 64 * h + 2 * lane);
          r[h][0][pl] = __uint_as_float(w << 16);
          r[h][1][pl] = __uint_as_float(w & 0xffff0000u);
          A = fmaf(fabsf(r[h][0][pl]), sYmax[64 * h + 2 * lane], A);
          A = fmaf(fabsf(r[h][1][pl]), sYmax[64 * h + 2 * lane + 1], A);
        }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) A += __shfl_xor_sync(0xffffffffu, A, o);
      const uint32_t l   = pair_list[slot];
      const int64_t row0 = list_offsets[l];
      const int nt       = static_cast<int>(min(static_cast<int64_t>(n_tiles), (list_offsets[l + 1] - row0) / 128));
      // 16-row groups of the scored tiles in order; the codes and half-norm of the next group load while this one is scored
      const uint8_t* first = stream + (row0 / 128) * blk;
      auto group_codes = [&](int tg, int h) {
        return *reinterpret_cast<const uint4*>(first + (tg >> 3) * blk + (tg & 7) * (NKB * 512) + h * 512 + lane * 16);
      };
      auto group_hn = [&](int tg) { return reinterpret_cast<const float*>(first + (tg >> 3) * blk + codes)[16 * (tg & 7) + (lane >> 1)]; };
      uint4 nxt[NKB];
      float nxt_hn = 0.f;
      if (nt > 0) {
#pragma unroll
        for (int h = 0; h < NKB; ++h) nxt[h] = group_codes(0, h);
        nxt_hn = group_hn(0);
      }
      for (int tg = 0; tg < 8 * nt; ++tg) {
        uint4 cur[NKB];
#pragma unroll
        for (int h = 0; h < NKB; ++h) cur[h] = nxt[h];
        const float hn = nxt_hn;
        if (tg + 1 < 8 * nt) {
#pragma unroll
          for (int h = 0; h < NKB; ++h) nxt[h] = group_codes(tg + 1, h);
          nxt_hn = group_hn(tg + 1);
        }
        {
          float part[16];
#pragma unroll
          for (int i = 0; i < 16; ++i) part[i] = 0.f;
#pragma unroll
          for (int h = 0; h < NKB; ++h) {
            const uint4 cw = cur[h];
            const uint32_t w4[4] = {cw.x, cw.y, cw.z, cw.w};
#pragma unroll
            for (int i = 0; i < 16; ++i) {
              const uint32_t c = __byte_perm(w4[i >> 2], 0u, 0x4440u | static_cast<uint32_t>(i & 3));
              uint32_t w;
              asm("ld.shared.u32 %0, [%1];" : "=r"(w) : "r"(cb_lane + static_cast<uint32_t>(h) * 32768u + (c << 7)));
              const float e0 = __uint_as_float(w << 16), e1 = __uint_as_float(w & 0xffff0000u);
#pragma unroll
              for (int pl = 0; pl < PASSES; ++pl) {
                part[i] = fmaf(r[h][0][pl], e0, part[i]);
                part[i] = fmaf(r[h][1][pl], e1, part[i]);
              }
            }
          }
          prime_reduce_step<8>(part, lane);
          prime_reduce_step<4>(part, lane);
          prime_reduce_step<2>(part, lane);
          prime_reduce_step<1>(part, lane);
          const float dot = part[0] + __shfl_xor_sync(0xffffffffu, part[0], 1);  // row 16 (tg % 8) + lane / 2 of the tile
          if ((lane & 1) == 0 && hn < INFINITY) {  // (padding rows: hn = +inf)
            const float sp = hn - dot;
            const float m  = __fmul_ru(0x1p-12f, __fadd_ru(fabsf(hn), A));
            float u        = __fmaf_rn(scale, __fadd_ru(sp, m), a);
#pragma unroll
            for (int j = 0; j < kPrimeKeep; ++j) {
              const float lo = fminf(best[j], u);
              u              = fmaxf(best[j], u);
              best[j]        = lo;
            }
          }
        }
      }
    }
    // k-th smallest of the kept values (odd lanes keep +inf): bisection over the order-preserving keys, the smallest key with
    // at least k kept keys at or below it, i.e. the k-th smallest kept value itself
    uint32_t key[kPrimeKeep];
#pragma unroll
    for (int j = 0; j < kPrimeKeep; ++j) key[j] = okey(__float_as_uint(best[j]));
    uint32_t lo = 0u, hi = 0xffffffffu;
    while (lo < hi) {  // (warp-uniform)
      const uint32_t mid = lo + ((hi - lo) >> 1);
      uint32_t c = 0;
#pragma unroll
      for (int j = 0; j < kPrimeKeep; ++j) c += key[j] <= mid ? 1u : 0u;
      if (__reduce_add_sync(0xffffffffu, c) >= static_cast<uint32_t>(k)) hi = mid;
      else lo = mid + 1u;
    }
    const float kth = __uint_as_float(okey_inv(lo));
    if (lane == 0 && kth < INFINITY) {
      const float B = __fadd_ru(__fadd_ru(kth, __fmul_ru(0x1p-21f, __fadd_ru(fabsf(kth), amax))), 1e-30f);
      if (B < INFINITY) {
        const int kb = __float_as_int(B);
        atomicMin(b_keys + q, kb >= 0 ? kb : kb ^ 0x7fffffff);
      }
    }
  }
}

__global__ void pq_cb_words_kernel(const float* __restrict__ pq_centers, int pq_dim, uint32_t* __restrict__ words)
{
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (pq_dim / 32) * 256 * 32) return;
  const int l = t & 31, c = (t >> 5) & 255, h = t >> 13;
  const int j = 32 * h + l;
  const __nv_bfloat16 e0 = __float2bfloat16_rn(pq_centers[(static_cast<int64_t>(j) * 2 + 0) * 256 + c]);
  const __nv_bfloat16 e1 = __float2bfloat16_rn(pq_centers[(static_cast<int64_t>(j) * 2 + 1) * 256 + c]);
  words[t] = static_cast<uint32_t>(__bfloat16_as_ushort(e0)) | (static_cast<uint32_t>(__bfloat16_as_ushort(e1)) << 16);
}

using encode_fn_t = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                 const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                 CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

encode_fn_t get_encode_fn()
{
  static encode_fn_t fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<encode_fn_t>(p);
  });
  B2_EXPECTS(fn != nullptr, "cuTensorMapEncodeTiled is not available from this driver");
  return fn;
}

// residual rows [rows, Kp] bf16, box = 64 columns x `group` rows, SWIZZLE_128B
CUtensorMap make_query_map(const __nv_bfloat16* ptr, int64_t rows, int Kp, int group)
{
  CUtensorMap m;
  cuuint64_t gdim[2]    = {static_cast<cuuint64_t>(Kp), static_cast<cuuint64_t>(rows)};
  cuuint64_t gstride[1] = {static_cast<cuuint64_t>(Kp) * sizeof(__nv_bfloat16)};
  cuuint32_t box[2]     = {64, static_cast<cuuint32_t>(group)};
  cuuint32_t estr[2]    = {1, 1};
  CUresult r = get_encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<__nv_bfloat16*>(ptr), gdim, gstride, box, estr,
                               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  B2_EXPECTS(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled (pq residual rows) failed with code %d (rows=%lld Kp=%d)", int(r), (long long)rows, Kp);
  return m;
}

int env_int(const char* name, int dflt)
{
  const char* v = getenv(name);
  return v ? atoi(v) : dflt;
}

// KC = 0: the store epilogue; otherwise the filtering one, which has no NQ = 128 two-pass kernel (pq_stream_scan rejects it)
template <int NQ, int NKB, int PASSES>
void launch(cudaStream_t stream, int sms, const CUtensorMap& mq_hi, const CUtensorMap& mq_lo, pq_args a, int n_items)
{
  using L          = layout<NQ, NKB, PASSES>;
  const bool store = a.KC == 0;
  auto kern        = pq_stream_scan_kernel<NQ, NKB, PASSES, true>;
  if constexpr (NQ < 128 || PASSES == 1)
    if (!store) kern = pq_stream_scan_kernel<NQ, NKB, PASSES>;
  // free slots between compactions: cap - KC.  Ping-pong keeps one buffer set per warpgroup (L::n_sets), each with KC + 16.
  a.cap = pq_pingpong(NQ, PASSES) ? a.KC + 16 : (a.KC <= 16 ? (NQ == 128 ? 32 : 64) : (a.KC <= 32 ? 64 : 128));
  if (const int cap_env = env_int("CUVS_B200_PQ_CAP", 0)) a.cap = std::max(a.KC + 8, std::min(128, cap_env));  // bisection knob
  if (store) a.cap = 0;  // no candidate buffers
  B2_EXPECTS(L::n_sets * a.cap <= 128, "pq_stream_scan: %d candidate buffer entries per query exceed the read-out's 128", L::n_sets * a.cap);
  const int fixed = L::off_cand + L::n_sets * NQ * a.cap * 8 + 1024 /*alignment slack of the dynamic segment*/;
  a.cstages = std::min(kMaxCStages, (kSmemLimit - fixed) / a.blk);
  B2_EXPECTS(a.cstages >= 2, "pq_stream_scan: shared memory budget exceeded (NQ=%d KC=%d passes=%d)", NQ, a.KC, PASSES);
  const size_t smem = static_cast<size_t>(fixed) + static_cast<size_t>(a.cstages) * a.blk;
  if (env_int("CUVS_B200_PQ_DEBUG", 0))  // the launch configuration, on stderr
    fprintf(stderr, "[pq_stream_scan] NQ=%d NKB=%d PASSES=%d KC=%d cap=%d cstages=%d blk=%d smem=%zu items<=%d\n", NQ, NKB, PASSES, a.KC, a.cap,
            a.cstages, a.blk, smem, n_items);
  B2_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  const int grid = n_items < sms ? n_items : sms;
  timed_section ts("pq_stream_scan", stream);
  count_launch();
  kern<<<grid, kThreads, smem, stream>>>(mq_hi, mq_lo, a);
  B2_CUDA(cudaGetLastError());
}

}  // namespace

bool pq_stream_supported(int device, int pq_dim, int pq_len, int pq_bits, bool per_subspace)
{
  int major = 0;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device) != cudaSuccess) return false;
  return major == 9 && pq_bits == 8 && per_subspace && pq_len == 2 && (pq_dim == 32 || pq_dim == 64);
}

void pq_stream_build(cudaStream_t s, const uint8_t* codes, const int64_t* ids, int64_t pad_id, int64_t rows_total, int pq_dim,
                     const float* pq_centers, bool ip, uint8_t* stream, uint32_t* cb_words)
{
  B2_EXPECTS(pq_dim == 32 || pq_dim == 64, "pq_stream_build: pq_dim must be 32 or 64");
  B2_EXPECTS(rows_total % 128 == 0, "pq_stream_build: lists must be padded to 128-row tiles");
  count_launch();
  pq_cb_words_kernel<<<(pq_dim / 32) * 256 * 32 / 256, 256, 0, s>>>(pq_centers, pq_dim, cb_words);
  if (rows_total > 0) {
    count_launch();
    pq_stream_build_kernel<<<static_cast<unsigned>(rows_total / 128), 128, 0, s>>>(codes, ids, pad_id, pq_dim, pq_centers, ip, stream);
  }
  B2_CUDA(cudaGetLastError());
}

void pq_stream_to_flat(cudaStream_t s, const uint8_t* stream, int64_t rows_total, int pq_dim, uint8_t* codes)
{
  B2_EXPECTS(pq_dim == 32 || pq_dim == 64, "pq_stream_to_flat: pq_dim must be 32 or 64");
  if (rows_total == 0) return;
  count_launch();
  pq_stream_to_flat_kernel<<<static_cast<unsigned>(rows_total / 128), 128, 0, s>>>(stream, pq_dim, codes);
  B2_CUDA(cudaGetLastError());
}

void pq_bound_prime(cudaStream_t s, int device, const uint8_t* code_stream, const uint32_t* cb_words, int pq_dim, const __nv_bfloat16* q_hi,
                    const __nv_bfloat16* q_lo, int Kp, int passes, const uint32_t* slot_of, const uint32_t* pair_list, const int64_t* list_offsets,
                    const float* add, float scale, int64_t nq, int n_probes, int k, int* b_keys)
{
  // Scored rows per query: the first 4 tiles (512 rows) of its nearest list.  Chosen by a sweep on the 50M x 128 flagship
  // (DESIGN.md §5): scan + pre-pass was lowest at P = 1, T = 4; more tiles still shorten the scan, but past 4 each costs
  // ~35 us per 10k queries (one more 8.7 KB tile per query, decoded by one warp), more than the scan then saves; a second
  // list saved less than more tiles of the first.
  constexpr int kPrimeProbes = 1, kPrimeTiles = 4;
  if (nq == 0) return;
  B2_EXPECTS(Kp == 2 * pq_dim && (pq_dim == 32 || pq_dim == 64), "pq_bound_prime: pq_dim must be 32 or 64 with pq_len 2 (Kp=%d)", Kp);
  B2_EXPECTS(passes == 1 || (passes == 2 && q_lo != nullptr), "pq_bound_prime: passes must be 1, or 2 with a lo plane");
  B2_EXPECTS(k >= 1 && k <= 16 * kPrimeKeep, "pq_bound_prime: k must be in [1, %d]", 16 * kPrimeKeep);
  const int nkb      = pq_dim / 32;
  const size_t smem  = static_cast<size_t>(nkb) * 32768 + static_cast<size_t>(nkb) * 64 * sizeof(float);
  const int64_t need = (nq + kPrimeWarps - 1) / kPrimeWarps;
  const int grid     = static_cast<int>(std::min<int64_t>(need, 3 * static_cast<int64_t>(sm_count_of(device))));  // 3 fit per SM
  auto run = [&](auto kern) {
    B2_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    count_launch();
    kern<<<grid, 32 * kPrimeWarps, smem, s>>>(code_stream, cb_words, q_hi, q_lo, slot_of, pair_list, list_offsets, add, scale, nq, n_probes,
                                              kPrimeProbes, kPrimeTiles, k, b_keys);
  };
  if (nkb == 1) passes == 1 ? run(pq_bound_prime_kernel<1, 1>) : run(pq_bound_prime_kernel<1, 2>);
  else passes == 1 ? run(pq_bound_prime_kernel<2, 1>) : run(pq_bound_prime_kernel<2, 2>);
  B2_CUDA(cudaGetLastError());
}

bool pq_stream_bound_enabled() { return env_int("CUVS_B200_PQ_NO_BOUND", 0) == 0; }

int pq_stream_group(double pairs_per_list, int KC, int passes)
{
  const int forced = env_int("CUVS_B200_PQ_GROUP", 0);  // tests and limiter experiments (read per call)
  int g = pairs_per_list <= 20.0 ? 32 : (pairs_per_list <= 80.0 ? 64 : 128);
  if (forced == 32 || forced == 64 || forced == 128) g = forced;
  if (KC == 0) return g;                           // store epilogue: no candidate buffers, every width fits
  if ((KC > 16 || passes == 2) && g > 64) g = 64;  // shared-memory budget: wide candidate buffers / two residual planes
  if (KC > 32) g = 32;                             // 128-entry buffers (k in 33..64): 32 query columns per item
  return g;
}

void pq_stream_scan(cudaStream_t stream, int device, const __nv_bfloat16* q_hi, const __nv_bfloat16* q_lo, int64_t a_rows, int Kp,
                    const uint8_t* code_stream, const uint32_t* cb_words, int pq_dim, const tc_item* items_dev, int n_items,
                    const int* n_items_dev, int group, int KC, int passes, float* out_score, uint32_t* out_pos, int64_t out_row_stride,
                    const tc_bound* bound)
{
  if (n_items == 0) return;
  B2_EXPECTS(Kp == 2 * pq_dim && (pq_dim == 32 || pq_dim == 64), "pq_stream_scan: pq_dim must be 32 or 64 with pq_len 2 (Kp=%d)", Kp);
  B2_EXPECTS(KC == 0 || KC == 16 || KC == 32 || KC == 64, "pq_stream_scan: KC must be 0 (store), 16, 32 or 64");
  B2_EXPECTS(passes == 1 || (passes == 2 && q_lo != nullptr), "pq_stream_scan: passes must be 1, or 2 with a lo plane");
  B2_EXPECTS(group == 32 || (group == 64 && KC <= 32) || (group == 128 && (KC == 0 || (KC == 16 && passes == 1))),
             "pq_stream_scan: unsupported group %d", group);
  B2_EXPECTS(a_rows >= group, "pq_stream_scan: the residual plane must hold at least one group of rows");
  pq_args a{};
  a.stream = code_stream;
  a.cb_words = cb_words;
  a.items = items_dev;
  a.n_items_dev = n_items_dev;
  a.out_score = out_score;
  a.out_pos = out_pos;
  a.out_row_stride = out_row_stride;
  if (KC > 0 && bound != nullptr && bound->keys != nullptr && pq_stream_bound_enabled()) {
    a.b_keys = bound->keys;
    a.b_idx = bound->idx;
    a.b_add = bound->add;
    a.b_scale = bound->scale;
    a.kth = bound->kth;
  } else {
    a.b_scale = 1.0f;
  }
  a.n_items_host = n_items;
  a.KC = KC;
  a.blk = static_cast<int>(pq_stream_tile_bytes(pq_dim));
  dbuf<int> sched(1, stream);
  B2_CUDA(cudaMemsetAsync(sched.data(), 0, sizeof(int), stream));
  a.sched = sched.data();
  const CUtensorMap mq  = make_query_map(q_hi, a_rows, Kp, group);
  const CUtensorMap mql = passes == 2 ? make_query_map(q_lo, a_rows, Kp, group) : mq;
  const int sms = sm_count_of(device);
  const int nkb = Kp / 64;
#define B2_PQ_CASE(NQ_, NKB_, P_) \
  if (group == NQ_ && nkb == NKB_ && passes == P_) return launch<NQ_, NKB_, P_>(stream, sms, mq, mql, a, n_items);
  B2_PQ_CASE(32, 1, 1) B2_PQ_CASE(64, 1, 1) B2_PQ_CASE(128, 1, 1) B2_PQ_CASE(32, 2, 1) B2_PQ_CASE(64, 2, 1) B2_PQ_CASE(128, 2, 1)
  B2_PQ_CASE(32, 1, 2) B2_PQ_CASE(64, 1, 2) B2_PQ_CASE(128, 1, 2) B2_PQ_CASE(32, 2, 2) B2_PQ_CASE(64, 2, 2) B2_PQ_CASE(128, 2, 2)
#undef B2_PQ_CASE
  B2_FAIL("pq_stream_scan: no kernel for group=%d Kp=%d passes=%d", group, Kp, passes);
}

}  // namespace b200
