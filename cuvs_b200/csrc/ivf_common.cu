// Shared IVF / k-means machinery: see ivf_common.cuh.
#include "ivf_common.cuh"

#include "exact.cuh"
#include "exact_device.cuh"
#include "hash.cuh"
#include "select_k.cuh"
#include "timing.hpp"

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <vector>

namespace b200 {
namespace {

// Fused coarse search, merge step: one CTA per query ranks the W = splits * lists * KC candidates its items kept
// (sorted lists of KC per centre range and column half) by (score, centre id) — the order select_k imposes on the dense
// score row, where position == centre id — and writes the n_probes best.  The scan rejects a centre only when its score is
// not below a full list's worst entry (its own list's, or through the bound shared between a query's items, another list's at
// an earlier time; such entries only decrease), so every centre outside the candidates scores >= floor = the minimum over
// the full lists of their worst entry.  If the n_probes-th candidate lies STRICTLY below the floor the selection — ties
// included — is the dense one; otherwise, or when fewer than n_probes candidates exist, the query is flagged: its id goes to
// flagged[*n_flagged] (in order of arrival) and the dense fallback recomputes its probes.
constexpr int kCoarseMergeThreads = 128;  // four queries per CTA, one warp each
constexpr int kCoarseMaxW         = 512;
constexpr int kCoarseSlotBits     = 10;  // W < 2^10: a candidate's slot rides in its sort key, below the centre id
constexpr int64_t kCoarseMaxCenters = int64_t(1) << (32 - kCoarseSlotBits);

// Ascending bitonic sort of the warp's 32 E keys, key i = v[i / 32] of lane i % 32: partners 32 or more apart sit in the
// lane's own registers, nearer ones in another lane (shuffles).
template <int E>
__device__ __forceinline__ void warp_bitonic_sort(unsigned long long (&v)[E], int lane)
{
#pragma unroll
  for (int size = 2; size <= 32 * E; size <<= 1) {
#pragma unroll
    for (int j = size >> 1; j > 0; j >>= 1) {
      if (j >= 32) {
#pragma unroll
        for (int e = 0; e < E; ++e) {
          const int f = e ^ (j / 32);
          if (f > e) {
            const bool up = ((e * 32 + lane) & size) == 0;
            const unsigned long long a = v[e], b = v[f];
            if ((a > b) == up) { v[e] = b; v[f] = a; }
          }
        }
      } else {
#pragma unroll
        for (int e = 0; e < E; ++e) {
          const unsigned long long o = __shfl_xor_sync(0xffffffffu, v[e], j);
          const bool up    = ((e * 32 + lane) & size) == 0;
          const bool lower = (lane & j) == 0;
          v[e] = (lower == up) ? (o < v[e] ? o : v[e]) : (o > v[e] ? o : v[e]);
        }
      }
    }
  }
}

// The W keys (score key << 32 | centre id << 10 | slot) of a query, padded to 32 E with ~0, are sorted by its warp; keys
// are unique, so sorted position r holds the candidate of rank r, whose score is read back through its slot.
template <int E>
__global__ void __launch_bounds__(kCoarseMergeThreads)
coarse_merge_kernel(const float* __restrict__ cs, const uint32_t* __restrict__ cp, int64_t nq, int W, int KC, int n_probes,
                    uint32_t* __restrict__ probes, float* __restrict__ probe_scores, int* __restrict__ n_flagged,
                    uint32_t* __restrict__ flagged)
{
  const int64_t q = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
  const int lane  = threadIdx.x & 31;
  if (q >= nq) return;
  float m = INFINITY;
  for (int l = lane; l * KC < W; l += 32) m = fminf(m, cs[q * W + l * KC + KC - 1]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
  const float floor = m;
  unsigned long long v[E];
  int n_valid = 0;
#pragma unroll
  for (int e = 0; e < E; ++e) {
    const int c = e * 32 + lane;
    v[e]        = ~0ull;
    if (c < W) {
      const uint32_t pos = cp[q * W + c];
      if (pos != 0xffffffffu) {
        uint32_t u = __float_as_uint(cs[q * W + c]);
        if ((u << 1) == 0) u = 0;  // -0.0 == +0.0, as in select_k
        u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
        v[e] = (static_cast<unsigned long long>(u) << 32) | (static_cast<unsigned long long>(pos) << kCoarseSlotBits) | c;
      }
    }
    n_valid += __popc(__ballot_sync(0xffffffffu, v[e] != ~0ull));
  }
  warp_bitonic_sort<E>(v, lane);
  bool flag = n_valid < n_probes;
#pragma unroll
  for (int e = 0; e < E; ++e) {
    const int r = e * 32 + lane;
    if (r < n_probes && v[e] != ~0ull) {
      const float score              = cs[q * W + static_cast<int>(v[e] & ((1u << kCoarseSlotBits) - 1))];
      probes[q * n_probes + r]       = static_cast<uint32_t>(v[e]) >> kCoarseSlotBits;
      probe_scores[q * n_probes + r] = score;
      if (r == n_probes - 1 && !(score < floor)) flag = true;  // (strict: also rules out boundary ties)
    }
  }
  if (__any_sync(0xffffffffu, flag) && lane == 0) flagged[atomicAdd(n_flagged, 1)] = static_cast<uint32_t>(q);
}

// Dense fallback of the fused coarse search, for the flagged queries only, in passes of at most `rows` of them (the dense
// score block of a pass is bounded, whatever the batch).  Every launch is sized for a full pass and reads the counts the
// merge left on the device, so the search never waits for the host.  Pass p serves flagged[p * rows ...]: cnt[2] = its
// queries, packed into rows [0, cnt[2]) of the planes, rows up to the next full tile zero; cnt[1] = their tiles, the
// scan's item count.  cnt[0] = all flagged queries.
__global__ void gather_flagged_rows_kernel(const uint4* __restrict__ hi, const uint4* __restrict__ lo, int row_vecs,
                                           const uint32_t* __restrict__ flagged, int* __restrict__ cnt, int64_t first,
                                           int64_t rows, uint4* __restrict__ f_hi, uint4* __restrict__ f_lo)
{
  const int64_t r   = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
  const int lane    = threadIdx.x & 31;
  const int64_t nf  = min(rows, max(static_cast<int64_t>(cnt[0]) - first, int64_t(0)));
  if (r == 0 && lane == 0) {
    cnt[1] = static_cast<int>((nf + kTcTile - 1) / kTcTile);
    cnt[2] = static_cast<int>(nf);
  }
  if (r >= (nf + kTcTile - 1) / kTcTile * kTcTile) return;
  const int64_t src = r < nf ? static_cast<int64_t>(flagged[first + r]) : -1;
  for (int j = lane; j < row_vecs; j += 32) {
    f_hi[r * row_vecs + j] = src >= 0 ? hi[src * row_vecs + j] : make_uint4(0, 0, 0, 0);
    if (f_lo) f_lo[r * row_vecs + j] = src >= 0 ? lo[src * row_vecs + j] : make_uint4(0, 0, 0, 0);
  }
}

// a pass's probes (its row i: flagged query flagged[first + i]) over the fused path's
__global__ void scatter_flagged_probes_kernel(const uint32_t* __restrict__ flagged, const int* __restrict__ cnt, int64_t first,
                                              int n_probes, int64_t total, const uint32_t* __restrict__ f_probes,
                                              const float* __restrict__ f_scores, uint32_t* __restrict__ probes,
                                              float* __restrict__ probe_scores)
{
  const int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (t >= total || t / n_probes >= cnt[2]) return;
  const int64_t at  = static_cast<int64_t>(flagged[first + t / n_probes]) * n_probes + t % n_probes;
  probes[at]        = f_probes[t];
  probe_scores[at]  = f_scores[t];
}

// best entry among the heads of the `lists` sorted candidate lists of each row
__global__ void first_of_rows_kernel(const uint32_t* __restrict__ pos, const float* __restrict__ score, int64_t n, int KC,
                                     int lists, uint32_t* __restrict__ labels, float* __restrict__ out_scores)
{
  int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const int64_t b = i * KC * lists;
  float best      = score[b];
  uint32_t bp     = pos[b];
  for (int j = 1; j < lists; ++j) {
    float s    = score[b + j * KC];
    uint32_t p = pos[b + j * KC];
    if (s < best || (s == best && p < bp)) { best = s; bp = p; }
  }
  labels[i] = bp;
  if (out_scores) out_scores[i] = best;
}

// ---- probe bucketing -----------------------------------------------------------------------
// Pairs are bucketed by (list, near/far bin): bin 0 holds a query's nearest `near_ranks` probes.  Inside a list the near
// pairs come first, so each list's FIRST 128-pair work item holds the lowest probe ranks; all first items are scheduled
// before any other item.  The per-query pruning bound (tc_bound) is therefore already tight — every query's closest
// lists have been scanned — when the bulk of the work starts, and the epilogue's insert path is rarely taken.
// Probes of empty lists (e.g. lists owned by another shard) are dropped here.
__global__ void count_probes_kernel(const uint32_t* __restrict__ probes, int64_t total, int n_probes, int probe_ld, int near_ranks,
                                    const int64_t* __restrict__ list_offsets, uint32_t* __restrict__ counts)
{
  int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (t >= total) return;
  uint32_t l = probes[(t / n_probes) * probe_ld + t % n_probes];
  if (l != 0xffffffffu && list_offsets[l + 1] > list_offsets[l])
    atomicAdd(&counts[2 * l + (static_cast<int>(t % n_probes) < near_ranks ? 0 : 1)], 1u);
}

// single CTA: exclusive scans over lists of (a) pair counts, (b) "has a first item", (c) further items ceil(cnt/group) - 1;
// per 1024-list chunk, warp-shuffle scans and one scan of the 32 warp totals
__global__ void __launch_bounds__(1024) scan_lists_kernel(const uint32_t* __restrict__ counts, int64_t n_lists, uint32_t group,
                                                           uint32_t* __restrict__ pair_off, uint32_t* __restrict__ first_off,
                                                           uint32_t* __restrict__ rest_off, int* __restrict__ n_items,
                                                           uint32_t* __restrict__ cursor)
{
  __shared__ uint3 w_tot[32];
  __shared__ uint32_t run_pairs, run_first, run_rest;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) { run_pairs = 0; run_first = 0; run_rest = 0; }
  __syncthreads();
  for (int64_t base = 0; base < n_lists; base += 1024) {
    int64_t l   = base + threadIdx.x;
    uint32_t c0 = l < n_lists ? counts[2 * l] : 0;
    uint32_t c  = c0 + (l < n_lists ? counts[2 * l + 1] : 0);
    uint32_t f  = c > 0 ? 1u : 0u;
    uint32_t g  = c > 0 ? (c + group - 1) / group - 1 : 0u;
    uint32_t sp = c, sf = f, sg = g;  // inclusive scans within the warp
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t a = __shfl_up_sync(0xffffffffu, sp, o), b = __shfl_up_sync(0xffffffffu, sf, o),
                     d = __shfl_up_sync(0xffffffffu, sg, o);
      if (lane >= o) { sp += a; sf += b; sg += d; }
    }
    if (lane == 31) w_tot[warp] = make_uint3(sp, sf, sg);
    __syncthreads();
    if (warp == 0) {  // exclusive scan of the warp totals
      const uint3 t = w_tot[lane];
      uint32_t ip = t.x, iff = t.y, ig = t.z;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t a = __shfl_up_sync(0xffffffffu, ip, o), b = __shfl_up_sync(0xffffffffu, iff, o),
                       d = __shfl_up_sync(0xffffffffu, ig, o);
        if (lane >= o) { ip += a; iff += b; ig += d; }
      }
      w_tot[lane] = make_uint3(ip - t.x, iff - t.y, ig - t.z);
    }
    __syncthreads();
    const uint3 w = w_tot[warp];
    sp += w.x; sf += w.y; sg += w.z;  // inclusive over the chunk
    if (l < n_lists) {
      pair_off[2 * l]     = run_pairs + sp - c;
      pair_off[2 * l + 1] = run_pairs + sp - c + c0;
      first_off[l]        = run_first + sf - f;
      rest_off[l]         = run_rest + sg - g;
      cursor[2 * l]       = 0;
      cursor[2 * l + 1]   = 0;
    }
    __syncthreads();
    if (threadIdx.x == 1023) { run_pairs += sp; run_first += sf; run_rest += sg; }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    n_items[0] = static_cast<int>(run_first + run_rest);
    n_items[1] = static_cast<int>(run_pairs);
    n_items[2] = static_cast<int>(run_first);
  }
}

__global__ void scatter_probes_kernel(const uint32_t* __restrict__ probes, int64_t total, int n_probes, int probe_ld, int near_ranks,
                                      const int64_t* __restrict__ list_offsets, const uint32_t* __restrict__ pair_off,
                                      uint32_t* __restrict__ cursor, uint32_t* __restrict__ slot_of,
                                      uint32_t* __restrict__ pair_query, uint32_t* __restrict__ pair_list)
{
  int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (t >= total) return;
  uint32_t l = probes[(t / n_probes) * probe_ld + t % n_probes];
  if (l == 0xffffffffu || list_offsets[l + 1] <= list_offsets[l]) { slot_of[t] = 0xffffffffu; return; }
  const uint32_t b = 2 * l + (static_cast<int>(t % n_probes) < near_ranks ? 0 : 1);
  uint32_t slot    = pair_off[b] + atomicAdd(&cursor[b], 1u);
  slot_of[t]       = slot;
  pair_query[slot] = static_cast<uint32_t>(t / n_probes);
  pair_list[slot]  = l;
}

__global__ void make_list_items_kernel(const uint32_t* __restrict__ counts, const uint32_t* __restrict__ pair_off,
                                       const uint32_t* __restrict__ first_off, const uint32_t* __restrict__ rest_off,
                                       const int* __restrict__ n_items, const int64_t* __restrict__ list_offsets,
                                       int64_t n_lists, int KC, uint32_t max_tiles, uint32_t group, tc_item* __restrict__ items)
{
  int64_t l = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (l >= n_lists) return;
  uint32_t c = counts[2 * l] + counts[2 * l + 1];
  if (c == 0) return;
  const uint32_t b_row0  = static_cast<uint32_t>(list_offsets[l]);
  const uint32_t n_tiles = min(max_tiles, static_cast<uint32_t>((list_offsets[l + 1] - list_offsets[l]) / 128));
  const uint32_t n_first = static_cast<uint32_t>(n_items[2]);
  uint32_t g = (c + group - 1) / group;
  for (uint32_t j = 0; j < g; ++j) {
    tc_item it;
    it.a_row0     = pair_off[2 * l] + j * group;
    it.b_row0     = b_row0;
    it.n_tiles    = n_tiles;
    it.valid_rows = min(group, c - j * group);
    it.out_off    = static_cast<uint64_t>(it.a_row0) * KC;
    items[j == 0 ? first_off[l] : n_first + rest_off[l] + (j - 1)] = it;
  }
}

// per pair: r = q[query] - c[list] (L2) or q[query] (IP) as bf16 A rows; add[slot] = |r|^2 (L2) or -(q . c) (IP: the B rows
// hold residuals, so the centre's part of q . x is the pair's).  Cosine (q and c already unit) adds 1 to the offset, so that
// every reader of `add` sees cosine distances 1 - q.c - q.(x - c).
__global__ void pair_rows_kernel(const float* __restrict__ q, const float* __restrict__ centers,
                                 const uint32_t* __restrict__ pair_query, const uint32_t* __restrict__ pair_list,
                                 const int* __restrict__ n_live, int64_t rows_total, int dim, int Kp, bool ip,
                                 __nv_bfloat16* __restrict__ a_hi,
                                 __nv_bfloat16* __restrict__ a_lo, float* __restrict__ add, bool cosine)
{
  int64_t r = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
  int lane  = threadIdx.x & 31;
  if (r >= rows_total) return;
  float nrm = 0.f;
  const bool live = r < *n_live;
  const float* qr = live ? q + static_cast<int64_t>(pair_query[r]) * dim : nullptr;
  const float* cr = live ? centers + static_cast<int64_t>(pair_list[r]) * dim : nullptr;
  for (int j = lane; j < Kp; j += 32) {
    float v = 0.f;
    if (live && j < dim) v = ip ? qr[j] : qr[j] - cr[j];
    __nv_bfloat16 h = __float2bfloat16_rn(v);
    a_hi[r * Kp + j] = h;
    if (a_lo) a_lo[r * Kp + j] = __float2bfloat16_rn(v - __bfloat162float(h));
    nrm = ip ? ((live && j < dim) ? fmaf(-qr[j], cr[j], nrm) : nrm) : fmaf(v, v, nrm);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) nrm += __shfl_xor_sync(0xffffffffu, nrm, o);
  if (lane == 0 && live) add[r] = cosine ? nrm + 1.0f : nrm;
}

// out[q, p*KCW + c] = add[slot] + scale * s   (per-query concatenation of its probes' candidates; `empty` where there is none)
__global__ void gather_cands_kernel(const float* __restrict__ cs, const uint32_t* __restrict__ cp,
                                    const uint32_t* __restrict__ slot_of, const float* __restrict__ add, float scale, float empty,
                                    int64_t total, int KCW, float* __restrict__ out_score, uint32_t* __restrict__ out_pos,
                                    int L, float* __restrict__ last)
{
  int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (t >= total) return;
  int64_t pair  = t / KCW;
  int c         = static_cast<int>(t % KCW);
  uint32_t slot = slot_of[pair];
  float s       = empty;
  uint32_t p    = 0xffffffffu;
  if (slot != 0xffffffffu) {
    // independent loads: the score is read before the position is known to be live
    const int64_t e = static_cast<int64_t>(slot) * KCW + c;
    p               = cp[e];
    const float v   = cs[e];
    const float a   = add ? add[slot] : 0.f;
    if (p != 0xffffffffu) s = a + scale * v;
  }
  out_score[t] = s;
  out_pos[t]   = p;
  if (last != nullptr && c % L == L - 1) last[t / L] = s;
}

// ---- k > 64: dense per-pair score segments.  Live slot i, a pair of list l, owns scores[seg_off[i] .. + padded size of l):
// its list's rows in list order.  seg_len[i] is the list's real size (the padding rows at its end are never selected) and
// seg_base[i] its first index row, so column c of the segment is index row seg_base[i] + c.  Slots past the live count get
// seg_len 0.  Slots are few (nq * n_probes): one CTA scans them, each thread a contiguous chunk.
__global__ void __launch_bounds__(1024) pair_segments_kernel(const uint32_t* __restrict__ pair_list, const int* __restrict__ n_live,
                                                             int64_t n_pairs, const int64_t* __restrict__ list_offsets,
                                                             const uint32_t* __restrict__ list_sizes, int64_t* __restrict__ seg_off,
                                                             uint32_t* __restrict__ seg_len, uint32_t* __restrict__ seg_base)
{
  __shared__ int64_t part[1024];
  const int tid      = threadIdx.x;
  const int64_t live = *n_live;
  const int64_t per  = (n_pairs + 1023) / 1024;
  const int64_t b = min(n_pairs, tid * per), e = min(n_pairs, b + per);
  int64_t sum = 0;
  for (int64_t i = b; i < min(e, live); ++i) sum += list_offsets[pair_list[i] + 1] - list_offsets[pair_list[i]];
  part[tid] = sum;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {
    const int64_t v = tid >= o ? part[tid - o] : 0;
    __syncthreads();
    part[tid] += v;
    __syncthreads();
  }
  int64_t run = part[tid] - sum;
  for (int64_t i = b; i < e; ++i) {
    seg_off[i] = run;
    if (i < live) {
      const uint32_t l = pair_list[i];
      seg_len[i]       = list_sizes[l];
      seg_base[i]      = static_cast<uint32_t>(list_offsets[l]);
      run += list_offsets[l + 1] - list_offsets[l];
    } else {
      seg_len[i]  = 0;
      seg_base[i] = 0;
    }
  }
}

// a store scan writes an item's pairs from the segment of its first slot on
__global__ void item_segments_kernel(tc_item* __restrict__ items, const int* __restrict__ n_items, const int64_t* __restrict__ seg_off)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < *n_items) items[i].out_off = static_cast<uint64_t>(seg_off[items[i].a_row0]);
}

// ---- per-query merge of the probes' candidate lists ------------------------------------------
// One CTA per query.  The scan left, for every (query, probe) pair, KCW candidates (score, position) and — shared by all
// pairs of the query — an upper bound B on the query's k-th best value (tc_bound).  Every candidate that can be among the k
// best satisfies value <= B, and at least k candidates do (the list that published B), so: filter by B into shared memory
// (typically a few dozen survivors out of n_probes * KCW), sort those, emit the k best.  Replaces a gather of all
// candidates into a [nq, n_probes * KCW] matrix followed by a radix select over it.
__device__ __forceinline__ uint32_t order_key(float f)
{
  uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float order_key_inv(uint32_t k)
{
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

constexpr int kMergeCap = 1024;

// kMergeThreads: 128 while a query has at most 2048 candidates (a filter trip takes 4 x 128 of them: the flagship's 48 x 32
// take three trips, and twice the CTAs fit an SM; 0.09 ms per 10k batch against 0.11 ms with 256), else 256 (more loads in
// flight per query: at 192 probes x 64 candidates the search took 0.7 ms longer per 10k batch with 128)
template <int kMergeThreads>
__global__ void __launch_bounds__(kMergeThreads)
merge_pairs_kernel(const float* __restrict__ cs, const uint32_t* __restrict__ cp, const uint32_t* __restrict__ slot_of,
                   const float* __restrict__ add, float scale, const int* __restrict__ bound_keys, int n_probes, int KCW,
                   int kcw_shift, int k, float* __restrict__ out_val, uint32_t* __restrict__ out_pos)
{
  __shared__ unsigned long long surv[kMergeCap];  // (order key << 32 | position)
  __shared__ unsigned long long red[kMergeThreads / 32];
  __shared__ int count;
  const int64_t q = blockIdx.x;
  if (threadIdx.x == 0) count = 0;
  __syncthreads();
  float bnd = INFINITY;
  if (bound_keys) {
    const int kb = bound_keys[q];
    bnd          = __int_as_float(kb >= 0 ? kb : kb ^ 0x7fffffff);
  }
  const int total          = n_probes * KCW;
  const uint32_t* my_slots = slot_of + q * n_probes;
  auto value_of = [&](int e, uint32_t& pos) -> float {  // candidate e of this query (FLT_MAX / 0xffffffff when empty)
    const int p         = e / KCW;
    const int c         = e - p * KCW;
    const uint32_t slot = my_slots[p];
    pos                 = 0xffffffffu;
    if (slot == 0xffffffffu) return FLT_MAX;
    pos = cp[static_cast<int64_t>(slot) * KCW + c];
    if (pos == 0xffffffffu) return FLT_MAX;
    return __fmaf_rn(scale, cs[static_cast<int64_t>(slot) * KCW + c], add ? add[slot] : 0.f);
  };
  // filter: four independent candidates per thread and trip keep the dependent slot -> position/score loads overlapped
  for (int e0 = threadIdx.x; e0 < total; e0 += 4 * kMergeThreads) {
    uint32_t slot[4], pos[4];
    float sc[4], ad[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int e = e0 + u * kMergeThreads;
      slot[u]     = e < total ? my_slots[kcw_shift >= 0 ? e >> kcw_shift : e / KCW] : 0xffffffffu;
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int e = e0 + u * kMergeThreads;
      const int c = kcw_shift >= 0 ? e & (KCW - 1) : e % KCW;
      pos[u] = 0xffffffffu; sc[u] = 0.f; ad[u] = 0.f;
      if (slot[u] != 0xffffffffu) {
        pos[u] = cp[static_cast<int64_t>(slot[u]) * KCW + c];
        sc[u]  = cs[static_cast<int64_t>(slot[u]) * KCW + c];
        ad[u]  = add ? add[slot[u]] : 0.f;
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (pos[u] == 0xffffffffu) continue;
      const float v = __fmaf_rn(scale, sc[u], ad[u]);
      if (v <= bnd) {
        const int at = atomicAdd(&count, 1);
        if (at < kMergeCap) surv[at] = (static_cast<unsigned long long>(order_key(v)) << 32) | pos[u];
      }
    }
  }
  __syncthreads();
  const int n = count;
  if (n <= kMergeCap) {
    int n2 = 1;
    while (n2 < n) n2 <<= 1;
    for (int i = n + threadIdx.x; i < n2; i += blockDim.x) surv[i] = ~0ull;
    __syncthreads();
    for (int size = 2; size <= n2; size <<= 1) {
      for (int stride = size >> 1; stride > 0; stride >>= 1) {
        for (int i = threadIdx.x; i < n2 / 2; i += blockDim.x) {
          const int lo = ((i & ~(stride - 1)) << 1) | (i & (stride - 1));  // (stride is a power of two)
          const int hi = lo + stride;
          const bool up = ((lo & size) == 0);
          const unsigned long long a = surv[lo], b = surv[hi];
          if ((a > b) == up) { surv[lo] = b; surv[hi] = a; }
        }
        __syncthreads();
      }
    }
    for (int j = threadIdx.x; j < k; j += blockDim.x) {
      float v      = FLT_MAX;
      uint32_t pos = 0xffffffffu;
      if (j < n) {
        v   = order_key_inv(static_cast<uint32_t>(surv[j] >> 32));
        pos = static_cast<uint32_t>(surv[j] & 0xffffffffu);
      }
      out_val[q * k + j] = v;
      out_pos[q * k + j] = pos;
    }
    return;
  }
  // More survivors than the buffer holds (no usable bound, or massive ties at it): k rounds of "smallest key above the
  // previous one" over all candidates.  Slow, but only for the rare query that gets here.
  unsigned long long last = 0;
  bool first = true;
  for (int j = 0; j < k; ++j) {
    unsigned long long best = ~0ull;
    for (int e = threadIdx.x; e < total; e += blockDim.x) {
      uint32_t pos;
      const float v = value_of(e, pos);
      if (pos == 0xffffffffu) continue;
      const unsigned long long key = (static_cast<unsigned long long>(order_key(v)) << 32) | pos;
      if ((first || key > last) && key < best) best = key;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
      best = other < best ? other : best;
    }
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = best;
    __syncthreads();
    best = red[0];
    for (int w = 1; w < kMergeThreads / 32; ++w) best = red[w] < best ? red[w] : best;
    __syncthreads();
    if (threadIdx.x == 0) {
      const bool have    = best != ~0ull;
      out_val[q * k + j] = have ? order_key_inv(static_cast<uint32_t>(best >> 32)) : FLT_MAX;
      out_pos[q * k + j] = have ? static_cast<uint32_t>(best & 0xffffffffu) : 0xffffffffu;
    }
    if (best == ~0ull) {  // exhausted: fill the rest
      for (int r = j + 1 + threadIdx.x; r < k; r += blockDim.x) { out_val[q * k + r] = FLT_MAX; out_pos[q * k + r] = 0xffffffffu; }
      return;
    }
    last  = best;
    first = false;
  }
}

// ---- k-means ---------------------------------------------------------------------------------
__global__ void strided_init_kernel(const float* __restrict__ x, int64_t n, int d, int k, float* __restrict__ centers)
{
  int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (t >= static_cast<int64_t>(k) * d) return;
  int64_t c   = t / d;
  int64_t row = (c * n) / k;  // evenly spaced rows
  centers[t]  = x[row * d + (t % d)];
}

__global__ void abs_max_kernel(const float* __restrict__ x, int64_t count, uint32_t* __restrict__ out)
{
  uint32_t m = 0;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < count; i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    m = max(m, __float_as_uint(fabsf(x[i])));  // non-negative floats order like their bit patterns
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(out, m);
}

__global__ void accumulate_kernel(const float* __restrict__ x, int64_t n, int d, const uint32_t* __restrict__ labels,
                                  const uint32_t* __restrict__ x_max_bits, unsigned long long* __restrict__ sums,
                                  unsigned long long* __restrict__ counts)
{
  // one warp per row; lanes stride over d
  int64_t row = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
  int lane    = threadIdx.x & 31;
  if (row >= n) return;
  const double scale = fixed_scale(*x_max_bits, n);
  uint32_t l = labels[row];
  for (int c = lane; c < d; c += 32) fixed_add(&sums[static_cast<int64_t>(l) * d + c], x[row * d + c], scale);
  if (lane == 0) atomicAdd(&counts[l], 1ull);
}

__global__ void finalize_centers_kernel(const unsigned long long* __restrict__ sums, const unsigned long long* __restrict__ counts,
                                        const uint32_t* __restrict__ x_max_bits, int64_t n, int k, int d, float* __restrict__ centers,
                                        float* __restrict__ counts_out)
{
  int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (t >= static_cast<int64_t>(k) * d) return;
  const unsigned long long c = counts[t / d];
  if (t % d == 0) counts_out[t / d] = static_cast<float>(c);
  if (c > 0) centers[t] = static_cast<float>(fixed_value(sums[t], fixed_scale(*x_max_bits, n)) / static_cast<double>(c));
}


// one thread per cluster: small clusters jump onto a member of a large cluster
__global__ void reseed_small_kernel(const float* __restrict__ x, int64_t n, int d, const uint32_t* __restrict__ labels,
                                    const float* __restrict__ counts, int k, float avg, int iter, float* __restrict__ centers,
                                    int* __restrict__ n_reseeded)
{
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= k) return;
  if (counts[c] >= 0.25f * avg) return;
  for (int tries = 0; tries < 64; ++tries) {
    uint64_t h  = mix64((static_cast<uint64_t>(iter) << 40) ^ (static_cast<uint64_t>(c) << 8) ^ tries);
    int64_t row = static_cast<int64_t>(h % static_cast<uint64_t>(n));
    if (counts[labels[row]] >= avg) {
      // move most of the way to the donor point; keep a little of the donor's centre to break symmetry
      const float* donor_c = centers + static_cast<int64_t>(labels[row]) * d;
      for (int j = 0; j < d; ++j) centers[static_cast<int64_t>(c) * d + j] = 0.75f * x[row * d + j] + 0.25f * donor_c[j];
      atomicAdd(n_reseeded, 1);
      return;
    }
  }
}

// The k-means cost in a fixed order: per-warp partials of a fixed grid, then one warp adds them up (a double atomic would round
// differently depending on arrival order, and `tol` would stop training after a different number of iterations).  A row's
// term is w_i * dist_i with dist_i = |x_i - c_{l_i}|^2 summed as the oracle's sqdiff (fmaf, ascending components), or its root;
// w_i is 1 without weights and weights[i] * n / *w_sum with a weight sum.  x == null: the terms are the weights alone.
constexpr int kCostBlocks = 256, kCostThreads = 256, kCostParts = kCostBlocks * kCostThreads / 32;
__global__ void __launch_bounds__(kCostThreads) cost_parts_kernel(const float* __restrict__ x, int64_t n, int d,
                                                                  const float* __restrict__ centers, const uint32_t* __restrict__ labels,
                                                                  const float* __restrict__ w, const double* __restrict__ w_sum,
                                                                  bool sqrt_dist, double* __restrict__ parts)
{
  const double scale = w_sum ? static_cast<double>(n) / *w_sum : 1.0;
  const bool vec4    = x != nullptr && exact_vec4(x, d, centers, d, d);
  double acc         = 0;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    if (x == nullptr) { acc += static_cast<double>(w[i]); continue; }
    const float dist = exact_accumulate(x + i * d, centers + static_cast<int64_t>(labels[i]) * d, d, vec4, L2Unexpanded);
    double t         = sqrt_dist ? sqrt(static_cast<double>(dist)) : static_cast<double>(dist);
    if (w) t *= static_cast<double>(w[i]) * scale;
    acc += t;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) parts[(blockIdx.x * blockDim.x + threadIdx.x) >> 5] = acc;
}

__global__ void sum_parts_kernel(const double* __restrict__ parts, double* __restrict__ out)
{
  double acc = 0;
  for (int i = threadIdx.x; i < kCostParts; i += 32) acc += parts[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (threadIdx.x == 0) *out = acc;
}

// one warp per row of dist [n, k]: the smallest entry, ties to the smaller column (the oracle's first minimum)
__global__ void row_argmin_kernel(const float* __restrict__ dist, int64_t n, int k, int64_t* __restrict__ idx, float* __restrict__ out)
{
  const int64_t r = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
  const int lane  = threadIdx.x & 31;
  if (r >= n) return;
  float best = INFINITY;
  int bj     = k;
  for (int j = lane; j < k; j += 32) {
    const float v = dist[r * k + j];
    if (v < best) { best = v; bj = j; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float v = __shfl_xor_sync(0xffffffffu, best, o);
    const int j   = __shfl_xor_sync(0xffffffffu, bj, o);
    if (v < best || (v == best && j < bj)) { best = v; bj = j; }
  }
  if (lane == 0) { idx[r] = bj < k ? bj : 0; out[r] = best; }
}

// a row whose scan kept no candidate at all (every score NaN or infinite) has no re-scored best: certify_candidates sees no
// row outside the empty list, so it is flagged here and takes the exact path
__global__ void flag_empty_rows_kernel(const int64_t* __restrict__ best_id, int64_t n, int* __restrict__ flags)
{
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i < n && best_id[i] < 0 && !flags[i]) { flags[i] = 1; atomicAdd(flags + n, 1); }
}

__global__ void i64_to_u32_kernel(const int64_t* __restrict__ in, uint32_t* __restrict__ out, int64_t n)
{
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i < n) out[i] = static_cast<uint32_t>(in[i]);
}

}  // namespace

void tc_rows::build(cudaStream_t s, const float* x, int64_t n_, int d_, const float* xn, bool with_lo, const float* row_scale)
{
  n = n_; d = d_;
  Kp       = tc_pad_k(d);
  rows_pad = tc_pad_rows(std::max<int64_t>(n, 1));
  hi.alloc(static_cast<size_t>(rows_pad) * Kp);
  if (with_lo) lo.alloc(static_cast<size_t>(rows_pad) * Kp); else lo.release();
  hx.alloc(static_cast<size_t>(rows_pad) * 16);
  tc_split_planes(s, x, n, d, d, Kp, hi.data(), with_lo ? lo.data() : nullptr, rows_pad, row_scale);
  tc_half_norms(s, xn, n, rows_pad, hx.data());
}

void tc_rows_tmp::build(cudaStream_t s, const float* x, int64_t n_, int d_, bool with_lo, int64_t extra_pad_rows,
                        const float* row_scale)
{
  n = n_; d = d_;
  Kp       = tc_pad_k(d);
  rows_pad = tc_pad_rows(std::max<int64_t>(n, 1)) + extra_pad_rows;
  hi.alloc(static_cast<size_t>(rows_pad) * Kp, s);
  if (with_lo) lo.alloc(static_cast<size_t>(rows_pad) * Kp, s);
  tc_split_planes(s, x, n, d, d, Kp, hi.data(), with_lo ? lo.data() : nullptr, rows_pad, row_scale);
}

// The dense coarse search of the queries in rows [0, n) of the planes a_hi / a_lo: every score, then select_k.  With
// n_rows_dev the planes' rows are sized for n queries and the count is the device's: launches past it exit at once.
static void coarse_select_dense(resources* res, const __nv_bfloat16* a_hi, const __nv_bfloat16* a_lo, int64_t n, int64_t a_rows_pad,
                                const tc_rows& centers, int n_probes, uint32_t* probes, float* probe_scores,
                                const int* n_rows_dev = nullptr, const int* n_tiles_dev = nullptr)
{
  auto s               = res->stream;
  const int m_tiles    = static_cast<int>(tc_pad_rows(n) / 128);
  const int64_t ld     = centers.rows_pad;
  dbuf<tc_item> items(static_cast<size_t>(m_tiles), s);
  tc_split_items(s, items.data(), m_tiles, 1, n, static_cast<uint32_t>(ld / 128), ld);
  dbuf<float> scores(static_cast<size_t>(tc_pad_rows(n)) * ld, s);
  const bool three = a_lo != nullptr && centers.lo.data() != nullptr;
  tc_scan_topk(s, res->device, a_hi, a_lo, a_rows_pad, centers.hi.data(), centers.lo.data(), centers.rows_pad, centers.Kp,
               centers.hx.data(), items.data(), m_tiles, n_tiles_dev, 0, three ? 3 : 1, scores.data(), nullptr, ld);
  select_k(s, scores.data(), nullptr, IDX_NONE, n, centers.n, ld, n_probes, probe_scores, probes, IDX_U32, true, n_rows_dev);
}

// Fused coarse search (large n_lists): instead of writing the dense [nq, n_lists] score block (655 MB at 10k x 16384) and
// selecting from it, the scan keeps KC candidates per (query, centre range, column half) in its epilogue — (query tile, centre
// range) items also give the SMs ~2 waves of work where one item per query tile gave 79 CTAs — and a small merge ranks
// the 2 * splits * KC candidates per query.  Exact (same scores, same (score, id) order as the dense select) for every query
// whose merge certificate holds; the queries it flags are packed and take the dense path, with launches sized for a fully
// flagged batch (a row's scores do not depend on where it sits in the planes, so their probes are the dense path's too).
// Nothing waits for the host: the whole search can be enqueued ahead of the device, or captured in a CUDA graph.  Returns
// false when the shape does not suit the fused scan.
static bool coarse_select_fused(resources* res, const tc_rows_tmp& q, const tc_rows& centers, int n_probes, uint32_t* probes,
                                float* probe_scores)
{
  const char* env = getenv("CUVS_B200_COARSE_FUSED");  // read per call (A/B inside one process): "0" = dense path
  if (env != nullptr && env[0] == '0') return false;
  // Lists of 16: the epilogue's insertions, not the tensor cores, set the scan's pace, and a list of 16 costs about half
  // of one of 32 (flagship shape, 10k queries x 8192 centres: 0.31 ms against 0.54 ms, the same probes).  More lists make
  // up the candidates: W >= 4 n_probes below.
  const int KC = 16;
  if (n_probes > 64 || centers.n < 4096 || centers.n > kCoarseMaxCenters) return false;
  auto s               = res->stream;
  const int64_t nq_pad = tc_pad_rows(q.n);
  const int m_tiles    = static_cast<int>(nq_pad / 128);
  const int64_t b_tiles = centers.rows_pad / 128;
  const int sms        = res->sm_count ? res->sm_count : 132;
  const int KCW = KC * kTcListsPerItem;
  // enough items for ~2 waves of CTAs, and enough lists that the n_probes best are spread thin (>= 4 n_probes candidates:
  // with only n_probes candidates the certificate could never hold and every batch would pay for both paths)
  int splits = std::max((2 * sms + m_tiles - 1) / m_tiles, (4 * n_probes + KCW - 1) / KCW);
  splits     = static_cast<int>(std::min<int64_t>(splits, std::min<int64_t>(16, b_tiles / 4)));
  splits     = std::max(splits, 1);
  const int W   = splits * KCW;
  if (W > kCoarseMaxW || W < 4 * n_probes) return false;
  const int n_items = m_tiles * splits;
  dbuf<tc_item> items(static_cast<size_t>(n_items), s);
  tc_split_items(s, items.data(), m_tiles, splits, q.n, static_cast<uint32_t>(b_tiles), KCW);  // (centre range, query tile) items
  dbuf<float> cs(static_cast<size_t>(nq_pad) * W, s);
  dbuf<uint32_t> cp(static_cast<size_t>(nq_pad) * W, s);
  dbuf<int> bkeys(static_cast<size_t>(nq_pad) + 3, s);
  B2_CUDA(cudaMemsetAsync(bkeys.data(), tc_bound_init_byte, sizeof(int) * nq_pad, s));
  int* n_flagged = bkeys.data() + nq_pad;  // [0] flagged queries, [1] [2] a fallback pass's tiles and queries
  B2_CUDA(cudaMemsetAsync(n_flagged, 0, sizeof(int), s));
  dbuf<uint32_t> flagged(static_cast<size_t>(q.n), s);
  tc_bound bnd;
  bnd.keys = bkeys.data();
  bnd.kth  = 0;  // lists prune at, and publish, their last (KC-th) entry: that is what the merge's certificate reasons about
  const bool three = q.lo.data() != nullptr && centers.lo.data() != nullptr;
  tc_scan_topk(s, res->device, q.hi.data(), q.lo.data(), q.rows_pad, centers.hi.data(), centers.lo.data(), centers.rows_pad,
               q.Kp, centers.hx.data(), items.data(), n_items, nullptr, KC, three ? 3 : 1, cs.data(), cp.data(), W, &bnd);
  count_launch();
  {
    const unsigned grid = static_cast<unsigned>(blocks_for(q.n * 32, kCoarseMergeThreads));
#define B2_CM(E_) coarse_merge_kernel<E_><<<grid, kCoarseMergeThreads, 0, s>>>(cs.data(), cp.data(), q.n, W, KC, n_probes, probes, probe_scores, n_flagged, flagged.data())
    if (W <= 64) B2_CM(2);
    else if (W <= 128) B2_CM(4);
    else if (W <= 256) B2_CM(8);
    else B2_CM(16);
#undef B2_CM
  }
  B2_CUDA(cudaGetLastError());
  cs.release();
  cp.release();
  // the flagged queries, in passes: packed planes, the dense scan + select, their probes scattered over the fused ones.  A
  // pass's dense scores stay within 256 MiB; the flagship batch (10k queries, 8192 centres) takes two passes, and each
  // pass past the flagged count costs four near-empty launches.
  const int64_t pass_rows = std::max<int64_t>(kTcTile, std::min<int64_t>(nq_pad, ((int64_t(1) << 26) / centers.rows_pad) / kTcTile * kTcTile));
  dbuf<__nv_bfloat16> f_hi(static_cast<size_t>(pass_rows) * q.Kp, s), f_lo;
  if (three) f_lo.alloc(static_cast<size_t>(pass_rows) * q.Kp, s);
  dbuf<uint32_t> f_probes(static_cast<size_t>(pass_rows) * n_probes, s);
  dbuf<float> f_scores(static_cast<size_t>(pass_rows) * n_probes, s);
  const int64_t total = pass_rows * n_probes;
  for (int64_t first = 0; first < q.n; first += pass_rows) {
    count_launch();
    gather_flagged_rows_kernel<<<blocks_for(pass_rows * 32, 256), 256, 0, s>>>(
      reinterpret_cast<const uint4*>(q.hi.data()), three ? reinterpret_cast<const uint4*>(q.lo.data()) : nullptr, q.Kp / 8,
      flagged.data(), n_flagged, first, pass_rows, reinterpret_cast<uint4*>(f_hi.data()),
      three ? reinterpret_cast<uint4*>(f_lo.data()) : nullptr);
    B2_CUDA(cudaGetLastError());
    coarse_select_dense(res, f_hi.data(), f_lo.data(), pass_rows, pass_rows, centers, n_probes, f_probes.data(), f_scores.data(),
                        n_flagged + 2, n_flagged + 1);
    count_launch();
    scatter_flagged_probes_kernel<<<blocks_for(total, 256), 256, 0, s>>>(flagged.data(), n_flagged, first, n_probes, total,
                                                                          f_probes.data(), f_scores.data(), probes, probe_scores);
    B2_CUDA(cudaGetLastError());
  }
  return true;
}

void coarse_select(resources* res, const tc_rows_tmp& q, const tc_rows& centers, int n_probes, uint32_t* probes,
                   float* probe_scores)
{
  auto s = res->stream;
  if (q.n == 0) return;
  B2_EXPECTS(q.Kp == centers.Kp, "coarse_select: dimension mismatch");
  dbuf<float> tmp_scores;
  if (!probe_scores) { tmp_scores.alloc(static_cast<size_t>(q.n) * n_probes, s); probe_scores = tmp_scores.data(); }
  if (coarse_select_fused(res, q, centers, n_probes, probes, probe_scores)) return;
  coarse_select_dense(res, q.hi.data(), q.lo.data(), q.n, q.rows_pad, centers, n_probes, probes, probe_scores);
}

void assign_nearest(resources* res, const __nv_bfloat16* x_hi, const __nv_bfloat16* x_lo, int64_t n, int64_t x_rows_pad,
                    int Kp, const tc_rows& centers, uint32_t* labels, float* scores)
{
  auto s = res->stream;
  if (n == 0) return;
  B2_EXPECTS(Kp == centers.Kp, "assign_nearest: dimension mismatch");
  const int KC         = 16;
  const int KCW        = KC * kTcListsPerItem;
  const int64_t chunk  = int64_t(1) << 20;  // rows per launch: bounds the (score,pos) scratch to 256 MiB
  const bool three     = x_lo != nullptr && centers.lo.data() != nullptr;
  dbuf<float> cs(static_cast<size_t>(std::min(chunk, tc_pad_rows(n))) * KCW, s);
  dbuf<uint32_t> cp(static_cast<size_t>(std::min(chunk, tc_pad_rows(n))) * KCW, s);
  dbuf<tc_item> items(static_cast<size_t>(std::min(chunk, tc_pad_rows(n)) / 128), s);
  for (int64_t r0 = 0; r0 < n; r0 += chunk) {
    const int64_t rows = std::min(chunk, n - r0);
    const int m_tiles  = static_cast<int>(tc_pad_rows(rows) / 128);
    tc_split_items(s, items.data(), m_tiles, 1, rows, static_cast<uint32_t>(centers.rows_pad / 128), KCW);
    tc_scan_topk(s, res->device, x_hi + r0 * Kp, x_lo ? x_lo + r0 * Kp : nullptr, x_rows_pad - r0, centers.hi.data(),
                 centers.lo.data(), centers.rows_pad, Kp, centers.hx.data(), items.data(), m_tiles, nullptr, KC,
                 three ? 3 : 1, cs.data(), cp.data(), KCW);
    count_launch();
    first_of_rows_kernel<<<blocks_for(rows, 256), 256, 0, s>>>(cp.data(), cs.data(), rows, KC, kTcListsPerItem, labels + r0,
                                                               scores ? scores + r0 : nullptr);
    B2_CUDA(cudaGetLastError());
  }
}

void assign_exact(resources* res, const float* x, const float* xn, const tc_rows_tmp& xp, const float* centers, const float* cn,
                  const tc_rows& cp, uint32_t* labels)
{
  auto s          = res->stream;
  const int64_t n = xp.n;
  const int d = xp.d, k = static_cast<int>(cp.n);
  if (n == 0) return;
  B2_EXPECTS(xp.Kp == cp.Kp, "assign_exact: dimension mismatch");
  // the certificate's budget (brute force's, DESIGN.md §3): A = 2 s + |x|^2 is within eps_rel (|x|^2 + max |c|^2) of the
  // exact distance (a non-finite max |c|^2 makes the budget infinite: every row then takes the exact path)
  approx_map am;
  am.sa = 2.f; am.sb = 1.f; am.eq = 1.f;
  const uint32_t cmax_bits = abs_max_host(s, cn, k);
  std::memcpy(&am.ec, &cmax_bits, sizeof(float));
  am.eps_rel = std::max(1.0f / 32768.0f, 1.0f / 65536.0f + static_cast<float>(xp.Kp) / 16777216.0f);
  const int KC        = 16;
  const int KCW       = KC * kTcListsPerItem;
  const int64_t chunk = int64_t(1) << 20;  // rows per launch: bounds the (score, pos) scratch to 256 MiB
  const int64_t rows0 = std::min(chunk, tc_pad_rows(n));
  dbuf<float> cs(static_cast<size_t>(rows0) * KCW, s), best(static_cast<size_t>(rows0), s), floor(static_cast<size_t>(rows0), s);
  dbuf<uint32_t> cpos(static_cast<size_t>(rows0) * KCW, s);
  dbuf<int64_t> best_id(static_cast<size_t>(rows0), s);
  dbuf<int> flags(static_cast<size_t>(rows0) + 1, s);
  dbuf<tc_item> items(static_cast<size_t>(rows0 / 128), s);
  // flagged rows per exact launch: their gathered rows and their distance tile each stay within 2^26 floats (256 MiB)
  const int64_t step = std::min<int64_t>(std::max<int64_t>(1, (int64_t(1) << 26) / std::max(k, d)), int64_t(64) * 65535);
  for (int64_t r0 = 0; r0 < n; r0 += chunk) {
    const int64_t rows = std::min(chunk, n - r0);
    const int m_tiles  = static_cast<int>(tc_pad_rows(rows) / 128);
    tc_split_items(s, items.data(), m_tiles, 1, rows, static_cast<uint32_t>(cp.rows_pad / 128), KCW);
    tc_scan_topk(s, res->device, xp.hi.data() + r0 * xp.Kp, xp.lo.data() + r0 * xp.Kp, xp.rows_pad - r0, cp.hi.data(), cp.lo.data(),
                 cp.rows_pad, xp.Kp, cp.hx.data(), items.data(), m_tiles, nullptr, KC, 3, cs.data(), cpos.data(), KCW);
    const float* xc  = x + r0 * d;
    const float* xnc = xn + r0;
    // oracle_kmeans_assign's arithmetic: expanded L2 clamped at 0, without the searches' self-neighbour rule
    rescore_topk(s, xc, rows, d, centers, d, d, xnc, cn, L2Expanded, cpos.data(), KCW, nullptr, 1, best_id.data(), best.data(), -1,
                 false);
    list_floors(s, cs.data(), rows, KCW, KC, floor.data());
    certify_candidates(s, cs.data(), cpos.data(), KCW, floor.data(), xnc, best.data(), 1, am, true, false, rows, flags.data());
    count_launch();
    flag_empty_rows_kernel<<<blocks_for(rows, 256), 256, 0, s>>>(best_id.data(), rows, flags.data());
    B2_CUDA(cudaGetLastError());
    // rows the certificate rejects: distances to every centre (exact_distance_tile, the re-score's arithmetic), first minimum
    rerun_flagged(s, flags.data(), rows, 1, best_id.data(), best.data(), [&](const int64_t* fr, int64_t nf, int64_t* fi, float* fd) {
      const int64_t m0 = std::min(step, nf);
      dbuf<float> fx(static_cast<size_t>(m0) * d, s), fxn(static_cast<size_t>(m0), s), tile(static_cast<size_t>(m0) * k, s);
      for (int64_t f0 = 0; f0 < nf; f0 += step) {
        const int64_t m = std::min(step, nf - f0);
        copy_rows(s, xc, fr + f0, fx.data(), nullptr, m, d);
        copy_rows(s, xnc, fr + f0, fxn.data(), nullptr, m, 1);
        exact_distance_tile(s, fx.data(), m, d, centers, k, d, d, fxn.data(), cn, L2Expanded, tile.data(), k, filter_view{}, 0, false);
        count_launch();
        row_argmin_kernel<<<blocks_for(m * 32, 256), 256, 0, s>>>(tile.data(), m, k, fi + f0, fd + f0);
        B2_CUDA(cudaGetLastError());
      }
    });
    count_launch();
    i64_to_u32_kernel<<<blocks_for(rows, 256), 256, 0, s>>>(best_id.data(), labels + r0, rows);
    B2_CUDA(cudaGetLastError());
  }
}

void kmeans_cost(cudaStream_t s, const float* x, int64_t n, int d, const float* centers, const uint32_t* labels, const float* weights,
                 bool normalize_weight, bool sqrt_dist, double* out)
{
  dbuf<double> parts(static_cast<size_t>(kCostParts), s), w_sum;
  if (weights != nullptr && normalize_weight) {
    w_sum.alloc(1, s);
    count_launch(2);
    cost_parts_kernel<<<kCostBlocks, kCostThreads, 0, s>>>(nullptr, n, 0, nullptr, nullptr, weights, nullptr, false, parts.data());
    sum_parts_kernel<<<1, 32, 0, s>>>(parts.data(), w_sum.data());
  }
  count_launch(2);
  cost_parts_kernel<<<kCostBlocks, kCostThreads, 0, s>>>(x, n, d, centers, labels, weights, w_sum.data(), sqrt_dist, parts.data());
  sum_parts_kernel<<<1, 32, 0, s>>>(parts.data(), out);
  B2_CUDA(cudaGetLastError());
}

void bucket_probes(resources* res, const uint32_t* probes, int64_t nq, int n_probes, int64_t n_lists,
                   const int64_t* list_offsets_dev, int KC, probe_buckets& out, int probe_ld, uint32_t max_tiles, int group)
{
  B2_EXPECTS(group >= 8 && group <= 128, "bucket_probes: group must be within [8, 128]");
  if (probe_ld <= 0) probe_ld = n_probes;
  auto s              = res->stream;
  const int64_t total = nq * n_probes;
  out.n_pairs         = total;
  out.max_items       = static_cast<int>(total / group + n_lists + 1);
  out.slot_of.alloc(static_cast<size_t>(total), s);
  out.pair_query.alloc(static_cast<size_t>(total), s);
  out.pair_list.alloc(static_cast<size_t>(total), s);
  out.items.alloc(static_cast<size_t>(out.max_items), s);
  out.n_items.alloc(4, s);
  const int near_ranks = std::max(1, n_probes / 8);
  dbuf<uint32_t> counts(static_cast<size_t>(2 * n_lists), s), pair_off(static_cast<size_t>(2 * n_lists), s),
    first_off(static_cast<size_t>(n_lists), s), rest_off(static_cast<size_t>(n_lists), s), cursor(static_cast<size_t>(2 * n_lists), s);
  B2_CUDA(cudaMemsetAsync(counts.data(), 0, sizeof(uint32_t) * 2 * n_lists, s));
  count_launch(4);
  count_probes_kernel<<<blocks_for(total, 256), 256, 0, s>>>(probes, total, n_probes, probe_ld, near_ranks, list_offsets_dev, counts.data());
  scan_lists_kernel<<<1, 1024, 0, s>>>(counts.data(), n_lists, static_cast<uint32_t>(group), pair_off.data(), first_off.data(), rest_off.data(), out.n_items.data(),
                                       cursor.data());
  scatter_probes_kernel<<<blocks_for(total, 256), 256, 0, s>>>(probes, total, n_probes, probe_ld, near_ranks, list_offsets_dev, pair_off.data(),
                                                                cursor.data(), out.slot_of.data(), out.pair_query.data(),
                                                                out.pair_list.data());
  make_list_items_kernel<<<blocks_for(n_lists, 128), 128, 0, s>>>(counts.data(), pair_off.data(), first_off.data(), rest_off.data(),
                                                                   out.n_items.data(), list_offsets_dev, n_lists, KC, max_tiles, static_cast<uint32_t>(group), out.items.data());
  B2_CUDA(cudaGetLastError());
}

float pair_residual_rows(cudaStream_t s, const float* q, const float* centers, int dim, int Kp, cuvsDistanceType metric,
                         const probe_buckets& pb, bool with_lo, residual_rows& a, dbuf<float>& add)
{
  const bool ip = is_ip(metric);
  a.rows        = pb.n_pairs + 128;
  a.hi.alloc(static_cast<size_t>(a.rows) * Kp, s);
  if (with_lo) a.lo.alloc(static_cast<size_t>(a.rows) * Kp, s);
  add.alloc(static_cast<size_t>(pb.n_pairs), s);
  count_launch();
  pair_rows_kernel<<<blocks_for(a.rows * 32, 256), 256, 0, s>>>(q, centers, pb.pair_query.data(), pb.pair_list.data(), pb.n_items.data() + 1,
                                                                 a.rows, dim, Kp, ip, a.hi.data(), a.lo.data(), add.data(), metric == CosineExpanded);
  B2_CUDA(cudaGetLastError());
  return ip ? 1.0f : 2.0f;
}

void gather_probe_candidates(cudaStream_t s, const float* cs, const uint32_t* cp, const uint32_t* slot_of, const float* add,
                             float scale, float empty, int64_t nq, int n_probes, int KCW, float* out_score, uint32_t* out_pos,
                             int L, float* last)
{
  const int64_t total = nq * n_probes * KCW;
  if (total == 0) return;
  count_launch();
  gather_cands_kernel<<<blocks_for(total, 256), 256, 0, s>>>(cs, cp, slot_of, add, scale, empty, total, KCW, out_score, out_pos, L,
                                                             last);
  B2_CUDA(cudaGetLastError());
}

void large_k_select(cudaStream_t s, const probe_buckets& pb, const list_layout& lists, int64_t nq, uint32_t n_probes, int kp,
                    const std::function<void(float* scores, const int64_t* seg_off)>& scan, dbuf<float>& cs,
                    dbuf<uint32_t>& cp)
{
  const int64_t n_pairs = pb.n_pairs;
  dbuf<int64_t> seg_off(static_cast<size_t>(n_pairs), s);
  dbuf<uint32_t> seg_len(static_cast<size_t>(n_pairs), s), seg_base(static_cast<size_t>(n_pairs), s);
  count_launch();
  pair_segments_kernel<<<1, 1024, 0, s>>>(pb.pair_list.data(), pb.n_items.data() + 1, n_pairs, lists.d_offsets.data(),
                                          lists.d_sizes.data(), seg_off.data(), seg_len.data(), seg_base.data());
  B2_CUDA(cudaGetLastError());
  dbuf<float> scores(static_cast<size_t>(std::max<int64_t>(1, nq * large_k_rows_per_query(lists, n_probes))), s);
  scan(scores.data(), seg_off.data());
  int64_t max_len = 0;
  for (int64_t v : lists.h_sizes) max_len = std::max(max_len, v);
  cs.alloc(static_cast<size_t>(n_pairs) * kp, s);
  cp.alloc(static_cast<size_t>(n_pairs) * kp, s);
  select_k_segments(s, scores.data(), seg_off.data(), seg_len.data(), seg_base.data(), n_pairs, max_len, kp, cs.data(), cp.data(), true);
}

void item_segments(cudaStream_t s, probe_buckets& pb, const int64_t* seg_off)
{
  count_launch();
  item_segments_kernel<<<blocks_for(pb.max_items, 256), 256, 0, s>>>(pb.items.data(), pb.n_items.data(), seg_off);
  B2_CUDA(cudaGetLastError());
}

int64_t large_k_rows_per_query(const list_layout& lists, uint32_t n_probes)
{
  const int64_t n_lists = lists.n_lists;
  std::vector<int64_t> pad(static_cast<size_t>(n_lists));
  for (int64_t l = 0; l < n_lists; ++l) pad[l] = lists.h_offsets[l + 1] - lists.h_offsets[l];
  const int64_t m = std::min<int64_t>(n_probes, n_lists);
  std::partial_sort(pad.begin(), pad.begin() + m, pad.end(), std::greater<int64_t>());
  int64_t rows = 0;
  for (int64_t i = 0; i < m; ++i) rows += pad[i];
  return rows;
}

int64_t query_batch_size(int64_t pair_bytes, uint32_t n_probes, int64_t large_k_query_bytes, const char* budget_env)
{
  int64_t batch = std::max<int64_t>(1, (int64_t(3) << 30) / (static_cast<int64_t>(n_probes) * pair_bytes));
  batch         = std::min<int64_t>(batch, (int64_t(1) << 31) / std::max<uint32_t>(n_probes, 1));
  if (large_k_query_bytes > 0) {
    int64_t budget = 0;
    if (const char* e = getenv(budget_env)) {
      budget = std::max<int64_t>(1, atoll(e)) << 20;
    } else {
      size_t free_b = 0, total_b = 0;
      B2_CUDA(cudaMemGetInfo(&free_b, &total_b));
      budget = std::min<int64_t>(int64_t(8) << 30, static_cast<int64_t>(free_b / 2));
    }
    batch = std::min<int64_t>(batch, std::max<int64_t>(1, budget / large_k_query_bytes));
  }
  return batch;
}

bool search_in_batches(int64_t batch, const DLTensor& qt, const DLTensor& nt, const DLTensor& dt,
                       const std::function<void(const DLTensor&, const DLTensor&, const DLTensor&)>& search)
{
  const int64_t nq = qt.shape[0];
  if (nq <= batch) return false;
  for (int64_t q0 = 0; q0 < nq; q0 += batch) {
    const int64_t rows = std::min(batch, nq - q0);
    dl_row_slice qs(qt, q0, rows), ns(nt, q0, rows), ds(dt, q0, rows);
    search(qs.t, ns.t, ds.t);
  }
  return true;
}

dbuf<float> train_subsample(cudaStream_t s, const DLTensor& ds, uint32_t n_lists, double fraction, int64_t& n_train)
{
  const int64_t n = ds.shape[0];
  const int d     = static_cast<int>(ds.shape[1]);
  const double frac = std::min(1.0, std::max(fraction, 0.0));
  n_train = std::max<int64_t>(n_lists, std::min<int64_t>(n, static_cast<int64_t>(std::llround(n * frac))));
  n_train = std::min<int64_t>(n_train, std::max<int64_t>(static_cast<int64_t>(n_lists) * 1024, 1 << 18));
  n_train = std::min(n_train, n);
  const int64_t stride = std::max<int64_t>(1, n / n_train);
  n_train = std::min(n_train, (n + stride - 1) / stride);
  dbuf<float> train(static_cast<size_t>(n_train) * d, s);
  if (dl_is(ds, kDLFloat, 32)) {
    B2_CUDA(cudaMemcpy2DAsync(train.data(), sizeof(float) * d, dl_ptr<float>(ds), sizeof(float) * d * stride, sizeof(float) * d, n_train,
                              cudaMemcpyDefault, s));
    return train;
  }
  // a narrower type: only the sample is widened
  const size_t row = static_cast<size_t>(d) * (ds.dtype.bits / 8);
  dbuf<uint8_t> raw(static_cast<size_t>(n_train) * row, s);
  B2_CUDA(cudaMemcpy2DAsync(raw.data(), row, dl_ptr<uint8_t>(ds), row * stride, row, n_train, cudaMemcpyDefault, s));
  widen_async(s, raw.data(), ds.dtype, n_train * d, train.data());
  return train;
}

bool merge_probe_candidates(cudaStream_t s, const float* cs, const uint32_t* cp, const uint32_t* slot_of, const float* add,
                            float scale, const int* bound_keys, int64_t nq, int n_probes, int KCW, int k, float* out_val,
                            uint32_t* out_pos)
{
  if (nq == 0) return true;
  // without a bound nothing is filtered: the generic gather + radix select is the better tool then
  if (bound_keys == nullptr && static_cast<int64_t>(n_probes) * KCW > kMergeCap) return false;
  count_launch();
  const int kcw_shift = (KCW & (KCW - 1)) == 0 ? __builtin_ctz(static_cast<unsigned>(KCW)) : -1;  // -1: not a power of two
  if (static_cast<int64_t>(n_probes) * KCW <= 2048)
    merge_pairs_kernel<128><<<static_cast<unsigned>(nq), 128, 0, s>>>(cs, cp, slot_of, add, scale, bound_keys, n_probes, KCW, kcw_shift,
                                                                     k, out_val, out_pos);
  else
    merge_pairs_kernel<256><<<static_cast<unsigned>(nq), 256, 0, s>>>(cs, cp, slot_of, add, scale, bound_keys, n_probes, KCW, kcw_shift,
                                                                     k, out_val, out_pos);
  B2_CUDA(cudaGetLastError());
  return true;
}

uint32_t abs_max_host(cudaStream_t s, const float* x, int64_t count)
{
  dbuf<uint32_t> bits(1, s);
  B2_CUDA(cudaMemsetAsync(bits.data(), 0, sizeof(uint32_t), s));
  uint32_t h = 0;
  if (count > 0) {
    count_launch();
    abs_max_kernel<<<static_cast<unsigned>(std::min<int64_t>(blocks_for(count, 256), 132 * 8)), 256, 0, s>>>(x, count, bits.data());
    B2_CUDA(cudaGetLastError());
  }
  B2_CUDA(cudaMemcpyAsync(&h, bits.data(), sizeof(h), cudaMemcpyDeviceToHost, s));
  B2_CUDA(cudaStreamSynchronize(s));
  return h;
}

void abs_max_bits(cudaStream_t s, const float* x, int64_t count, uint32_t* out_bits)
{
  B2_CUDA(cudaMemsetAsync(out_bits, 0, sizeof(uint32_t), s));
  if (count == 0) return;
  count_launch();
  abs_max_kernel<<<static_cast<unsigned>(std::min<int64_t>(blocks_for(count, 256), 132 * 8)), 256, 0, s>>>(x, count, out_bits);
  B2_CUDA(cudaGetLastError());
  uint32_t bits = 0;
  B2_CUDA(cudaMemcpyAsync(&bits, out_bits, sizeof(bits), cudaMemcpyDeviceToHost, s));
  B2_CUDA(cudaStreamSynchronize(s));
  B2_EXPECTS(bits < 0x7f800000u, "training data contains NaN or infinity");  // the fixed-point scale needs a finite maximum
}

void update_centers(cudaStream_t s, const float* x, int64_t n, int d, const uint32_t* labels, const uint32_t* x_max_bits, int k,
                    float* centers, float* counts_out)
{
  dbuf<unsigned long long> sums(static_cast<size_t>(k) * d, s), counts(static_cast<size_t>(k), s);
  B2_CUDA(cudaMemsetAsync(sums.data(), 0, sizeof(unsigned long long) * static_cast<size_t>(k) * d, s));
  B2_CUDA(cudaMemsetAsync(counts.data(), 0, sizeof(unsigned long long) * k, s));
  count_launch(2);
  accumulate_kernel<<<blocks_for(n * 32, 256), 256, 0, s>>>(x, n, d, labels, x_max_bits, sums.data(), counts.data());
  finalize_centers_kernel<<<blocks_for(static_cast<int64_t>(k) * d, 256), 256, 0, s>>>(sums.data(), counts.data(), x_max_bits, n, k, d,
                                                                                      centers, counts_out);
  B2_CUDA(cudaGetLastError());
}

void kmeans_train(resources* res, const float* x, int64_t n, int d, int k, int n_iters, float* centers, bool init_from_data,
                  bool balance, double* inertia, int* iters_done, double tol, bool sqrt_cost, bool exact_loop)
{
  auto s = res->stream;
  B2_EXPECTS(n >= 1 && k >= 1, "kmeans: empty input");
  B2_EXPECTS(tc_supported(res->device, d), "kmeans: dim %d is not supported: it pads to more than %d columns, the widest the tensor-core kernels take", d, kTcMaxK);
  if (init_from_data) {
    count_launch();
    strided_init_kernel<<<blocks_for(static_cast<int64_t>(k) * d, 256), 256, 0, s>>>(x, n, d, k, centers);
    B2_CUDA(cudaGetLastError());
  }
  // data-side planes (the dataset plays the "query" role of the scan)
  tc_rows_tmp xp;
  xp.build(s, x, n, d, true);
  dbuf<float> xn(static_cast<size_t>(n), s), cn(static_cast<size_t>(k), s), counts(static_cast<size_t>(k), s);
  dbuf<uint32_t> x_max(1, s);
  abs_max_bits(s, x, n * d, x_max.data());
  dbuf<uint32_t> labels(static_cast<size_t>(n), s);
  dbuf<double> acc(1, s);
  dbuf<int> n_reseeded(1, s);
  row_norms(s, x, n, d, d, xn.data());
  tc_rows cp;
  double prev = -1.0;
  int it      = 0;
  for (; it < std::max(n_iters, 1); ++it) {
    row_norms(s, centers, k, d, d, cn.data());
    cp.build(s, centers, k, d, cn.data(), true);
    if (exact_loop) assign_exact(res, x, xn.data(), xp, centers, cn.data(), cp, labels.data());
    else assign_nearest(res, xp.hi.data(), xp.lo.data(), n, xp.rows_pad, xp.Kp, cp, labels.data(), nullptr);
    if (n_iters == 0) break;  // assignment only
    // the convergence sum: the cost of this iteration's centres, before the update moves them
    if (tol > 0.0) kmeans_cost(s, x, n, d, centers, labels.data(), nullptr, false, sqrt_cost, acc.data());
    update_centers(s, x, n, d, labels.data(), x_max.data(), k, centers, counts.data());
    if (balance && k > 1) {
      B2_CUDA(cudaMemsetAsync(n_reseeded.data(), 0, sizeof(int), s));
      count_launch();
      reseed_small_kernel<<<blocks_for(k, 128), 128, 0, s>>>(x, n, d, labels.data(), counts.data(), k,
                                                              static_cast<float>(n) / k, it, centers, n_reseeded.data());
      B2_CUDA(cudaGetLastError());
    }
    if (tol > 0.0) {
      double cur = 0;
      B2_CUDA(cudaMemcpyAsync(&cur, acc.data(), sizeof(double), cudaMemcpyDeviceToHost, s));
      B2_CUDA(cudaStreamSynchronize(s));
      if (prev >= 0 && std::abs(prev - cur) <= tol * std::max(prev, 1e-30)) { prev = cur; ++it; break; }
      prev = cur;
    }
  }
  if (iters_done) *iters_done = it;
  if (inertia) {
    // inertia of the returned centres: exact labels, cost from differences
    row_norms(s, centers, k, d, d, cn.data());
    cp.build(s, centers, k, d, cn.data(), true);
    assign_exact(res, x, xn.data(), xp, centers, cn.data(), cp, labels.data());
    kmeans_cost(s, x, n, d, centers, labels.data(), nullptr, false, sqrt_cost, acc.data());
    B2_CUDA(cudaMemcpyAsync(inertia, acc.data(), sizeof(double), cudaMemcpyDeviceToHost, s));
    B2_CUDA(cudaStreamSynchronize(s));
  }
}

}  // namespace b200
