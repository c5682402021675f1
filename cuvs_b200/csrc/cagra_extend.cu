// CAGRA extend (cuvsCagraExtend): new rows join the graph without a rebuild, entirely on the device.
//
// Reference: cpp/src/neighbors/detail/cagra/add_nodes.cuh:23-484 (add_node_core, add_graph_nodes, extend_core), C wrapper
// c/src/neighbors/cagra.cpp:172-199, :631-637.  The reference searches on the GPU and does the rest on the host (graph
// copied to host memory, OpenMP ranking, a single-threaded reverse-edge loop, the dataset staged through host memory).
// Here every step is a kernel; the semantics, and where they deliberately differ from the reference, are in DESIGN.md §6
// ("Extend") and restated in numpy in tests/cagra_extend_ref.py.
//
// Per chunk of new rows (n0 = rows in the index when the chunk starts, d = graph degree, B = 2d):
//   0. in_degree_kernel     cnt[v] = occurrences of v in the chunk-start graph; cnt of the chunk's own rows = d/2
//   1. cagra_search         the chunk's rows as queries, k = B, itopk max(2B, 256), search width 1, algorithm pinned
//   2. rank_kernel          rank-based reordering of the B candidates, the first d become the provisional row
//   3. claim / commit       reverse edges in deterministic-reservation rounds (exactly the sequential node order)
#include "cagra.cuh"
#include "ptx_sm90.cuh"
#include "timing.hpp"

#include <cuvs/neighbors/cagra.h>

#include <algorithm>
#include <memory>

namespace b200 {
namespace {

constexpr uint32_t kInvalid       = 0xffffffffu;
constexpr int kMaxExtendDegree    = 256;  // rank_kernel's mask is B x B bits in shared memory (32 KiB at d = 256)
constexpr int kRankThreads        = 256;
constexpr size_t kRankRowBytes    = 128 * 1024;  // staged candidate rows per stage: all of them up to d = 128
constexpr int kCommitWarps        = 8;

// step 0: in-degree of every row in the chunk-start graph (ids outside [0, n0) are not counted); the chunk's own rows get
// d/2, the value the reference assigns each new row once its reverse edges are in (add_nodes.cuh:233) — a new row's count is
// only read after that row has been written into a target's row, so setting it up front is the same.
__global__ void in_degree_kernel(const uint32_t* __restrict__ graph, int64_t entries, int64_t n0, int64_t n_chunk, uint32_t half,
                                 uint32_t* __restrict__ cnt)
{
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i < entries) {
    const uint32_t v = graph[i];
    if (v < n0) atomicAdd(cnt + v, 1u);
  }
  if (i < n_chunk) cnt[n0 + i] = half;
}

__device__ __forceinline__ uint32_t rank_slot(uint32_t id, uint32_t bits) { return (id * 0x9E3779B1u) >> (32 - bits); }

// step 2, one CTA per new row.  cand: the row's B search results.  The graph rows of the valid candidates (id < n0) are
// staged in shared memory (one bulk copy per row on an mbarrier when rows are 16-byte multiples), ids map to ranks through a
// small open-addressing table, and an entry a of candidate j's row with rank(a) > j sets bit j of mask[rank(a)]: the count
// of rank i is popc(mask[i]), the number of closer candidates whose row holds it (a duplicate entry counted once, as the
// reference's `break`).  An invalid candidate counts B + 1.  Candidates are ordered by (count, rank) — a stable sort — and
// the first d written as the provisional row.  A provisional row whose first d/2 entries hold an invalid id records the
// row in err (the reference fails on it, add_nodes.cuh:199-202).
template <bool BULK>
__global__ void __launch_bounds__(kRankThreads) rank_kernel(const uint32_t* __restrict__ cand, const uint32_t* __restrict__ graph, int64_t n0,
                                                            int degree, int rows_per_stage, uint32_t hash_bits, uint32_t* __restrict__ out,
                                                            unsigned long long* __restrict__ err)
{
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int B = 2 * degree, W = (B + 31) / 32, tid = threadIdx.x;
  const uint32_t H = 1u << hash_bits;
  uint32_t* rows  = reinterpret_cast<uint32_t*>(smem_raw);  // [rows_per_stage, degree]
  uint64_t* bar   = reinterpret_cast<uint64_t*>(rows + static_cast<size_t>(rows_per_stage) * degree + ((rows_per_stage * degree) & 1));
  uint32_t* ids   = reinterpret_cast<uint32_t*>(bar + 1);  // [B]
  uint32_t* hkey  = ids + B;                               // [H]
  uint32_t* hval  = hkey + H;                              // [H]
  uint32_t* mask  = hval + H;                              // [B, W]
  uint32_t* key   = mask + B * W;                          // [B]
  const int64_t node = blockIdx.x;
  for (int j = tid; j < B; j += blockDim.x) ids[j] = cand[node * B + j];
  for (uint32_t j = tid; j < H; j += blockDim.x) hkey[j] = kInvalid;
  for (int j = tid; j < B * W; j += blockDim.x) mask[j] = 0;
  if (BULK && tid == 0) {
    ptx::mbar_init(bar, 1);
    ptx::fence_barrier_init();
  }
  __syncthreads();
  for (int j = tid; j < B; j += blockDim.x) {
    const uint32_t id = ids[j];
    if (id >= n0) continue;
    for (uint32_t s = rank_slot(id, hash_bits);; s = (s + 1) & (H - 1)) {
      const uint32_t old = atomicCAS(hkey + s, kInvalid, id);
      if (old == kInvalid) { hval[s] = static_cast<uint32_t>(j); break; }
      if (old == id) break;  // (search results are distinct)
    }
  }
  __syncthreads();
  uint32_t phase = 0;
  for (int s0 = 0; s0 < B; s0 += rows_per_stage) {
    const int ns = min(rows_per_stage, B - s0);
    if constexpr (BULK) {
      const uint32_t row_bytes = static_cast<uint32_t>(degree) * 4u;
      const bool mine = tid < ns && ids[s0 + tid] < n0;
      const int nvalid = __syncthreads_count(mine);
      if (nvalid == 0) continue;
      if (tid == 0) ptx::mbar_arrive_expect_tx(bar, static_cast<uint32_t>(nvalid) * row_bytes);
      __syncthreads();
      if (mine) ptx::bulk_load_1d(rows + static_cast<size_t>(tid) * degree, graph + static_cast<int64_t>(ids[s0 + tid]) * degree, row_bytes, bar);
      ptx::mbar_wait(bar, phase);
      phase ^= 1u;
    } else {
      for (int e = tid; e < ns * degree; e += blockDim.x) {
        const uint32_t id = ids[s0 + e / degree];
        if (id < n0) rows[e] = graph[static_cast<int64_t>(id) * degree + e % degree];
      }
      __syncthreads();
    }
    for (int e = tid; e < ns * degree; e += blockDim.x) {
      const int j = s0 + e / degree;
      if (ids[j] >= n0) continue;
      const uint32_t a = rows[e];
      for (uint32_t s = rank_slot(a, hash_bits);; s = (s + 1) & (H - 1)) {
        const uint32_t k = hkey[s];
        if (k == kInvalid) break;
        if (k == a) {
          const uint32_t r = hval[s];
          if (r > static_cast<uint32_t>(j)) atomicOr(mask + r * W + (j >> 5), 1u << (j & 31));
          break;
        }
      }
    }
    __syncthreads();  // the next stage overwrites the rows
    if constexpr (BULK) ptx::fence_proxy_async();
  }
  for (int i = tid; i < B; i += blockDim.x) {
    uint32_t c = static_cast<uint32_t>(B) + 1;
    if (ids[i] < n0) {
      c = 0;
      for (int w = 0; w < W; ++w) c += __popc(mask[i * W + w]);
    }
    key[i] = (c << 16) | static_cast<uint32_t>(i);  // ranks < 1024, counts <= B + 1
  }
  __syncthreads();
  for (int i = tid; i < B; i += blockDim.x) {
    const uint32_t ki = key[i];
    int pos = 0;
    for (int j = 0; j < B; ++j) pos += key[j] < ki;
    if (pos < degree) {
      out[node * degree + pos] = ids[i];
      if (pos < degree / 2 && ids[i] >= n0) atomicMin(err, static_cast<unsigned long long>(node));
    }
  }
}

// step 3, claims: every pending row asks for each of its d/2 targets; the lowest row asking wins the target.  The stamp's
// upper half falls with the round, so a claim from an earlier round (or chunk) never blocks a later one and the table needs
// no reset.
__global__ void claim_kernel(const uint32_t* __restrict__ graph, int64_t n0, int degree, const uint32_t* __restrict__ pending, int64_t n_pending,
                             unsigned long long stamp_hi, unsigned long long* __restrict__ owner)
{
  const int half  = degree / 2;
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n_pending * half) return;
  const uint32_t node = pending[i / half];
  const uint32_t t    = graph[(n0 + node) * degree + i % half];
  if (t < n0) atomicMin(owner + t, stamp_hi | node);
}

// step 3, commits, one warp per pending row.  A row that holds all of its targets runs the reference's sequential step on
// them (add_nodes.cuh:191-275): for each target t of the first d/2 provisional entries, the neighbour with the largest
// in-degree among slots d-1 .. d/2 of t's row (ties to the higher slot, neighbours already taken for this row skipped) is
// replaced by the new row and remembered; with no such neighbour slot 0 is overwritten and nothing remembered.  The new row
// then alternates provisional entries and remembered neighbours, skipping invalid ids and duplicates.  Rows that hold some
// but not all targets go to the next round's list.  Every earlier row sharing a target has committed before a row can hold
// it, and committing rows touch disjoint target rows, so the graph is the one the sequential loop writes.
__global__ void __launch_bounds__(kCommitWarps * 32) commit_kernel(uint32_t* __restrict__ graph, const uint32_t* __restrict__ cnt, int64_t n0,
                                                                   int64_t n_end, int degree, const uint32_t* __restrict__ pending, int64_t n_pending,
                                                                   const unsigned long long* __restrict__ owner, unsigned long long stamp_hi,
                                                                   uint32_t* __restrict__ next, uint32_t* __restrict__ n_next,
                                                                   unsigned long long* __restrict__ err)
{
  extern __shared__ __align__(16) uint32_t commit_smem[];
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31, half = degree / 2;
  const int64_t p = blockIdx.x * static_cast<int64_t>(kCommitWarps) + wid;
  if (p >= n_pending) return;
  uint32_t* prov = commit_smem + static_cast<size_t>(wid) * (2 * degree + half);  // [degree]
  uint32_t* temp = prov + degree;                                                 // [degree]
  uint32_t* rev  = temp + degree;                                                 // [half]
  const uint32_t node = pending[p];
  const int64_t new_id = n0 + node;
  uint32_t* row = graph + new_id * degree;
  bool held = true, bad = false;
  for (int s = lane; s < half; s += 32) {
    const uint32_t t = row[s];
    if (t >= n0) bad = true;
    else held &= owner[t] == (stamp_hi | node);
  }
  if (__any_sync(0xffffffffu, bad)) return;  // an invalid target: recorded by rank_kernel, the extend fails
  if (!__all_sync(0xffffffffu, held)) {
    if (lane == 0) next[atomicAdd(n_next, 1u)] = node;
    return;
  }
  for (int s = lane; s < degree; s += 32) prov[s] = row[s];
  __syncwarp();
  for (int i = 0; i < half; ++i) {
    uint32_t* trow = graph + static_cast<int64_t>(prov[i]) * degree;
    unsigned long long best = 0;  // (in-degree << 32) | slot; 0 = none (an in-degree must be > 0 to qualify)
    for (int j = half + lane; j < degree; j += 32) {
      const uint32_t v = trow[j];
      if (v >= n_end) { atomicMin(err, static_cast<unsigned long long>(node)); continue; }
      const uint32_t c = cnt[v];
      if (c == 0) continue;
      bool dup = false;
      for (int k = 0; k < i; ++k) dup |= rev[k] == v;
      if (!dup) best = max(best, (static_cast<unsigned long long>(c) << 32) | static_cast<uint32_t>(j));
    }
    for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
    if (lane == 0) {
      const uint32_t j = static_cast<uint32_t>(best);
      rev[i]  = best ? trow[j] : kInvalid;
      trow[j] = static_cast<uint32_t>(new_id);
    }
    __syncwarp();
  }
  int na = 0, ri = 0, vi = 0;
  // takes the next entry of list L (from *ix) that is valid and not yet in temp
  auto take = [&](const uint32_t* L, int& ix, int len) {
    for (; ix < len; ++ix) {
      const uint32_t c = L[ix];
      if (c >= n_end) continue;
      bool dup = false;
      for (int q = lane; q < na; q += 32) dup |= temp[q] == c;
      if (!__any_sync(0xffffffffu, dup)) {
        if (lane == 0) temp[na] = c;
        __syncwarp();
        ++na;
        ++ix;
        return;
      }
    }
  };
  for (int sw = 0; na < degree && (ri < degree || vi < half); sw ^= 1) {
    if (sw == 0) take(prov, ri, degree);
    else take(rev, vi, half);
  }
  if (na < degree) {
    if (lane == 0) atomicMin(err + 1, (static_cast<unsigned long long>(node) << 32) | static_cast<uint32_t>(na));
    return;
  }
  for (int s = lane; s < degree; s += 32) row[s] = temp[s];
}

__global__ void iota_kernel(uint32_t* __restrict__ out, int64_t n)
{
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i < n) out[i] = static_cast<uint32_t>(i);
}

size_t rank_smem_bytes(int degree, int rows_per_stage, uint32_t hash_bits)
{
  const size_t B = 2 * static_cast<size_t>(degree), W = (B + 31) / 32;
  const size_t rows_words = static_cast<size_t>(rows_per_stage) * degree;
  return (rows_words + (rows_words & 1)) * 4 + 8 + (B + (size_t(2) << hash_bits) + B * W + B) * 4;
}

struct search_params_guard {
  cuvsCagraSearchParams_t p = nullptr;
  ~search_params_guard() { if (p) cuvsCagraSearchParamsDestroy(p); }
};

}  // namespace

// One chunk (rows [n0, n0 + nc) of g, whose graph rows [0, n0) are the chunk-start graph).  `round` counts reservation
// rounds over the whole extend (the claim stamps).
static void extend_chunk(resources* r, cagra_index& g, int64_t n0, int64_t nc, uint32_t* cnt, unsigned long long* owner, uint32_t& round,
                         unsigned long long* err)
{
  auto s = r->stream;
  const int d = g.degree, B = 2 * d, half = d / 2;
  const size_t es = row_bytes(g.type);
  uint32_t* graph = const_cast<uint32_t*>(g.graph);
  // ---- step 0
  B2_CUDA(cudaMemsetAsync(cnt, 0, sizeof(uint32_t) * static_cast<size_t>(n0 + nc), s));
  count_launch();
  in_degree_kernel<<<blocks_for(std::max<int64_t>(n0 * d, nc), 256), 256, 0, s>>>(graph, n0 * d, n0, nc, static_cast<uint32_t>(half), cnt);
  B2_CUDA(cudaGetLastError());
  // ---- step 1: the chunk-start index searched with the chunk's rows, exactly as cuvsCagraSearch would (fp32 queries)
  dbuf<uint32_t> cand(static_cast<size_t>(nc) * B, s);
  {
    timed_section ts("cagra_extend_search", s);
    dbuf<unsigned char> rows(static_cast<size_t>(nc) * g.dim * es, s);
    B2_CUDA(cudaMemcpy2DAsync(rows.data(), es * g.dim, static_cast<const unsigned char*>(g.data) + static_cast<size_t>(n0) * g.ld * es, es * g.ld,
                              es * g.dim, nc, cudaMemcpyDeviceToDevice, s));
    const dl_view q(rows.data(), DLDevice{kDLCUDA, r->device}, dtype_of(g.type), nc, g.dim);
    f32_rows wq;
    widen_to_f32(r, q.t(), wq);
    search_params_guard sp;
    B2_EXPECTS(cuvsCagraSearchParamsCreate(&sp.p) == CUVS_SUCCESS, "cagra extend: search parameters");
    sp.p->itopk_size   = std::max<size_t>(2 * static_cast<size_t>(B), 256);
    sp.p->search_width = 1;
    sp.p->algo         = sp.p->itopk_size <= 512 ? SINGLE_CTA : MULTI_CTA;  // pinned: AUTO would switch on the chunk size
    dbuf<float> dist(static_cast<size_t>(nc) * B, s);
    const int64_t n_total = g.n;
    g.n = n0;  // the chunk-start index: rows and graph rows [0, n0)
    try {
      cagra_search(r, g, *sp.p, dl_ptr<float>(wq.t), nc, B, cand.data(), nullptr, dist.data());
    } catch (...) {
      g.n = n_total;
      throw;
    }
    g.n = n_total;
  }
  // ---- step 2
  {
    timed_section ts("cagra_extend_rank", s);
    const int rows_per_stage = static_cast<int>(std::min<size_t>(B, kRankRowBytes / (4 * static_cast<size_t>(d))));
    uint32_t hash_bits = 6;
    while ((1u << hash_bits) < 2u * B) ++hash_bits;
    const size_t smem = rank_smem_bytes(d, rows_per_stage, hash_bits);
    const bool bulk = (4 * d) % 16 == 0;
    auto kern = bulk ? rank_kernel<true> : rank_kernel<false>;
    B2_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    count_launch();
    kern<<<static_cast<unsigned>(nc), kRankThreads, smem, s>>>(cand.data(), graph, n0, d, rows_per_stage, hash_bits, graph + n0 * d, err);
    B2_CUDA(cudaGetLastError());
  }
  // ---- step 3: rounds until no row is pending
  if (half == 0) return;
  dbuf<uint32_t> list_a(static_cast<size_t>(nc), s), list_b(static_cast<size_t>(nc), s), n_next(1, s);
  count_launch();
  iota_kernel<<<blocks_for(nc, 256), 256, 0, s>>>(list_a.data(), nc);
  uint32_t* pending = list_a.data();
  uint32_t* next    = list_b.data();
  int64_t n_pending = nc;
  const size_t commit_smem = sizeof(uint32_t) * kCommitWarps * (2 * d + half);
  B2_CUDA(cudaFuncSetAttribute(commit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(commit_smem)));
  while (n_pending > 0) {
    timed_section ts("cagra_extend_round", s);
    const unsigned long long stamp_hi = static_cast<unsigned long long>(0xffffffffu - round) << 32;
    ++round;
    B2_CUDA(cudaMemsetAsync(n_next.data(), 0, sizeof(uint32_t), s));
    count_launch(2);
    claim_kernel<<<blocks_for(n_pending * half, 256), 256, 0, s>>>(graph, n0, d, pending, n_pending, stamp_hi, owner);
    commit_kernel<<<blocks_for(n_pending, kCommitWarps), kCommitWarps * 32, commit_smem, s>>>(graph, cnt, n0, n0 + nc, d, pending, n_pending, owner,
                                                                                              stamp_hi, next, n_next.data(), err);
    B2_CUDA(cudaGetLastError());
    uint32_t left = 0;
    B2_CUDA(cudaMemcpyAsync(&left, n_next.data(), sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    B2_CUDA(cudaStreamSynchronize(s));
    B2_EXPECTS(static_cast<int64_t>(left) < n_pending, "cagra extend: a reservation round committed no row");
    n_pending = left;
    std::swap(pending, next);
  }
}

static void cagra_extend(resources* r, const cuvsCagraExtendParams& ep, const DLTensor& add, cuvsCagraIndex_t index)
{
  auto& idx = index_of<cagra_index>(index);
  B2_EXPECTS(dl_is_dataset_dtype(add), "Unsupported dataset DLtensor dtype: %d and bits: %d", add.dtype.code, add.dtype.bits);
  B2_EXPECTS(row_type_of(add.dtype) == idx.type, "type mismatch between index and additional dataset");
  B2_EXPECTS(add.ndim == 2 && dl_is_c_contiguous(add), "additional dataset must be a row-major 2-D tensor");
  B2_EXPECTS(add.shape[1] == idx.dim, "additional dataset dim (%lld) != index dim (%d)", (long long)add.shape[1], idx.dim);
  const int64_t n_add = add.shape[0], n0 = idx.n, n_total = n0 + n_add;
  if (n_add == 0) return;
  B2_EXPECTS(n_total < (int64_t(1) << 31), "cagra extend: at most 2^31 - 1 rows (the index MSB flags visited parents)");
  const int d = idx.degree;
  B2_EXPECTS(d >= 1 && d <= kMaxExtendDegree, "cagra extend: graph degree %d is outside [1, %d]", d, kMaxExtendDegree);
  auto s = r->stream;
  // the grown index is built beside the old one and replaces it only when every chunk succeeded
  auto g    = std::make_unique<cagra_index>();
  g->device = idx.device; g->metric = idx.metric; g->type = idx.type; g->dim = idx.dim; g->ld = idx.ld; g->degree = d; g->n = n_total;
  const size_t es = row_bytes(idx.type);
  {
    timed_section ts("cagra_extend_copy", s);
    g->data_own.alloc(static_cast<size_t>(n_total) * idx.ld * es);
    unsigned char* rows = g->data_own.data();
    B2_CUDA(cudaMemcpyAsync(rows, idx.data, static_cast<size_t>(n0) * idx.ld * es, cudaMemcpyDeviceToDevice, s));
    unsigned char* tail = rows + static_cast<size_t>(n0) * idx.ld * es;
    B2_CUDA(cudaMemsetAsync(tail, 0, static_cast<size_t>(n_add) * idx.ld * es, s));
    B2_CUDA(cudaMemcpy2DAsync(tail, es * idx.ld, add.data, es * idx.dim, es * idx.dim, n_add, cudaMemcpyDefault, s));
    g->data = rows;
    g->graph_own.alloc(static_cast<size_t>(n_total) * d);
    B2_CUDA(cudaMemcpyAsync(g->graph_own.data(), idx.graph, sizeof(uint32_t) * n0 * d, cudaMemcpyDeviceToDevice, s));
    g->graph = g->graph_own.data();
    set_inv_norms(r, *g);  // per row, so the old rows keep their bits
    if (idx.data16.data() != nullptr) set_half_rows(r, *g);
  }
  const int64_t chunk = ep.max_chunk_size == 0 ? n_add : static_cast<int64_t>(ep.max_chunk_size);
  dbuf<uint32_t> cnt(static_cast<size_t>(n_total), s);
  dbuf<unsigned long long> owner(static_cast<size_t>(n_total), s), err(2, s);
  B2_CUDA(cudaMemsetAsync(owner.data(), 0xff, sizeof(unsigned long long) * n_total, s));
  B2_CUDA(cudaMemsetAsync(err.data(), 0xff, sizeof(unsigned long long) * 2, s));
  uint32_t round = 0;
  for (int64_t c0 = 0; c0 < n_add; c0 += chunk) {
    const int64_t nc = std::min(chunk, n_add - c0);
    extend_chunk(r, *g, n0 + c0, nc, cnt.data(), owner.data(), round, err.data());
    unsigned long long e[2];
    B2_CUDA(cudaMemcpyAsync(e, err.data(), sizeof(e), cudaMemcpyDeviceToHost, s));
    B2_CUDA(cudaStreamSynchronize(s));
    // the reference stops at the first failing row of the chunk (add_nodes.cuh:199-202, :266-271)
    const unsigned long long bad_row = e[0], short_row = e[1] == ~0ull ? ~0ull : e[1] >> 32;
    if (bad_row != ~0ull && bad_row <= short_row)
      B2_FAIL("cagra extend: Invalid node ID found in updated_graph (new row %lld: the search found fewer than %d neighbours)",
              (long long)(n0 + c0 + static_cast<int64_t>(bad_row)), d / 2);
    if (short_row != ~0ull)
      B2_FAIL("Number of edges is not enough (target_new_node_id:%lld, num_add:%u, degree:%d)", (long long)(n0 + c0 + static_cast<int64_t>(short_row)),
              static_cast<uint32_t>(e[1]), d);
  }
  B2_CUDA(cudaStreamSynchronize(s));
  set_index(index, g.release(), index->dtype);
}

}  // namespace b200

using namespace b200;

extern "C" cuvsError_t cuvsCagraExtend(cuvsResources_t res, cuvsCagraExtendParams_t params, DLManagedTensor* additional_dataset,
                                       cuvsCagraIndex_t index)
{
  return guarded([=] {
    auto r = as_res(res);
    B2_EXPECTS(params && additional_dataset && index, "null argument");
    cagra_extend(r, *params, additional_dataset->dl_tensor, index);
  });
}
