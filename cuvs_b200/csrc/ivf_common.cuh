// Building blocks shared by IVF-Flat, IVF-PQ and k-means (host API).
//
// Reference counterparts:
//   coarse search        cpp/src/neighbors/ivf_pq/ivf_pq_search.cuh:60-168, ivf_flat/ivf_flat_search.cuh:105-187
//   probe bookkeeping    cpp/src/neighbors/ivf_common.cuh:49-169 (chunk indices, sample -> id translation)
//   balanced k-means     cpp/src/cluster/detail/kmeans_balanced.cuh:76-1100 (EM + re-seeding of small clusters)
//   assignment step      cpp/src/cluster/detail/minClusterDistanceCompute.cu:18-165
//
// Formulation: instead of one CTA per (query, probe) that re-reads the probed list for every
// query (reference a8/a11), (query, probe) pairs are bucketed BY LIST on the device; each work item is
// "<= 128 queries that probe list l" x "the 128-row tiles of list l", which is a dense contraction the
// wgmma scan kernel (scan_tc.cu) executes with a fused top-k' epilogue.  List rows are read once per
// 128 probing queries instead of once per query.
#pragma once
#include "common.hpp"
#include "ivf_lists.cuh"
#include "scan_tc.cuh"

#include <cuda_bf16.h>

#include <functional>

namespace b200 {

/** bf16 split planes + half-norms of a set of row vectors, padded to 128-row tiles (the "B side"). */
struct tc_rows {
  int64_t n = 0, rows_pad = 0;
  int d = 0, Kp = 0;
  owned<__nv_bfloat16> hi, lo;
  owned<__nv_bfloat16> hx;  // [rows_pad, 16] half-norm plane
  void build(cudaStream_t s, const float* x, int64_t n_, int d_, const float* xn /*|x|^2 or null => hn = 0*/, bool with_lo,
             const float* row_scale = nullptr);
};

/** Temporary (stream-ordered) version of the above for query-side operands. */
struct tc_rows_tmp {
  int64_t n = 0, rows_pad = 0;
  int d = 0, Kp = 0;
  dbuf<__nv_bfloat16> hi, lo;
  void build(cudaStream_t s, const float* x, int64_t n_, int d_, bool with_lo, int64_t extra_pad_rows = 0,
             const float* row_scale = nullptr);
};

/**
 * Top-`n_probes` rows of `centers` for every query (smallest s = hn - q.c first): dense wgmma score
 * block + select_k.  probes: [nq, n_probes] uint32 (0xffffffff padding when n_probes > n_centers).
 */
void coarse_select(resources* res, const tc_rows_tmp& queries, const tc_rows& centers, int n_probes, uint32_t* probes,
                   float* probe_scores /*nullable*/);

/** labels[i] = argmin_j (hn[j] - x_i . c_j)  (nearest centre, approx = fp32-grade split products); optional score out. */
void assign_nearest(resources* res, const __nv_bfloat16* x_hi, const __nv_bfloat16* x_lo, int64_t n, int64_t x_rows_pad,
                    int Kp, const tc_rows& centers, uint32_t* labels, float* scores /*nullable*/);

/**
 * Exact nearest centres (DESIGN.md §8): labels[i] = the first j minimising the oracle's expanded distance
 * fmaf(-2, x_i.c_j, |x_i|^2 + |c_j|^2), clamped at 0 (oracle_kmeans_assign: rescore_topk's L2Expanded arithmetic without the
 * self-neighbour rule).  The scan of assign_nearest proposes 2 x 16 candidates per row, rescore_topk scores them exactly,
 * certify_candidates checks with brute force's budget that no other centre can come first, and the rows it rejects, and rows
 * with no candidate, are scored against every centre (exact_distance_tile), in launches of bounded size.  Every label is
 * below k.
 * x [n, d] fp32 rows with their squared norms xn (row_norms) and planes xp (with lo); centers [k, d] with cn and planes cp
 * (with lo).  Synchronises the stream.
 */
void assign_exact(resources* res, const float* x, const float* xn, const tc_rows_tmp& xp, const float* centers, const float* cn,
                  const tc_rows& cp, uint32_t* labels);

/**
 * The k-means cost sum_i w_i dist_i into *out (device double): dist_i = |x_i - c_{labels_i}|^2, summed in fp32 as the oracle's
 * sqdiff (fmaf, ascending components), or with sqrt_dist its square root; w_i = 1 without weights, weights[i] with them, and
 * weights[i] * n / sum(weights) with normalize_weight.  The terms are added in double in a fixed order, so a cost has the same
 * bits in every run and for every caller.
 */
void kmeans_cost(cudaStream_t s, const float* x, int64_t n, int d, const float* centers, const uint32_t* labels, const float* weights,
                 bool normalize_weight, bool sqrt_dist, double* out);

/**
 * (query, probe) pairs bucketed by list, on the device.
 *   slot_of[q * n_probes + p]  -> row of the pair in list-major order (0xffffffff for padded probes)
 *   pair_query[slot]           -> query id
 *   items / n_items            -> work list for tc_scan_topk (A rows = slots, B rows = list ranges)
 */
struct probe_buckets {
  dbuf<uint32_t> slot_of, pair_query, pair_list;
  dbuf<tc_item> items;
  dbuf<int> n_items;   // device: [0] = number of work items, [1] = number of live pairs (slots in use)
  int max_items = 0;   // host upper bound
  int64_t n_pairs = 0;
};
void bucket_probes(resources* res, const uint32_t* probes, int64_t nq, int n_probes, int64_t n_lists,
                   const int64_t* list_offsets_dev /*[n_lists+1], padded row offsets (multiples of 128)*/, int KC,
                   probe_buckets& out, int probe_ld = 0 /*row stride of `probes` (0: n_probes)*/,
                   uint32_t max_tiles = 0xffffffffu /*scan at most this many tiles of each list (bound warm-up)*/,
                   int group = 128 /*pairs (A rows) per work item*/);

/** The A rows of an IVF fine scan, one per pair slot (slots of dropped pairs are never read; the 128 rows past the pairs are
 *  zero). */
struct residual_rows {
  int64_t rows = 0;
  dbuf<__nv_bfloat16> hi, lo;
};
/**
 * Per pair slot, for a scan of list rows that hold residuals x - c (with half norms |x - c|^2/2 for L2, 0 otherwise), from the
 * fp32 query rows q [nq, dim] and list centres [n_lists, dim] (cosine: both unit): bf16 planes of q - c (L2) or q (inner
 * product, cosine), hi and, `with_lo`, lo, and add[slot], the pair's offset: |q - c|^2 (L2), -q.c (inner product), 1 - q.c
 * (cosine).  Returns `scale`: a pair's distance is add[slot] + scale * score, 2 for L2 (|q - x|^2 = |q - c|^2 +
 * 2 (|x - c|^2/2 - (q - c).(x - c))) and 1 otherwise.  Scores of different pairs are only comparable in these units.
 */
float pair_residual_rows(cudaStream_t s, const float* q, const float* centers, int dim, int Kp, cuvsDistanceType metric,
                         const probe_buckets& pb, bool with_lo, residual_rows& a, dbuf<float>& add);

/**
 * Per query, concatenate the KCW candidates of each of its probes: out [nq, n_probes * KCW], value add[slot] + scale * score
 * (add null: 0).  Empty entries, of a dropped pair or with position 0xffffffff, become (`empty`, 0xffffffff).
 * With `last`, the KCW entries of a pair are read as lists of L and the last value of every list is also written to
 * last[q, p * (KCW / L) + j] (list j of probe p): what IVF-Flat's certificate reads of them.
 */
void gather_probe_candidates(cudaStream_t s, const float* cs, const uint32_t* cp, const uint32_t* slot_of, const float* add,
                             float scale, float empty, int64_t nq, int n_probes, int KCW, float* out_score, uint32_t* out_pos,
                             int L = 0, float* last = nullptr);

/**
 * Per query: the k best (value, position) among its probes' candidates, value = add[slot] + scale * score, sorted
 * ascending (ties: smaller position), missing entries (FLT_MAX, 0xffffffff).  `bound_keys` [nq] is the scan's tc_bound
 * state — an upper bound on each query's k-th best value in the same units (null: no bound).  Returns false (nothing
 * launched) when the shape needs the generic gather + select_k path instead.
 */
bool merge_probe_candidates(cudaStream_t s, const float* cs, const uint32_t* cp, const uint32_t* slot_of, const float* add,
                            float scale, const int* bound_keys, int64_t nq, int n_probes, int KCW, int k, float* out_val,
                            uint32_t* out_pos);

/**
 * Queries per batch of an IVF search (DESIGN.md §4a).  A (query, probe) pair's workspace takes `pair_bytes`; a batch's pairs
 * stay within ~3 GiB and, slots being uint32, below 2^31.  k > 64 (`large_k_query_bytes` > 0, a query's workspace): a batch
 * also stays within min(8 GiB, half of the free device memory), or within the env variable `budget_env` (MiB), read on every
 * call, when it is set.
 */
int64_t query_batch_size(int64_t pair_bytes, uint32_t n_probes, int64_t large_k_query_bytes = 0, const char* budget_env = nullptr);
/** When nq > batch: runs `search` on the (queries, neighbors, distances) rows of each batch in turn and returns true. */
bool search_in_batches(int64_t batch, const DLTensor& qt, const DLTensor& nt, const DLTensor& dt,
                       const std::function<void(const DLTensor&, const DLTensor&, const DLTensor&)>& search);

/**
 * k > 64 (DESIGN.md §4a): the `kp` best rows of every pair.  Gives each live pair a dense segment of scores, one per row of
 * its list in list order, and calls scan(scores, seg_off) to fill them (seg_off[slot]: the slot's segment; a tensor-core
 * scan points its items there with item_segments).  Then a segmented select keeps each pair's kp best rows into cs / cp
 * [n_pairs, kp] (positions are index rows, ties go to the smaller row, missing entries (FLT_MAX, 0xffffffff)), and the
 * scores are released.
 */
void large_k_select(cudaStream_t s, const probe_buckets& pb, const list_layout& lists, int64_t nq, uint32_t n_probes, int kp,
                    const std::function<void(float* scores, const int64_t* seg_off)>& scan, dbuf<float>& cs,
                    dbuf<uint32_t>& cp);
/** Points every work item's out_off at the segment of its first slot; a store scan with a per-item row stride (n_tiles x 128)
 *  then writes each pair's scores into its own segment. */
void item_segments(cudaStream_t s, probe_buckets& pb, const int64_t* seg_off);
/** Upper bound on the dense score rows of one query: the sum of the n_probes largest padded lists. */
int64_t large_k_rows_per_query(const list_layout& lists, uint32_t n_probes);

/**
 * Training rows of an IVF build: an evenly strided subsample of the rows of `ds` ([n, d], device or host; float16, int8 and
 * uint8 rows are widened after sampling), every
 * stride-th row from row 0.  About fraction x n rows (fraction clamped to [0, 1]), at least n_lists, at most
 * max(n_lists x 1024, 2^18) (ivf_flat_build.cuh:430-455 uses the same rule).  n_train receives the row count.
 */
dbuf<float> train_subsample(cudaStream_t s, const DLTensor& ds, uint32_t n_lists, double fraction, int64_t& n_train);

/**
 * Balanced-ish Lloyd k-means on the device (fp32 data, wgmma assignment).  `centers` [k, d] is
 * initialised from evenly strided rows when `init_from_data`, then refined for `n_iters` iterations;
 * clusters smaller than 1/4 of the average are re-seeded from members of large clusters each iteration.
 * Each iteration assigns with assign_exact when `exact_loop` (cuvsKMeansFit: every update is the mean over the oracle's
 * labels), else with the approximate assign_nearest (IVF builds' coarse training, DESIGN.md §8).
 * With `tol` > 0 training stops once the cost changes by at most tol x the previous cost.  `inertia` != null receives the
 * kmeans_cost of the returned centres over exact labels (sqrt_cost: sum of distances, L2SqrtExpanded).
 */
void kmeans_train(resources* res, const float* x, int64_t n, int d, int k, int n_iters, float* centers,
                  bool init_from_data, bool balance, double* inertia, int* iters_done, double tol = 0.0, bool sqrt_cost = false,
                  bool exact_loop = false);

/**
 * Deterministic sums for the training loops (k-means centres, PQ codebooks).  Float atomics round differently depending on
 * the order in which threads arrive, so two builds from the same data would train different indexes.  Instead every value is
 * added as a fixed-point int64, v * 2^e rounded, and integer addition does not depend on the order.  e is chosen from the
 * largest |v| of the input (abs_max_bits) and the number of terms n so that no sum can overflow:  |v| * 2^e * n < 2^62.
 */
void abs_max_bits(cudaStream_t s, const float* x, int64_t count, uint32_t* out_bits /*device, one word*/);
/** max |v| over the count values of x as fp32 bits, on the host (0x7f800000 or more: x holds an infinity or a NaN).
 *  Synchronises the stream. */
uint32_t abs_max_host(cudaStream_t s, const float* x, int64_t count);
__device__ __forceinline__ double fixed_scale(uint32_t max_bits, int64_t n)
{
  int ex = 0;
  frexpf(__uint_as_float(max_bits), &ex);  // max |v| < 2^ex
  const int nb = 64 - __clzll(static_cast<unsigned long long>(n > 0 ? n : 1));  // n < 2^nb
  return ldexp(1.0, min(62 - ex - nb, 1000));
}
__device__ __forceinline__ void fixed_add(unsigned long long* acc, float v, double scale)
{
  atomicAdd(acc, static_cast<unsigned long long>(__double2ll_rn(static_cast<double>(v) * scale)));
}
__device__ __forceinline__ double fixed_value(unsigned long long acc, double scale) { return static_cast<double>(static_cast<long long>(acc)) / scale; }

/** Sum of member rows and member counts per label (deterministic fixed-point sums), then centers = sums / counts where
 *  counts > 0; counts_out[k] receives the member counts.  x_max_bits = abs_max_bits of x. */
void update_centers(cudaStream_t s, const float* x, int64_t n, int d, const uint32_t* labels, const uint32_t* x_max_bits, int k,
                    float* centers, float* counts_out);

}  // namespace b200
