/*
 * cuvs_b200 extensions to the cuVS C ABI (not part of the reference's surface):
 * per-kernel CUDA-event timing for bench.py's roofline block, and introspection hooks used by the
 * parity tests.  None of these is needed by a binding that only uses the reference's API.
 */
#pragma once
#include <cuvs/core/c_api.h>
#include <cuvs/neighbors/brute_force.h>
#include <cuvs/neighbors/cagra.h>
#include <cuvs/neighbors/ivf_flat.h>
#include <cuvs/neighbors/ivf_pq.h>
#include <stdbool.h>
#ifdef __cplusplus
extern "C" {
#endif

/* Enable/disable recording of CUDA events around the library's dominant kernels (on the stream they
 * are launched on).  Disabled by default (zero overhead). */
CUVS_EXPORT void cuvsB200TimingEnable(int on);
/* Discards everything recorded so far. */
CUVS_EXPORT void cuvsB200TimingReset(void);
/* Synchronises the recorded events of section `name` ("tc_scan", "pq_scan", "cagra_search", ...)
 * and returns their summed duration in milliseconds; *count receives the number of launches. */
CUVS_EXPORT double cuvsB200TimingTotalMs(const char* name, int* count);

/* Number of queries of the calling thread's last cuvsBruteForceSearch (or last IVF-Flat query batch) that failed the
 * candidate certificate and were recomputed on the exact path, and the number of kernels that search launched. */
CUVS_EXPORT int cuvsB200LastFlagged(void);
CUVS_EXPORT long long cuvsB200KernelLaunches(void);

/* Raw candidate output of the tensor-core scan of brute force (after the per-split merge):
 * cand_pos [nq, kc] uint32, cand_score [nq, kc] f32, the scan's score s = |x|^2/2 - q.x (L2 metrics), -q.x (inner product)
 * or -cos of the unit rows (cosine), kc in {16, 32}.  queries: float32, or the index's own row type, as
 * cuvsBruteForceSearch takes them.  On int8 / uint8 L2 and inner-product indexes the scores are exact (half the integer
 * |x|^2 - 2 q.x for L2), and kc = 32 needs a dimension of at most 128. */
CUVS_EXPORT cuvsError_t cuvsB200BruteForceCandidates(cuvsResources_t res,
                                                     cuvsBruteForceIndex_t index,
                                                     DLManagedTensor* queries,
                                                     DLManagedTensor* cand_pos,
                                                     DLManagedTensor* cand_score);
/* Brute force: the element type the index keeps its rows in (*row_type: 0 float32, 1 float16, 2 int8, 3 uint8) and the device
 * bytes the index owns (a float32 index built on a device view does not own the rows). */
CUVS_EXPORT cuvsError_t cuvsB200BruteForceIndexInfo(cuvsBruteForceIndex_t index, int* row_type, int64_t* device_bytes);
/* IVF-Flat list introspection (the reference exposes the equivalent only for IVF-PQ:
 * cuvsIvfPqIndexGetListSizes / cuvsIvfPqIndexGetListIndices).  Non-owning views into the index. */
CUVS_EXPORT cuvsError_t cuvsB200IvfFlatGetListSizes(cuvsIvfFlatIndex_t index, DLManagedTensor* list_sizes /*[n_lists] u32*/);
CUVS_EXPORT cuvsError_t cuvsB200IvfFlatGetListIndices(cuvsIvfFlatIndex_t index, uint32_t label, DLManagedTensor* ids /*[size] i64*/);
CUVS_EXPORT cuvsError_t cuvsB200IvfFlatGetSize(cuvsIvfFlatIndex_t index, int64_t* size);
/* Replace the coarse centres of an (empty) index — used by the list-sharded multi-GPU build so that every rank
 * partitions the data with bit-identical centres (trained on one rank, broadcast over NCCL). centers: [n_lists, dim] f32. */
CUVS_EXPORT cuvsError_t cuvsB200IvfFlatSetCenters(cuvsResources_t res, cuvsIvfFlatIndex_t index, DLManagedTensor* centers);
/* IVF-Flat fine-scan candidates of a search at k (1..64) with n_probes, as its certificate sees them (DESIGN.md §4): per
 * query the kc2 = cand_ids.shape[1] merged candidates (kc2 must be max(32, 2k)) by their approximate distance in the scan's
 * units (|q - x|^2 for L2, 2 (1 - cos) for cosine, -q.x for inner product; INT64_MAX / +inf for empty slots), and for each
 * the error budget of its own (query, list) pair against the exact fp32 distance (+inf for empty slots).  queries: f32
 * device [nq, dim], one query batch. */
CUVS_EXPORT cuvsError_t cuvsB200IvfFlatCandidates(cuvsResources_t res, cuvsIvfFlatIndex_t index, uint32_t n_probes, int k,
                                                  DLManagedTensor* queries, DLManagedTensor* cand_ids /*[nq, kc2] i64*/,
                                                  DLManagedTensor* cand_dist /*[nq, kc2] f32*/, DLManagedTensor* bound /*[nq, kc2] f32*/);

/* IVF-PQ: which fine-scan kernel cuvsIvfPqSearch will use on this index by default, and the device bytes the index holds.
 * *path: bit 1 (value 2) = the index holds the code stream (code-streaming wgmma scan, scan_pq.cu), bit 0 (value 1) = it holds
 * decoded bf16 rows (decoded-row wgmma scan, scan_tc.cu; on a streamed index: the small-index cache used by densely probing
 * batches), 0 = LUT kernel only. */
CUVS_EXPORT cuvsError_t cuvsB200IvfPqIndexInfo(cuvsIvfPqIndex_t index, int* path, int64_t* device_bytes);
/* IVF-PQ bound pre-pass (DESIGN.md §5): with on != 0, every later code-stream search that runs the pre-pass keeps, for the
 * calling thread, each query's pruning bound (distance units; 3.39e38 = none) as the pre-pass left it, before the scan.
 * cuvsB200IvfPqPrimedBounds copies up to cap of the last search's (last query batch's) bounds to out and returns their count. */
CUVS_EXPORT void cuvsB200IvfPqKeepPrimedBounds(int on);
CUVS_EXPORT int64_t cuvsB200IvfPqPrimedBounds(float* out, int64_t cap);

/* ---- multi-GPU exchange step (one process per GPU; DESIGN.md §7) ------------------------------------------------
 * The index is sharded by IVF list: every rank searches the lists it owns for the whole query batch and holds a partial
 * top-k [n_queries, k] with GLOBAL ids.  cuvsB200AllGatherMergeTopK enqueues, on the handle's stream, ONE ncclAllGather of
 * the packed partials (n_queries*k*12 bytes per rank) and the k-way merge; the merged result is identical on all ranks.
 * No host synchronisation.  Bootstrap: rank 0 calls cuvsB200NcclUniqueId, the 128 bytes travel to the other ranks by any
 * means (torch.distributed broadcast, MPI, a file), every rank calls cuvsB200CommCreate.  NCCL is dlopen'ed on first use. */
typedef struct cuvsB200Comm* cuvsB200Comm_t;
CUVS_EXPORT cuvsError_t cuvsB200NcclUniqueId(void* id128);
CUVS_EXPORT cuvsError_t cuvsB200CommCreate(cuvsResources_t res, const void* id128, int rank, int world, cuvsB200Comm_t* comm);
CUVS_EXPORT cuvsError_t cuvsB200CommDestroy(cuvsB200Comm_t comm);
CUVS_EXPORT cuvsError_t cuvsB200AllGatherMergeTopK(cuvsResources_t res,
                                                   cuvsB200Comm_t comm,
                                                   DLManagedTensor* distances,     /* [n_queries, k] f32, this rank's partial */
                                                   DLManagedTensor* neighbors,     /* [n_queries, k] i64, global ids */
                                                   DLManagedTensor* out_distances, /* [n_queries, k] f32 */
                                                   DLManagedTensor* out_neighbors, /* [n_queries, k] i64 */
                                                   bool select_min);

/* CAGRA: the graph walk is bound by random row gathers from HBM.  bits = 16 makes the index keep an fp16 copy of the
 * vectors that the walk reads instead (half the bytes); the best 32 entries of every query's final list are re-ranked
 * with the fp32 rows before the k results are returned (k <= 32).  bits = 32 (default) restores the exact fp32 walk.
 * This is for float32 indexes.  An index keeps its rows in the element type it was given, so a float16 index is walked
 * as it is stored, at any k and with nothing wider to re-rank with: 16 and 32 both succeed and change nothing.  On an
 * int8 / uint8 index 32 succeeds and changes nothing, and 16 is refused (the rows are already narrower than fp16). */
CUVS_EXPORT cuvsError_t cuvsB200CagraSetWalkPrecision(cuvsResources_t res, cuvsCagraIndex_t index, int bits);

#ifdef __cplusplus
}
#endif
