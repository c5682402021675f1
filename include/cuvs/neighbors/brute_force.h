/*
 * Exact kNN ("brute force") C boundary.
 * Replaces c/include/cuvs/neighbors/brute_force.h: index handle :28-33,
 * Create/Destroy :41/:48, Build :94, Search :150, Serialize/Deserialize :186/:213.
 *
 * Path behind cuvsBruteForceSearch (cuvs_b200/csrc/brute_force.cu):
 * split-bf16 Q.D^T on wgmma (sm_90a) with the |x|^2 term folded into the K extension,
 * a per-row register top-k' epilogue from the register accumulators, exact fp32
 * re-scoring of the k' candidates and a certificate check (DESIGN.md §3).
 */
#pragma once
#include <cuvs/core/c_api.h>
#include <cuvs/core/export.h>
#include <cuvs/distance/distance.h>
#include <cuvs/neighbors/common.h>
#include <dlpack/dlpack.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
  uintptr_t addr;   /* heap object owned by the library */
  DLDataType dtype; /* dtype the index was built from */
} cuvsBruteForceIndex;
typedef cuvsBruteForceIndex* cuvsBruteForceIndex_t;

CUVS_EXPORT cuvsError_t cuvsBruteForceIndexCreate(cuvsBruteForceIndex_t* index);
CUVS_EXPORT cuvsError_t cuvsBruteForceIndexDestroy(cuvsBruteForceIndex_t index);

/* dataset: [n, dim] float32, float16, int8 or uint8, host or device, C- or F-contiguous.  A float32 dataset that is
 * C-contiguous in device memory is viewed, not copied, and must outlive the index.  float16, int8 and uint8 rows are copied
 * into the index and kept in their own type (into the scan's zero-padded layout where the scan reads them), even when they
 * are in device memory. */
CUVS_EXPORT cuvsError_t cuvsBruteForceBuild(cuvsResources_t res,
                                            DLManagedTensor* dataset,
                                            cuvsDistanceType metric,
                                            float metric_arg,
                                            cuvsBruteForceIndex_t index);

/* queries [nq, dim] device, of the index's own type (a float16 index also takes float32 queries);
 * neighbors [nq, k] int64; distances [nq, k] f32. */
CUVS_EXPORT cuvsError_t cuvsBruteForceSearch(cuvsResources_t res,
                                             cuvsBruteForceIndex_t index,
                                             DLManagedTensor* queries,
                                             DLManagedTensor* neighbors,
                                             DLManagedTensor* distances,
                                             cuvsFilter prefilter);

CUVS_EXPORT cuvsError_t cuvsBruteForceSerialize(cuvsResources_t res,
                                                const char* filename,
                                                cuvsBruteForceIndex_t index);
CUVS_EXPORT cuvsError_t cuvsBruteForceDeserialize(cuvsResources_t res,
                                                  const char* filename,
                                                  cuvsBruteForceIndex_t index);
#ifdef __cplusplus
}
#endif
