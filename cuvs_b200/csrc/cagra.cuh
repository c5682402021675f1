// CAGRA index state and the host entry points that cagra.cu (walk, build, index files, C boundary) shares with
// cagra_extend.cu (adding rows to an index).
#pragma once
#include "common.hpp"
#include <cuda_fp16.h>

#include <cuvs/neighbors/cagra.h>

namespace b200 {

struct cagra_index {
  int device              = 0;
  cuvsDistanceType metric = L2Expanded;
  int64_t n               = 0;
  int dim                 = 0;
  row_type type           = row_type::f32;  // element type of the rows
  int ld                  = 0;  // row pitch in elements (rows padded to 16 bytes, cagra.hpp:610)
  int degree              = 0;
  const void* data        = nullptr;  // rows in the element type they were given in; a view of the caller's buffer or data_own
  const uint32_t* graph   = nullptr;
  owned<unsigned char> data_own;
  owned<uint32_t> graph_own;
  const float* rows_f32() const { return static_cast<const float*>(data); }  // float32 indexes only
  // float32 indexes only: optional fp16 copy of the vectors for the walk (cuvsB200CagraSetWalkPrecision): the walk is bound
  // by random row gathers from HBM, half-width rows halve its bytes; the returned neighbours are re-ranked with the fp32 rows.
  owned<__half> data16;
  int ld16 = 0;  // row pitch in halves (rows padded to 16 bytes)
  // CosineExpanded only: 1 / |x_i| of the rows (0 for a zero row), recomputed whenever the rows are set or loaded
  // (cagra.hpp:580-680 keeps dataset norms the same way).  The rows themselves stay as given.
  owned<float> inv_norm;
};

/** The graph walk over `nq` fp32 queries (device), the algorithm chosen by `sp.algo` (AUTO as cuvsCagraSearch). */
void cagra_search(resources* res, const cagra_index& idx, const cuvsCagraSearchParams& sp, const float* queries, int64_t nq, int k,
                  uint32_t* out32, int64_t* out64, float* out_dist, const uint32_t* keep_bits = nullptr, int64_t n_bits = 0);
/** Cosine: (re)computes inv_norm from the rows; other metrics keep none. */
void set_inv_norms(resources* r, cagra_index& idx);
/** float32 indexes: (re)computes the fp16 walk copy data16 from the rows. */
void set_half_rows(resources* r, cagra_index& idx);

}  // namespace b200
