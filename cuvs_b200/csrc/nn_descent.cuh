// NN-descent kNN graph construction (nn_descent.cu), shared with CAGRA's build (build_algo = NN_DESCENT).
#pragma once
#include "common.hpp"

namespace b200 {

/**
 * The NN-descent graph of n device rows (element type `rt`; row pitch `ld` elements).
 * Writes the `degree` best neighbours of every row, exactly re-scored, to graph [n, degree] (device), and their
 * post-processed exact distances to dist [n, degree] (device) when it is not null.  `intermediate` is the list length kept
 * while iterating (raised to `degree` and rounded up to a multiple of 32); `dist_comp` a cuvsNNDescentDistCompDtype.
 */
void nn_descent_graph(resources* r, const void* rows, row_type rt, int64_t n, int dim, int64_t ld, cuvsDistanceType metric, int degree,
                      int intermediate, int max_iterations, float termination_threshold, int dist_comp, uint32_t* graph, float* dist);

}  // namespace b200
