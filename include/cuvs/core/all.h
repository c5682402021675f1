/* Umbrella include for the part of the cuVS C ABI this library implements
 * (reference: c/include/cuvs/core/all.h).  Headers outside the scan+top-k hot
 * path and the scalar and binary quantizers (hnsw, vamana, ivf_sq,
 * tiered_index, pca, the product quantizer) are intentionally absent — see
 * DESIGN.md "out of scope". */
#pragma once
#include <cuvs/cluster/kmeans.h>
#include <cuvs/core/c_api.h>
#include <cuvs/distance/distance.h>
#include <cuvs/distance/pairwise_distance.h>
#include <cuvs/neighbors/brute_force.h>
#include <cuvs/neighbors/cagra.h>
#include <cuvs/neighbors/common.h>
#include <cuvs/neighbors/ivf_flat.h>
#include <cuvs/neighbors/ivf_pq.h>
#include <cuvs/neighbors/mg_common.h>
#include <cuvs/neighbors/mg_ivf_flat.h>
#include <cuvs/neighbors/nn_descent.h>
#include <cuvs/neighbors/refine.h>
#include <cuvs/preprocessing/quantize/binary.h>
#include <cuvs/preprocessing/quantize/scalar.h>
#include <cuvs/selection/select_k.h>
