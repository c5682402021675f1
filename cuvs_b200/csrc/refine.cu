// Exact re-ranking of ANN candidates (cuvsRefine).
// Reference: cpp/src/neighbors/refine/refine_device.cuh:30-130 (re-uses the IVF-Flat scan over a fake
// one-list-per-query index), c/src/neighbors/refine.cpp.  Here: one warp per query (up to 256 candidates; one CTA per query
// up to 2048) gathers its candidates' rows and scores them in fp32 (oracle arithmetic), then ranks by (distance, id) —
// exact.cu.
#include "common.hpp"
#include "exact.cuh"
#include "timing.hpp"

#include <cuvs/neighbors/refine.h>

namespace b200 {
namespace {
__global__ void ids_to_pos_kernel(const int64_t* __restrict__ ids, int64_t count, int64_t n, uint32_t* __restrict__ pos)
{
  int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= count) return;
  int64_t v = ids[i];
  pos[i]    = (v >= 0 && v < n) ? static_cast<uint32_t>(v) : 0xffffffffu;
}
}  // namespace
}  // namespace b200

using namespace b200;

extern "C" cuvsError_t cuvsRefine(cuvsResources_t res, DLManagedTensor* dataset_t, DLManagedTensor* queries_t,
                                  DLManagedTensor* candidates_t, cuvsDistanceType metric, DLManagedTensor* indices_t,
                                  DLManagedTensor* distances_t)
{
  return guarded([=] {
    auto r = as_res(res);
    B2_EXPECTS(dataset_t && queries_t && candidates_t && indices_t && distances_t, "null argument");
    const DLTensor& ds = dataset_t->dl_tensor;
    const DLTensor& q  = queries_t->dl_tensor;
    const DLTensor& c  = candidates_t->dl_tensor;
    const DLTensor& oi = indices_t->dl_tensor;
    const DLTensor& od = distances_t->dl_tensor;
    B2_EXPECTS(dl_is_device(ds) && dl_is_device(q) && dl_is_device(c) && dl_is_device(oi) && dl_is_device(od),
               "refine: this build implements the device path only (all tensors must be device accessible)");
    B2_EXPECTS(dl_is(ds, kDLFloat, 32) && dl_is(q, kDLFloat, 32), "refine: dataset/queries must be float32");
    B2_EXPECTS(dl_is(c, kDLInt, 64) && dl_is(oi, kDLInt, 64), "refine: candidates/indices must be int64");
    B2_EXPECTS(dl_is(od, kDLFloat, 32), "refine: distances must be float32");
    B2_EXPECTS(ds.ndim == 2 && q.ndim == 2 && c.ndim == 2 && oi.ndim == 2 && od.ndim == 2, "refine: 2-D tensors expected");
    B2_EXPECTS(dl_is_c_contiguous(ds) && dl_is_c_contiguous(q) && dl_is_c_contiguous(c) && dl_is_c_contiguous(oi) && dl_is_c_contiguous(od),
               "refine: tensors must be row-major contiguous");
    const int64_t n = ds.shape[0], nq = q.shape[0];
    const int d = static_cast<int>(ds.shape[1]), n_cand = static_cast<int>(c.shape[1]), k = static_cast<int>(oi.shape[1]);
    B2_EXPECTS(q.shape[1] == d && c.shape[0] == nq && oi.shape[0] == nq && od.shape[0] == nq && od.shape[1] == k, "refine: shape mismatch");
    B2_EXPECTS(k <= n_cand, "refine: k (%d) must not exceed the number of candidates (%d)", k, n_cand);
    B2_EXPECTS(n_cand <= 2048, "refine: at most 2048 candidates per query are supported (got %d)", n_cand);
    B2_EXPECTS(n < (int64_t(1) << 32) - 1, "refine: dataset too large");
    if (nq == 0) return;
    auto s = r->stream;
    dbuf<uint32_t> pos(static_cast<size_t>(nq) * n_cand, s);
    count_launch();
    ids_to_pos_kernel<<<static_cast<unsigned>((nq * n_cand + 255) / 256), 256, 0, s>>>(dl_ptr<int64_t>(c), nq * n_cand, n, pos.data());
    B2_CUDA(cudaGetLastError());
    cuvsDistanceType fine = metric;
    if (metric == L2Expanded) fine = L2Unexpanded;          // refine_device.cuh scores with the fine-scan arithmetic
    if (metric == L2SqrtExpanded) fine = L2SqrtUnexpanded;
    const bool need_norms = fine == CosineExpanded;
    dbuf<float> qn, xn;
    if (need_norms) {
      qn.alloc(static_cast<size_t>(nq), s);
      xn.alloc(static_cast<size_t>(n), s);
      row_norms(s, dl_ptr<float>(q), nq, d, d, qn.data());
      row_norms(s, dl_ptr<float>(ds), n, d, d, xn.data());
    }
    timed_section ts("refine", s);
    rescore_topk(s, dl_ptr<float>(q), nq, d, dl_ptr<float>(ds), d, d, need_norms ? qn.data() : nullptr, need_norms ? xn.data() : nullptr,
                 fine, pos.data(), n_cand, nullptr, k, dl_ptr<int64_t>(oi), dl_ptr<float>(od), -1);
    postprocess_distances(s, dl_ptr<float>(od), nq * k, fine);
  });
}
