// Single-process multi-GPU IVF-Flat (cuvsMultiGpuIvfFlat*) and dense pairwise distance.
//
// Reference: cpp/src/neighbors/mg/snmg.cuh:92-707 (replicated / row-sharded index, OpenMP thread per GPU, ncclSend/ncclRecv
// of the partials to a root + knn_merge_parts on the root, results through the host), c/src/neighbors/mg_ivf_flat.cpp.
// Same C contract (HOST dataset / queries / outputs, handle from cuvsMultiGpuResourcesCreate), data plan:
//   SHARDED     the index is sharded by IVF LIST (BASELINE north_star): one set of coarse centres trained on device 0 and
//               installed on every device, list l lives on device l % n_devices with GLOBAL row ids; a search sends the
//               whole query batch to every device, each scans the probed lists it owns, and the partial top-k are
//               exchanged by ONE grouped ncclAllGather over NVLink (comm.cu) and merged on device 0 — no host merge,
//               no id translation, one D2H of the final [nq, k] result.
//   REPLICATED  every device holds the full index; the query batch is split across devices (no exchange step).
#include "comm.cuh"
#include "common.hpp"
#include "exact.cuh"
#include "timing.hpp"

#include <cuvs/cluster/kmeans.h>
#include <cuvs/distance/pairwise_distance.h>
#include <cuvs/neighbors/mg_ivf_flat.h>
#include <cuvs_b200/ext.h>

#include <algorithm>
#include <cfloat>
#include <memory>
#include <vector>

namespace b200 {
namespace {

struct mg_shard {
  int device = 0;
  cuvsResources_t res = 0;
  cuvsIvfFlatIndex_t index = nullptr;
  int64_t row0 = 0, rows = 0;
};

struct mg_index {
  cuvsMultiGpuDistributionMode mode = CUVS_NEIGHBORS_MG_SHARDED;
  cuvsDistanceType metric = L2Expanded;
  int dim = 0;
  std::vector<mg_shard> shards;
  comm_group* comm = nullptr;  // SHARDED: NCCL communicators over the handle's devices
  ~mg_index()
  {
    if (comm) destroy_comm_group(comm);
    int cur = 0;
    cudaGetDevice(&cur);
    for (auto& s : shards) {
      cudaSetDevice(s.device);
      if (s.index) cuvsIvfFlatIndexDestroy(s.index);
      if (s.res) cuvsResourcesDestroy(s.res);
    }
    cudaSetDevice(cur);
  }
};

struct device_guard {
  int prev = 0;
  explicit device_guard(int d) { cudaGetDevice(&prev); cudaSetDevice(d); }
  ~device_guard() { cudaSetDevice(prev); }
};

void check_c(cuvsError_t e, const char* what)
{
  if (e != CUVS_SUCCESS) {
    const char* t = cuvsGetLastErrorText();
    std::string msg = t ? t : "unknown error";
    B2_FAIL("%s: %s", what, msg.c_str());
  }
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

cuvsError_t cuvsMultiGpuIvfFlatIndexParamsCreate(cuvsMultiGpuIvfFlatIndexParams_t* index_params)
{
  return guarded([=] {
    cuvsIvfFlatIndexParams_t base;
    check_c(cuvsIvfFlatIndexParamsCreate(&base), "cuvsIvfFlatIndexParamsCreate");
    *index_params = new cuvsMultiGpuIvfFlatIndexParams{base, CUVS_NEIGHBORS_MG_SHARDED};
  });
}
cuvsError_t cuvsMultiGpuIvfFlatIndexParamsDestroy(cuvsMultiGpuIvfFlatIndexParams_t p)
{
  return guarded([=] { if (p) { cuvsIvfFlatIndexParamsDestroy(p->base_params); delete p; } });
}
cuvsError_t cuvsMultiGpuIvfFlatSearchParamsCreate(cuvsMultiGpuIvfFlatSearchParams_t* params)
{
  return guarded([=] {
    cuvsIvfFlatSearchParams_t base;
    check_c(cuvsIvfFlatSearchParamsCreate(&base), "cuvsIvfFlatSearchParamsCreate");
    *params = new cuvsMultiGpuIvfFlatSearchParams{base, CUVS_NEIGHBORS_MG_LOAD_BALANCER, CUVS_NEIGHBORS_MG_TREE_MERGE, 1LL << 20};
  });
}
cuvsError_t cuvsMultiGpuIvfFlatSearchParamsDestroy(cuvsMultiGpuIvfFlatSearchParams_t p)
{
  return guarded([=] { if (p) { cuvsIvfFlatSearchParamsDestroy(p->base_params); delete p; } });
}
cuvsError_t cuvsMultiGpuIvfFlatIndexCreate(cuvsMultiGpuIvfFlatIndex_t* index)
{
  return guarded([=] { *index = new cuvsMultiGpuIvfFlatIndex{}; });
}
cuvsError_t cuvsMultiGpuIvfFlatIndexDestroy(cuvsMultiGpuIvfFlatIndex_t index)
{
  return guarded([=] {
    if (!index) return;
    drop_index<mg_index>(index);
    delete index;
  });
}

cuvsError_t cuvsMultiGpuIvfFlatBuild(cuvsResources_t res, cuvsMultiGpuIvfFlatIndexParams_t params, DLManagedTensor* dataset_tensor,
                                     cuvsMultiGpuIvfFlatIndex_t index)
{
  return guarded([=] {
    auto r = as_res(res);
    B2_EXPECTS(params && dataset_tensor && index, "null argument");
    B2_EXPECTS(!r->mg_devices.empty(), "cuvsMultiGpuIvfFlatBuild needs a handle from cuvsMultiGpuResourcesCreate");
    const DLTensor& ds = dataset_tensor->dl_tensor;
    B2_EXPECTS(dl_is(ds, kDLFloat, 32) && ds.ndim == 2 && dl_is_c_contiguous(ds), "dataset must be a row-major float32 matrix");
    B2_EXPECTS(dl_is_host(ds), "multi-GPU build requires the dataset in host memory");
    auto mg     = std::make_unique<mg_index>();
    mg->mode    = params->mode;
    mg->metric  = params->base_params->metric;
    mg->dim     = static_cast<int>(ds.shape[1]);
    const int64_t n = ds.shape[0];
    const int d     = mg->dim;
    const int nd    = static_cast<int>(r->mg_devices.size());
    const float* x  = dl_ptr<float>(ds);
    const bool sharded = mg->mode == CUVS_NEIGHBORS_MG_SHARDED && nd > 1;
    for (int i = 0; i < nd; ++i) {
      mg_shard sh;
      sh.device = r->mg_devices[i];
      sh.row0   = 0;
      sh.rows   = n;
      device_guard g(sh.device);
      check_c(cuvsResourcesCreate(&sh.res), "cuvsResourcesCreate");
      check_c(cuvsStreamSet(sh.res, r->mg_streams[i]), "cuvsStreamSet");
      check_c(cuvsIvfFlatIndexCreate(&sh.index), "cuvsIvfFlatIndexCreate");
      mg->shards.push_back(sh);
    }
    cuvsIvfFlatIndexParams p = *params->base_params;
    p.n_lists                = static_cast<uint32_t>(std::max<int64_t>(1, std::min<int64_t>(p.n_lists, n)));
    if (!sharded) {
      // REPLICATED (or a single device): the full index on every device
      for (int i = 0; i < nd; ++i) {
        device_guard g(mg->shards[i].device);
        dl_view full(x, DLDevice{kDLCPU, 0}, ds.dtype, n, d);
        check_c(cuvsIvfFlatBuild(mg->shards[i].res, &p, &full.m, mg->shards[i].index), "cuvsIvfFlatBuild (replica)");
      }
    } else {
      // SHARDED by IVF list.  (1) train the coarse centres once, on device 0, on the build's usual subsample.
      cuvsIvfFlatIndexParams p0 = p;
      p0.add_data_on_build      = false;
      std::vector<float> centers(static_cast<size_t>(p.n_lists) * d);
      {
        device_guard g(mg->shards[0].device);
        dl_view full(x, DLDevice{kDLCPU, 0}, ds.dtype, n, d);
        check_c(cuvsIvfFlatBuild(mg->shards[0].res, &p0, &full.m, mg->shards[0].index), "cuvsIvfFlatBuild (train)");
        DLManagedTensor cv{};
        check_c(cuvsIvfFlatIndexGetCenters(mg->shards[0].index, &cv), "cuvsIvfFlatIndexGetCenters");
        B2_CUDA(cudaMemcpyAsync(centers.data(), cv.dl_tensor.data, centers.size() * sizeof(float), cudaMemcpyDeviceToHost, r->mg_streams[0]));
        B2_CUDA(cudaStreamSynchronize(r->mg_streams[0]));
      }
      // (2) every other device: an empty index with the SAME centres (bit-identical partition rule everywhere)
      for (int i = 1; i < nd; ++i) {
        device_guard g(mg->shards[i].device);
        dl_view seed(centers.data(), DLDevice{kDLCPU, 0}, ds.dtype, p.n_lists, d);
        cuvsIvfFlatIndexParams pi = p0;
        pi.kmeans_n_iters           = 1;
        pi.kmeans_trainset_fraction = 1.0;
        check_c(cuvsIvfFlatBuild(mg->shards[i].res, &pi, &seed.m, mg->shards[i].index), "cuvsIvfFlatBuild (empty shard)");
        check_c(cuvsB200IvfFlatSetCenters(mg->shards[i].res, mg->shards[i].index, &seed.m), "cuvsB200IvfFlatSetCenters");
      }
      // (3) label the rows chunk by chunk on device 0 and route every row to the owner of its list (list % n_devices)
      //     with its GLOBAL row id
      cuvsKMeansParams_t kp;
      check_c(cuvsKMeansParamsCreate(&kp), "cuvsKMeansParamsCreate");
      kp->n_clusters = static_cast<int>(p.n_lists);
      kp->metric     = mg->metric == InnerProduct ? InnerProduct : L2Expanded;
      const int64_t chunk = std::max<int64_t>(1, (int64_t(1) << 26) / d);  // 256 MiB of rows per step
      std::vector<int> labels(static_cast<size_t>(std::min(chunk, n)));
      std::vector<std::vector<float>> rows_of(nd);
      std::vector<std::vector<int64_t>> ids_of(nd);
      float *d_x = nullptr, *d_c = nullptr;
      int* d_l = nullptr;
      {
        device_guard g(mg->shards[0].device);
        auto st = r->mg_streams[0];
        B2_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&d_x), sizeof(float) * std::min(chunk, n) * d, st));
        B2_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&d_c), sizeof(float) * centers.size(), st));
        B2_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&d_l), sizeof(int) * std::min(chunk, n), st));
        B2_CUDA(cudaMemcpyAsync(d_c, centers.data(), sizeof(float) * centers.size(), cudaMemcpyHostToDevice, st));
      }
      for (int64_t r0 = 0; r0 < n; r0 += chunk) {
        const int64_t rows = std::min(chunk, n - r0);
        {
          device_guard g(mg->shards[0].device);
          auto st = r->mg_streams[0];
          B2_CUDA(cudaMemcpyAsync(d_x, x + r0 * d, sizeof(float) * rows * d, cudaMemcpyHostToDevice, st));
          const DLDevice dev{kDLCUDA, mg->shards[0].device};
          dl_view tx(d_x, dev, DLDataType{kDLFloat, 32, 1}, rows, d), tc(d_c, dev, DLDataType{kDLFloat, 32, 1}, p.n_lists, d);
          dl_view tl(d_l, dev, DLDataType{kDLInt, 32, 1}, rows);
          double inertia = 0;
          check_c(cuvsKMeansPredict(mg->shards[0].res, kp, &tx.m, nullptr, &tc.m, &tl.m, false, &inertia), "cuvsKMeansPredict (routing)");
          B2_CUDA(cudaMemcpyAsync(labels.data(), d_l, sizeof(int) * rows, cudaMemcpyDeviceToHost, st));
          B2_CUDA(cudaStreamSynchronize(st));
        }
        for (int i = 0; i < nd; ++i) { rows_of[i].clear(); ids_of[i].clear(); }
        for (int64_t j = 0; j < rows; ++j) {
          const int owner = labels[j] % nd;
          rows_of[owner].insert(rows_of[owner].end(), x + (r0 + j) * d, x + (r0 + j + 1) * d);
          ids_of[owner].push_back(r0 + j);
        }
        for (int i = 0; i < nd; ++i) {
          const int64_t m = static_cast<int64_t>(ids_of[i].size());
          if (m == 0) continue;
          device_guard g(mg->shards[i].device);
          auto st = r->mg_streams[i];
          float* dv = nullptr;
          int64_t* di = nullptr;
          B2_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&dv), sizeof(float) * m * d, st));
          B2_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&di), sizeof(int64_t) * m, st));
          B2_CUDA(cudaMemcpyAsync(dv, rows_of[i].data(), sizeof(float) * m * d, cudaMemcpyHostToDevice, st));
          B2_CUDA(cudaMemcpyAsync(di, ids_of[i].data(), sizeof(int64_t) * m, cudaMemcpyHostToDevice, st));
          dl_view tv(dv, DLDevice{kDLCUDA, mg->shards[i].device}, DLDataType{kDLFloat, 32, 1}, m, d);
          dl_view ti(di, DLDevice{kDLCUDA, mg->shards[i].device}, DLDataType{kDLInt, 64, 1}, m);
          check_c(cuvsIvfFlatExtend(mg->shards[i].res, &tv.m, &ti.m, mg->shards[i].index), "cuvsIvfFlatExtend (shard)");
          B2_CUDA(cudaFreeAsync(dv, st));
          B2_CUDA(cudaFreeAsync(di, st));
          B2_CUDA(cudaStreamSynchronize(st));  // the host staging vectors are reused by the next chunk
        }
      }
      {
        device_guard g(mg->shards[0].device);
        auto st = r->mg_streams[0];
        B2_CUDA(cudaFreeAsync(d_x, st));
        B2_CUDA(cudaFreeAsync(d_c, st));
        B2_CUDA(cudaFreeAsync(d_l, st));
      }
      check_c(cuvsKMeansParamsDestroy(kp), "cuvsKMeansParamsDestroy");
      mg->comm = make_local_comm_group(r->mg_devices);
    }
    set_index(index, mg.release(), ds.dtype);
  });
}

cuvsError_t cuvsMultiGpuIvfFlatSearch(cuvsResources_t res, cuvsMultiGpuIvfFlatSearchParams_t params, cuvsMultiGpuIvfFlatIndex_t index,
                                      DLManagedTensor* queries_tensor, DLManagedTensor* neighbors_tensor, DLManagedTensor* distances_tensor)
{
  return guarded([=] {
    as_res(res);
    B2_EXPECTS(params && queries_tensor && neighbors_tensor && distances_tensor, "null argument");
    auto& mg = index_of<mg_index>(index);
    const DLTensor& q  = queries_tensor->dl_tensor;
    const DLTensor& nb = neighbors_tensor->dl_tensor;
    const DLTensor& dd = distances_tensor->dl_tensor;
    B2_EXPECTS(dl_is_host(q) && dl_is_host(nb) && dl_is_host(dd), "multi-GPU search takes host queries / neighbors / distances");
    B2_EXPECTS(dl_is(q, kDLFloat, 32) && dl_is(nb, kDLInt, 64) && dl_is(dd, kDLFloat, 32), "queries f32, neighbors int64, distances f32 expected");
    const int64_t nq = q.shape[0];
    const int k      = static_cast<int>(nb.shape[1]);
    const int ns     = static_cast<int>(mg.shards.size());
    const bool select_min = mg.metric != InnerProduct;
    const bool sharded    = mg.comm != nullptr;
    struct part { float* dq = nullptr; int64_t* di = nullptr; float* dv = nullptr; int64_t q0 = 0, qn = 0; cudaStream_t st = nullptr; };
    std::vector<part> parts(ns);
    int64_t* out_i = dl_ptr<int64_t>(nb);
    float* out_v   = dl_ptr<float>(dd);
    // every device: queries in (the whole batch when sharded, a slice when replicated), local search on its own stream
    for (int s = 0; s < ns; ++s) {
      auto& sh = mg.shards[s];
      auto& pt = parts[s];
      if (sharded) { pt.q0 = 0; pt.qn = nq; }
      else { pt.q0 = nq * s / ns; pt.qn = nq * (s + 1) / ns - pt.q0; }
      device_guard g(sh.device);
      check_c(cuvsStreamGet(sh.res, &pt.st), "cuvsStreamGet");
      if (pt.qn == 0) continue;
      B2_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&pt.dq), sizeof(float) * pt.qn * mg.dim, pt.st));
      B2_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&pt.di), sizeof(int64_t) * pt.qn * k, pt.st));
      B2_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&pt.dv), sizeof(float) * pt.qn * k, pt.st));
      B2_CUDA(cudaMemcpyAsync(pt.dq, dl_ptr<float>(q) + pt.q0 * mg.dim, sizeof(float) * pt.qn * mg.dim, cudaMemcpyHostToDevice, pt.st));
      const DLDevice dev{kDLCUDA, sh.device};
      dl_view tq(pt.dq, dev, DLDataType{kDLFloat, 32, 1}, pt.qn, mg.dim), ti(pt.di, dev, DLDataType{kDLInt, 64, 1}, pt.qn, k),
          tv(pt.dv, dev, DLDataType{kDLFloat, 32, 1}, pt.qn, k);
      check_c(cuvsIvfFlatSearch(sh.res, params->base_params, sh.index, &tq.m, &ti.m, &tv.m, cuvsFilter{0, NO_FILTER}), "cuvsIvfFlatSearch (shard)");
      if (!sharded) {
        B2_CUDA(cudaMemcpyAsync(out_i + pt.q0 * k, pt.di, sizeof(int64_t) * pt.qn * k, cudaMemcpyDeviceToHost, pt.st));
        B2_CUDA(cudaMemcpyAsync(out_v + pt.q0 * k, pt.dv, sizeof(float) * pt.qn * k, cudaMemcpyDeviceToHost, pt.st));
      }
    }
    if (sharded && nq > 0) {
      // the one exchange step: grouped ncclAllGather of the packed partial top-k over NVLink, k-way merge on device 0
      std::vector<cudaStream_t> streams(ns);
      std::vector<const float*> pd(ns);
      std::vector<const int64_t*> pi(ns);
      std::vector<float*> od(ns, nullptr);
      std::vector<int64_t*> oi(ns, nullptr);
      for (int s = 0; s < ns; ++s) { streams[s] = parts[s].st; pd[s] = parts[s].dv; pi[s] = parts[s].di; }
      float* m_v   = nullptr;
      int64_t* m_i = nullptr;
      {
        device_guard g(mg.shards[0].device);
        B2_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&m_v), sizeof(float) * nq * k, parts[0].st));
        B2_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&m_i), sizeof(int64_t) * nq * k, parts[0].st));
      }
      od[0] = m_v;
      oi[0] = m_i;
      allgather_merge_topk_all(*mg.comm, streams, pd, pi, nq, k, select_min, od, oi, 0);
      device_guard g(mg.shards[0].device);
      B2_CUDA(cudaMemcpyAsync(out_i, m_i, sizeof(int64_t) * nq * k, cudaMemcpyDeviceToHost, parts[0].st));
      B2_CUDA(cudaMemcpyAsync(out_v, m_v, sizeof(float) * nq * k, cudaMemcpyDeviceToHost, parts[0].st));
      B2_CUDA(cudaFreeAsync(m_v, parts[0].st));
      B2_CUDA(cudaFreeAsync(m_i, parts[0].st));
    }
    for (int s = 0; s < ns; ++s) {
      device_guard g(mg.shards[s].device);
      auto& pt = parts[s];
      if (pt.dq) B2_CUDA(cudaFreeAsync(pt.dq, pt.st));
      if (pt.di) B2_CUDA(cudaFreeAsync(pt.di, pt.st));
      if (pt.dv) B2_CUDA(cudaFreeAsync(pt.dv, pt.st));
      check_c(cuvsStreamSync(mg.shards[s].res), "cuvsStreamSync");  // host outputs are complete when the call returns
    }
  });
}

cuvsError_t cuvsMultiGpuIvfFlatExtend(cuvsResources_t, cuvsMultiGpuIvfFlatIndex_t, DLManagedTensor*, DLManagedTensor*)
{
  return guarded([=] { B2_FAIL("cuvsMultiGpuIvfFlatExtend is not implemented in this build (use the per-shard cuvsIvfFlatExtend through cuvs_b200.distributed)"); });
}
cuvsError_t cuvsMultiGpuIvfFlatSerialize(cuvsResources_t, cuvsMultiGpuIvfFlatIndex_t, const char*)
{
  return guarded([=] { B2_FAIL("cuvsMultiGpuIvfFlatSerialize is not implemented in this build"); });
}
cuvsError_t cuvsMultiGpuIvfFlatDeserialize(cuvsResources_t, const char*, cuvsMultiGpuIvfFlatIndex_t)
{
  return guarded([=] { B2_FAIL("cuvsMultiGpuIvfFlatDeserialize is not implemented in this build"); });
}
cuvsError_t cuvsMultiGpuIvfFlatDistribute(cuvsResources_t, const char*, cuvsMultiGpuIvfFlatIndex_t)
{
  return guarded([=] { B2_FAIL("cuvsMultiGpuIvfFlatDistribute is not implemented in this build"); });
}

// x [m,k], y [n,k] -> dist [m,n]; exact fp32 in the oracle's arithmetic (reference: c/src/distance/pairwise_distance.cpp,
// cpp/src/distance/detail/distance.cuh:308-333).  L2 / inner product / cosine.
cuvsError_t cuvsPairwiseDistance(cuvsResources_t res, DLManagedTensor* x_t, DLManagedTensor* y_t, DLManagedTensor* dist_t,
                                 cuvsDistanceType metric, float /*metric_arg*/)
{
  return guarded([=] {
    auto r = as_res(res);
    B2_EXPECTS(x_t && y_t && dist_t, "null argument");
    const DLTensor& x = x_t->dl_tensor;
    const DLTensor& y = y_t->dl_tensor;
    const DLTensor& d = dist_t->dl_tensor;
    B2_EXPECTS(dl_is_device(x) && dl_is_device(y) && dl_is_device(d), "x, y and dist should have device compatible memory");
    B2_EXPECTS(dl_is(x, kDLFloat, 32) && dl_is(y, kDLFloat, 32) && dl_is(d, kDLFloat, 32), "pairwise_distance: float32 tensors expected");
    B2_EXPECTS(x.ndim == 2 && y.ndim == 2 && d.ndim == 2 && x.shape[1] == y.shape[1] && d.shape[0] == x.shape[0] && d.shape[1] == y.shape[0], "shape mismatch");
    B2_EXPECTS(dl_is_c_contiguous(x) && dl_is_c_contiguous(y) && dl_is_c_contiguous(d), "row-major contiguous tensors expected");
    B2_EXPECTS(metric == L2Expanded || metric == L2SqrtExpanded || metric == L2Unexpanded || metric == L2SqrtUnexpanded || metric == InnerProduct || metric == CosineExpanded,
               "pairwise_distance: metric %d is outside the scan+top-k hot path of this library", int(metric));
    const int64_t m = x.shape[0], n = y.shape[0];
    const int k = static_cast<int>(x.shape[1]);
    auto s = r->stream;
    const bool norms = metric == L2Expanded || metric == L2SqrtExpanded || metric == CosineExpanded;
    dbuf<float> xn, yn;
    if (norms) {
      xn.alloc(static_cast<size_t>(m), s); yn.alloc(static_cast<size_t>(n), s);
      row_norms(s, dl_ptr<float>(x), m, k, k, xn.data());
      row_norms(s, dl_ptr<float>(y), n, k, k, yn.data());
    }
    const int64_t chunk = 65535 * 64;
    for (int64_t r0 = 0; r0 < m; r0 += chunk) {
      int64_t rows = std::min(chunk, m - r0);
      exact_distance_tile(s, dl_ptr<float>(x) + r0 * k, rows, k, dl_ptr<float>(y), n, k, k, norms ? xn.data() + r0 : nullptr,
                          norms ? yn.data() : nullptr, metric, dl_ptr<float>(d) + r0 * n, n, filter_view{}, 0);
    }
    postprocess_distances(s, dl_ptr<float>(d), m * n, metric);
  });
}

}  // extern "C"
