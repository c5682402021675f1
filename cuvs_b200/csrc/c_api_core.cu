// Core C boundary: errors, logging, resources, allocation, matrix copy.
// Same observable behaviour as the reference's c/src/core/c_api.cpp (:30-380), implemented on the
// CUDA runtime only: the per-thread default stream is the handle's initial stream (the reference
// is built with CUDA_API_PER_THREAD_DEFAULT_STREAM, cpp/cmake/modules/ConfigureCUDA.cmake:44-46),
// temporary memory comes from the device's stream-ordered pool (cudaMallocAsync) whose release
// threshold is lifted so that search calls stop hitting the driver after warm-up.
#include "common.hpp"
#include "timing.hpp"

#include <cuda_fp16.h>

#include <atomic>
#include <cstring>
#include <string>
#include <type_traits>

namespace b200 {

template <typename T>
__global__ void widen_kernel(const T* __restrict__ in, int64_t n, float* __restrict__ out)
{
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i < n) out[i] = static_cast<float>(in[i]);
}

void widen_async(cudaStream_t s, const void* in, DLDataType dt, int64_t count, float* out)
{
  const row_type rt = row_type_of(dt);
  B2_EXPECTS(rt != row_type::f32, "widen_async: the rows are float32 already");
  if (count == 0) return;
  const unsigned grid = static_cast<unsigned>((count + 255) / 256);
  count_launch();
  with_row_type(rt, [&](auto t) {
    using T = decltype(t);
    if constexpr (!std::is_same_v<T, float>) widen_kernel<T><<<grid, 256, 0, s>>>(static_cast<const T*>(in), count, out);
  });
  B2_CUDA(cudaGetLastError());
}

static void alloc_on(owned<float>& b, size_t count, cudaStream_t) { b.alloc(count); }
static void alloc_on(dbuf<float>& b, size_t count, cudaStream_t s) { b.alloc(count, s); }

template <typename Buf>
static void widen_into(resources* res, const DLTensor& src, f32_widened<Buf>& out)
{
  B2_EXPECTS(src.ndim == 2 && dl_is_c_contiguous(src), "matrix must be a row-major 2-D tensor");
  B2_EXPECTS(dl_is_dataset_dtype(src), "Unsupported DLtensor dtype: %d and bits: %d", src.dtype.code, src.dtype.bits);
  out.t        = src;
  out.shape[0] = src.shape[0];
  out.shape[1] = src.shape[1];
  out.t.shape  = out.shape;
  out.t.strides = nullptr;
  if (dl_is(src, kDLFloat, 32)) return;
  const int64_t count = src.shape[0] * src.shape[1];
  const size_t esize  = src.dtype.bits / 8;
  auto s              = res->stream;
  alloc_on(out.own, static_cast<size_t>(std::max<int64_t>(count, 1)), s);
  const void* in = dl_ptr<char>(src);
  dbuf<uint8_t> stage;
  const bool dev = dl_is_device(src) && src.device.device_type != kDLCUDAHost;
  if (!dev && count) {
    stage.alloc(static_cast<size_t>(count) * esize, s);
    B2_CUDA(cudaMemcpyAsync(stage.data(), in, static_cast<size_t>(count) * esize, cudaMemcpyHostToDevice, s));
    in = stage.data();
  }
  widen_async(s, in, src.dtype, count, out.own.data());
  out.t.data        = out.own.data();
  out.t.byte_offset = 0;
  out.t.dtype       = DLDataType{kDLFloat, 32, 1};
  out.t.device      = DLDevice{kDLCUDA, res->device};
}
void widen_to_f32(resources* res, const DLTensor& src, f32_matrix& out) { widen_into(res, src, out); }
void widen_to_f32(resources* res, const DLTensor& src, f32_rows& out) { widen_into(res, src, out); }

void check_search_tensors(const DLTensor& queries, const DLTensor& neighbors, const DLTensor& distances, int64_t dim,
                          bool uint32_neighbors)
{
  B2_EXPECTS(dl_is_device(queries), "queries should have device compatible memory");
  B2_EXPECTS(dl_is_device(neighbors), "neighbors should have device compatible memory");
  B2_EXPECTS(dl_is_device(distances), "distances should have device compatible memory");
  if (uint32_neighbors)
    B2_EXPECTS(dl_is(neighbors, kDLUInt, 32) || dl_is(neighbors, kDLInt, 64), "neighbors should be of type uint32_t or int64_t");
  else
    B2_EXPECTS(dl_is(neighbors, kDLInt, 64), "neighbors should be of type int64_t");
  B2_EXPECTS(dl_is(distances, kDLFloat, 32), "distances should be of type float32");
  B2_EXPECTS(queries.ndim == 2 && neighbors.ndim == 2 && distances.ndim == 2, "queries/neighbors/distances must be 2-D");
  B2_EXPECTS(dl_is_c_contiguous(neighbors) && dl_is_c_contiguous(distances), "neighbors/distances must be row-major contiguous");
  B2_EXPECTS(neighbors.shape[0] == queries.shape[0] && distances.shape[0] == neighbors.shape[0] && distances.shape[1] == neighbors.shape[1],
             "neighbors/distances shape mismatch");
  B2_EXPECTS(queries.shape[1] == dim, "queries dim (%lld) != index dim (%lld)", (long long)queries.shape[1], (long long)dim);
}

filter_view read_prefilter(cuvsFilter filter, bool bitmap_ok, const char* unsupported)
{
  if (filter.type == NO_FILTER) return filter_view{};
  B2_EXPECTS(filter.type == BITSET || (bitmap_ok && filter.type == BITMAP), "%s", unsupported);
  auto ft = reinterpret_cast<const DLManagedTensor*>(filter.addr);
  B2_EXPECTS(ft != nullptr && dl_is_device(ft->dl_tensor), "prefilter should have device compatible memory");
  const DLTensor& t = ft->dl_tensor;
  B2_EXPECTS(dl_is(t, kDLUInt, 32) && t.ndim == 1 && dl_is_c_contiguous(t), "prefilter must be a contiguous 1-D uint32 tensor (got dtype code %d, bits %d, ndim %d)",
             int(t.dtype.code), int(t.dtype.bits), t.ndim);
  return filter_view{dl_ptr<uint32_t>(t), filter.type == BITSET ? 1 : 2, t.shape[0] * 32};
}


static thread_local std::string g_last_error;
static std::atomic<int> g_log_level{CUVS_LOG_LEVEL_INFO};

void set_last_error(const char* msg) { g_last_error = msg ? msg : ""; }

void dl_fill_view(DLManagedTensor* out, void* data, int device, DLDataType dt, int ndim, const int64_t* shape)
{
  B2_EXPECTS(out != nullptr, "output DLManagedTensor is null");
  DLTensor& t   = out->dl_tensor;
  t.data        = data;
  t.device      = DLDevice{kDLCUDA, device};
  t.ndim        = ndim;
  t.dtype       = dt;
  t.shape       = new int64_t[ndim];
  for (int i = 0; i < ndim; ++i) t.shape[i] = shape[i];
  t.strides     = nullptr;
  t.byte_offset = 0;
  out->manager_ctx = nullptr;
  out->deleter     = [](DLManagedTensor* self) {
    delete[] self->dl_tensor.shape;
    self->dl_tensor.shape = nullptr;
  };
}

static void lift_pool_threshold(int device)
{
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
    uint64_t thr = UINT64_MAX;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
  }
  cudaGetLastError();
}

}  // namespace b200

using namespace b200;

extern "C" {

const char* cuvsGetLastErrorText() { return g_last_error.empty() ? nullptr : g_last_error.c_str(); }
void cuvsSetLastErrorText(const char* error) { set_last_error(error); }

cuvsLogLevel_t cuvsGetLogLevel() { return static_cast<cuvsLogLevel_t>(g_log_level.load()); }
void cuvsSetLogLevel(cuvsLogLevel_t lvl) { g_log_level.store(static_cast<int>(lvl)); }

cuvsError_t cuvsResourcesCreate(cuvsResources_t* res)
{
  return guarded([=] {
    B2_EXPECTS(res != nullptr, "res is null");
    auto r = new resources{};
    try {
      B2_CUDA(cudaGetDevice(&r->device));
      r->sm_count = sm_count_of(r->device);
      lift_pool_threshold(r->device);
    } catch (...) {
      delete r;
      throw;
    }
    *res = reinterpret_cast<uintptr_t>(r);
  });
}

cuvsError_t cuvsResourcesDestroy(cuvsResources_t res)
{
  return guarded([=] { delete reinterpret_cast<resources*>(res); });
}

cuvsError_t cuvsStreamSet(cuvsResources_t res, cudaStream_t stream)
{
  return guarded([=] { as_res(res)->stream = stream; });
}

cuvsError_t cuvsStreamGet(cuvsResources_t res, cudaStream_t* stream)
{
  return guarded([=] {
    B2_EXPECTS(stream != nullptr, "stream is null");
    *stream = as_res(res)->stream;
  });
}

cuvsError_t cuvsStreamSync(cuvsResources_t res)
{
  return guarded([=] { B2_CUDA(cudaStreamSynchronize(as_res(res)->stream)); });
}

cuvsError_t cuvsDeviceIdGet(cuvsResources_t res, int* device_id)
{
  return guarded([=] {
    B2_EXPECTS(device_id != nullptr, "device_id is null");
    *device_id = as_res(res)->device;
  });
}

static void make_mg(resources* r, const std::vector<int>& ids)
{
  int cur = 0;
  B2_CUDA(cudaGetDevice(&cur));
  r->device     = cur;
  r->sm_count   = sm_count_of(cur);
  r->mg_devices = ids;
  for (int d : ids) {
    B2_CUDA(cudaSetDevice(d));
    cudaStream_t s;
    B2_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    r->mg_streams.push_back(s);
    lift_pool_threshold(d);
  }
  B2_CUDA(cudaSetDevice(cur));
}

cuvsError_t cuvsMultiGpuResourcesCreate(cuvsResources_t* res)
{
  return guarded([=] {
    B2_EXPECTS(res != nullptr, "res is null");
    int n = 0;
    B2_CUDA(cudaGetDeviceCount(&n));
    std::vector<int> ids(n);
    for (int i = 0; i < n; ++i) ids[i] = i;
    auto r = new resources{};
    try { make_mg(r, ids); } catch (...) { delete r; throw; }
    *res = reinterpret_cast<uintptr_t>(r);
  });
}

cuvsError_t cuvsMultiGpuResourcesCreateWithDeviceIds(cuvsResources_t* res, DLManagedTensor* device_ids)
{
  return guarded([=] {
    B2_EXPECTS(res != nullptr, "res is null");
    // same validation as c/src/core/c_api.cpp:56-76
    B2_EXPECTS(device_ids != nullptr && device_ids->dl_tensor.data != nullptr, "device_ids cannot be null");
    const DLTensor& t = device_ids->dl_tensor;
    B2_EXPECTS(dl_is(t, kDLInt, 32), "device_ids must be int32");
    B2_EXPECTS(t.device.device_type == kDLCPU, "device_ids must be on host memory");
    const int* p = dl_ptr<int>(t);
    std::vector<int> ids(p, p + t.shape[0]);
    auto r = new resources{};
    try { make_mg(r, ids); } catch (...) { delete r; throw; }
    *res = reinterpret_cast<uintptr_t>(r);
  });
}

cuvsError_t cuvsMultiGpuResourcesDestroy(cuvsResources_t res)
{
  return guarded([=] {
    auto r = reinterpret_cast<resources*>(res);
    if (r) {
      for (auto s : r->mg_streams) cudaStreamDestroy(s);
      delete r;
    }
  });
}

cuvsError_t cuvsMultiGpuResourcesSetMemoryPool(cuvsResources_t res, int percent_of_free_memory)
{
  return guarded([=] {
    auto r = as_res(res);
    B2_EXPECTS(percent_of_free_memory >= 0 && percent_of_free_memory <= 100, "percent must be in [0,100]");
    // The stream-ordered pools already retain memory (threshold lifted at creation); pre-warm them.
    int cur = 0;
    B2_CUDA(cudaGetDevice(&cur));
    for (size_t i = 0; i < r->mg_devices.size(); ++i) {
      B2_CUDA(cudaSetDevice(r->mg_devices[i]));
      size_t free_b = 0, total_b = 0;
      B2_CUDA(cudaMemGetInfo(&free_b, &total_b));
      size_t want = free_b / 100 * static_cast<size_t>(percent_of_free_memory);
      void* p = nullptr;
      if (want && cudaMallocAsync(&p, want, r->mg_streams[i]) == cudaSuccess) cudaFreeAsync(p, r->mg_streams[i]);
      cudaGetLastError();
    }
    B2_CUDA(cudaSetDevice(cur));
  });
}

cuvsError_t cuvsRMMAlloc(cuvsResources_t res, void** ptr, size_t bytes)
{
  return guarded([=] {
    B2_EXPECTS(ptr != nullptr, "ptr is null");
    B2_CUDA(cudaMallocAsync(ptr, bytes, as_res(res)->stream));
  });
}

cuvsError_t cuvsRMMFree(cuvsResources_t res, void* ptr, size_t /*bytes*/)
{
  return guarded([=] { B2_CUDA(cudaFreeAsync(ptr, as_res(res)->stream)); });
}

cuvsError_t cuvsRMMPoolMemoryResourceEnable(int initial_pool_size_percent, int max_pool_size_percent, bool managed)
{
  return guarded([=] {
    (void)managed;  // a managed pool only changes where the pages may migrate; allocations of this library stay on the device
    B2_EXPECTS(initial_pool_size_percent >= 0 && initial_pool_size_percent <= 100 && max_pool_size_percent >= 0 &&
                 max_pool_size_percent <= 100, "pool size percentages must be in [0,100]");
    int dev = 0;
    B2_CUDA(cudaGetDevice(&dev));
    lift_pool_threshold(dev);
    size_t free_b = 0, total_b = 0;
    B2_CUDA(cudaMemGetInfo(&free_b, &total_b));
    size_t want = total_b / 100 * static_cast<size_t>(initial_pool_size_percent);
    if (want > free_b) want = free_b / 2;
    void* p = nullptr;
    if (want && cudaMallocAsync(&p, want, cudaStreamPerThread) == cudaSuccess) cudaFreeAsync(p, cudaStreamPerThread);
    cudaGetLastError();
  });
}

cuvsError_t cuvsRMMMemoryResourceReset()
{
  return guarded([=] {
    int dev = 0;
    B2_CUDA(cudaGetDevice(&dev));
    cudaMemPool_t pool;
    B2_CUDA(cudaDeviceGetDefaultMemPool(&pool, dev));
    uint64_t thr = 0;
    B2_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr));
    B2_CUDA(cudaMemPoolTrimTo(pool, 0));
  });
}

cuvsError_t cuvsRMMHostAlloc(void** ptr, size_t bytes)
{
  return guarded([=] {
    B2_EXPECTS(ptr != nullptr, "ptr is null");
    B2_CUDA(cudaMallocHost(ptr, bytes));
  });
}

cuvsError_t cuvsRMMHostFree(void* ptr, size_t /*bytes*/)
{
  return guarded([=] { B2_CUDA(cudaFreeHost(ptr)); });
}

cuvsError_t cuvsVersionGet(uint16_t* major, uint16_t* minor, uint16_t* patch)
{
  // ABI level of the reference this library stands in for (VERSION: 26.08.00)
  if (major) *major = 26;
  if (minor) *minor = 8;
  if (patch) *patch = 0;
  return CUVS_SUCCESS;
}

void cuvsMatrixDestroy(DLManagedTensor* tensor)
{
  if (!tensor) return;
  delete[] tensor->dl_tensor.shape;
  tensor->dl_tensor.shape = nullptr;
  delete[] tensor->dl_tensor.strides;
  tensor->dl_tensor.strides = nullptr;
}

cuvsError_t cuvsMatrixCopy(cuvsResources_t res, DLManagedTensor* src_m, DLManagedTensor* dst_m)
{
  return guarded([=] {
    B2_EXPECTS(src_m && dst_m, "src/dst tensor is null");
    const DLTensor& src = src_m->dl_tensor;
    DLTensor& dst       = dst_m->dl_tensor;
    B2_EXPECTS(src.ndim == dst.ndim, "src and dst tensors should have the same dimensions");
    for (int i = 0; i < src.ndim; ++i)
      B2_EXPECTS(src.shape[i] == dst.shape[i], "shape mismatch between src and dst tensors");
    B2_EXPECTS(src.dtype.code == dst.dtype.code, "dtype mismatch between src and dst tensors");
    B2_EXPECTS(src.dtype.bits == dst.dtype.bits, "dtype bits width mismatch between src and dst tensors");
    const size_t esz = src.dtype.bits / 8;
    B2_EXPECTS(esz >= 1 && esz <= 8, "Unsupported dtype: %d and bits: %d", src.dtype.code, src.dtype.bits);
    auto stream = as_res(res)->stream;
    if (src.ndim == 2) {
      B2_EXPECTS((src.strides == nullptr || src.strides[1] == 1) && (dst.strides == nullptr || dst.strides[1] == 1),
                 "cuvsMatrixCopy needs unit stride along the last dimension");
      int64_t sp = src.strides ? src.strides[0] : src.shape[1];
      int64_t dp = dst.strides ? dst.strides[0] : dst.shape[1];
      B2_CUDA(cudaMemcpy2DAsync(dl_ptr<char>(dst), dp * esz, dl_ptr<char>(src), sp * esz, src.shape[1] * esz,
                                src.shape[0], cudaMemcpyDefault, stream));
    } else {
      B2_EXPECTS(src.strides == nullptr && dst.strides == nullptr, "cuvsCopyMatrix only supports strides with 2D inputs");
      size_t elements = 1;
      for (int i = 0; i < src.ndim; ++i) elements *= src.shape[i];
      B2_CUDA(cudaMemcpyAsync(dl_ptr<char>(dst), dl_ptr<char>(src), elements * esz, cudaMemcpyDefault, stream));
    }
  });
}

cuvsError_t cuvsMatrixSliceRows(cuvsResources_t, DLManagedTensor* src_m, int64_t start, int64_t end, DLManagedTensor* dst_m)
{
  return guarded([=] {
    B2_EXPECTS(src_m && dst_m, "src/dst tensor is null");
    B2_EXPECTS(end >= start, "end index must be greater than start index");
    const DLTensor& src = src_m->dl_tensor;
    DLTensor& dst       = dst_m->dl_tensor;
    B2_EXPECTS(src.ndim <= 2 && src.ndim >= 1, "src should be a 1 or 2 dimensional tensor");
    B2_EXPECTS(src.shape != nullptr, "shape should be initialized in the src tensor");
    dst.dtype       = src.dtype;
    dst.device      = src.device;
    dst.ndim        = src.ndim;
    dst.byte_offset = 0;
    dst.shape       = new int64_t[dst.ndim];
    dst.shape[0]    = end - start;
    dst.strides     = nullptr;
    int64_t row_stride = 1;
    if (dst.ndim == 2) {
      dst.shape[1] = src.shape[1];
      row_stride   = src.shape[1];
      if (src.strides) {
        dst.strides    = new int64_t[2];
        dst.strides[0] = row_stride = src.strides[0];
        dst.strides[1] = src.strides[1];
      }
    }
    dst.data           = static_cast<char*>(src.data) + start * row_stride * (dst.dtype.bits / 8);
    dst_m->manager_ctx = nullptr;
    dst_m->deleter     = cuvsMatrixDestroy;
  });
}

}  // extern "C"
