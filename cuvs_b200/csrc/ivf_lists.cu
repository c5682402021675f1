// List layout and insertion (see ivf_lists.cuh).
#include "ivf_lists.cuh"
#include "timing.hpp"

#include <cub/device/device_radix_sort.cuh>

#include <algorithm>

namespace b200 {
namespace {
__global__ void count_labels_kernel(const uint32_t* __restrict__ labels, int64_t n, unsigned long long* __restrict__ counts)
{
  int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i < n) atomicAdd(&counts[labels[i]], 1ull);
}

__global__ void iota_kernel(uint32_t* __restrict__ p, int64_t n)
{
  int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i < n) p[i] = static_cast<uint32_t>(i);
}

// rows sorted stably by label: sorted position i of a row of list l is start[l] + its rank in l, and base[l] = offsets[l] +
// base_fill[l] - start[l]
__global__ void place_sorted_kernel(const uint32_t* __restrict__ labels, const uint32_t* __restrict__ rows, int64_t n,
                                    const int64_t* __restrict__ base, int64_t* __restrict__ dst)
{
  int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i < n) dst[rows[i]] = base[labels[i]] + i;
}

// new row of every old (padded) row: same position inside its list, -1 on padding rows.  One CTA per list.
__global__ void remap_rows_kernel(const int64_t* __restrict__ old_off, const int64_t* __restrict__ new_off,
                                  const uint32_t* __restrict__ old_sizes, int64_t* __restrict__ dst_rows)
{
  const int64_t l = blockIdx.x;
  for (int64_t i = threadIdx.x; i < old_off[l + 1] - old_off[l]; i += blockDim.x)
    dst_rows[old_off[l] + i] = i < old_sizes[l] ? new_off[l] + i : -1;
}

template <typename T>
__global__ void scatter_rows_kernel(const T* __restrict__ src, int64_t n, int64_t width, const int64_t* __restrict__ dst_rows,
                                    T* __restrict__ dst)
{
  int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (t >= n * width) return;
  const int64_t r = t / width, o = dst_rows[r];
  if (o >= 0) dst[o * width + t % width] = src[t];
}

__global__ void write_ids_kernel(const int64_t* __restrict__ dst_rows, const int64_t* __restrict__ src_ids, int64_t id0, int64_t n,
                                 int64_t* __restrict__ ids)
{
  int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i < n) ids[dst_rows[i]] = src_ids ? src_ids[i] : id0 + i;
}

__global__ void fill_i64_kernel(int64_t* p, int64_t n, int64_t v)
{
  int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i < n) p[i] = v;
}

/** counts[l] = number of rows with that label (host vector, synchronises the stream). */
std::vector<int64_t> count_labels(cudaStream_t s, const uint32_t* labels, int64_t n, int64_t n_lists)
{
  dbuf<unsigned long long> c(static_cast<size_t>(n_lists), s);
  B2_CUDA(cudaMemsetAsync(c.data(), 0, sizeof(unsigned long long) * n_lists, s));
  if (n) {
    count_launch();
    count_labels_kernel<<<blocks_for(n, 256), 256, 0, s>>>(labels, n, c.data());
    B2_CUDA(cudaGetLastError());
  }
  std::vector<unsigned long long> h(static_cast<size_t>(n_lists));
  B2_CUDA(cudaMemcpyAsync(h.data(), c.data(), sizeof(unsigned long long) * n_lists, cudaMemcpyDeviceToHost, s));
  B2_CUDA(cudaStreamSynchronize(s));
  return std::vector<int64_t>(h.begin(), h.end());
}

/**
 * dst_rows[i] = offsets[l] + base_fill[l] + (number of earlier rows of this call in list l), l = labels[i]: the rows of a list
 * land behind its base_fill[l] present rows in input order.  counts = count_labels of these rows.  The ranks come from a
 * stable radix sort of (label, row) over the label bits, so the placement does not depend on thread timing.
 */
void place_rows(cudaStream_t s, const uint32_t* labels, int64_t n, const list_layout& layout, const std::vector<int64_t>& base_fill,
                const std::vector<int64_t>& counts, int64_t* dst_rows)
{
  if (n == 0) return;
  std::vector<int64_t> base(static_cast<size_t>(layout.n_lists));
  for (int64_t l = 0, start = 0; l < layout.n_lists; start += counts[l], ++l) base[l] = layout.h_offsets[l] + base_fill[l] - start;
  int end_bit = 1;
  while ((int64_t(1) << end_bit) < layout.n_lists) ++end_bit;
  dbuf<uint32_t> rows_in(static_cast<size_t>(n), s), rows_out(static_cast<size_t>(n), s), labels_out(static_cast<size_t>(n), s);
  dbuf<int64_t> d_base(base.size(), s);
  B2_CUDA(cudaMemcpyAsync(d_base.data(), base.data(), sizeof(int64_t) * base.size(), cudaMemcpyHostToDevice, s));
  count_launch();
  iota_kernel<<<blocks_for(n, 256), 256, 0, s>>>(rows_in.data(), n);
  B2_CUDA(cudaGetLastError());
  size_t tmp_bytes = 0;
  B2_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, labels, labels_out.data(), rows_in.data(), rows_out.data(), n, 0, end_bit, s));
  dbuf<unsigned char> tmp(tmp_bytes, s);
  B2_CUDA(cub::DeviceRadixSort::SortPairs(tmp.data(), tmp_bytes, labels, labels_out.data(), rows_in.data(), rows_out.data(), n, 0, end_bit, s));
  count_launch();
  place_sorted_kernel<<<blocks_for(n, 256), 256, 0, s>>>(labels_out.data(), rows_out.data(), n, d_base.data(), dst_rows);
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaStreamSynchronize(s));  // `base` is a host vector
}

// rows of `t` as fp32 device-resident chunks of at most 512 MiB (host tensors are staged through one reusable buffer; int8 and
// uint8 rows are widened one chunk at a time)
template <typename Fn>
void for_device_chunks(resources* res, const DLTensor& t, Fn&& fn)
{
  const int64_t n = t.shape[0];
  const int d     = static_cast<int>(t.shape[1]);
  const int64_t chunk = std::max<int64_t>(1, (int64_t(1) << 27) / std::max(d, 1));  // 512 MiB of floats per step
  const bool dev  = dl_is_device(t) && t.device.device_type != kDLCUDAHost;
  const bool f32  = dl_is(t, kDLFloat, 32);
  const size_t es = t.dtype.bits / 8;
  dbuf<float> buf;
  dbuf<uint8_t> raw;
  if (!dev || !f32) buf.alloc(static_cast<size_t>(std::min(n, chunk)) * d, res->stream);
  if (!dev && !f32) raw.alloc(static_cast<size_t>(std::min(n, chunk)) * d * es, res->stream);
  for (int64_t r0 = 0; r0 < n; r0 += chunk) {
    int64_t rows = std::min(chunk, n - r0);
    const uint8_t* src = dl_ptr<uint8_t>(t) + r0 * d * es;
    if (f32 && dev) {
      fn(reinterpret_cast<const float*>(src), rows, r0);
    } else if (f32) {
      B2_CUDA(cudaMemcpyAsync(buf.data(), src, sizeof(float) * rows * d, cudaMemcpyHostToDevice, res->stream));
      fn(buf.data(), rows, r0);
    } else {
      if (!dev) {
        B2_CUDA(cudaMemcpyAsync(raw.data(), src, es * rows * d, cudaMemcpyHostToDevice, res->stream));
        src = raw.data();
      }
      widen_async(res->stream, src, t.dtype, rows * d, buf.data());
      fn(buf.data(), rows, r0);
    }
  }
}
}  // namespace

void list_layout::set_sizes(cudaStream_t s, const std::vector<int64_t>& sizes)
{
  n_lists = static_cast<int64_t>(sizes.size());
  h_sizes = sizes;
  h_offsets.assign(n_lists + 1, 0);
  size = 0;
  for (int64_t l = 0; l < n_lists; ++l) {
    h_offsets[l + 1] = h_offsets[l] + (sizes[l] + 127) / 128 * 128;
    size += sizes[l];
  }
  rows_total = h_offsets[n_lists];
  d_offsets.alloc(static_cast<size_t>(n_lists + 1));
  d_sizes.alloc(static_cast<size_t>(std::max<int64_t>(n_lists, 1)));
  std::vector<uint32_t> s32(sizes.begin(), sizes.end());
  B2_CUDA(cudaMemcpyAsync(d_offsets.data(), h_offsets.data(), sizeof(int64_t) * (n_lists + 1), cudaMemcpyHostToDevice, s));
  if (n_lists) B2_CUDA(cudaMemcpyAsync(d_sizes.data(), s32.data(), sizeof(uint32_t) * n_lists, cudaMemcpyHostToDevice, s));
  B2_CUDA(cudaStreamSynchronize(s));  // host vectors go out of scope
}

template <typename T>
void alloc_list_storage(cudaStream_t s, const list_layout& lists, int64_t width, owned<T>& payload, owned<int64_t>& ids)
{
  const int64_t R = lists.rows_total;
  payload.alloc(static_cast<size_t>(std::max<int64_t>(R, 1)) * width);
  ids.alloc(static_cast<size_t>(std::max<int64_t>(R, 1)));
  B2_CUDA(cudaMemsetAsync(payload.data(), 0, sizeof(T) * static_cast<size_t>(R) * width, s));
  if (R == 0) return;
  count_launch();
  fill_i64_kernel<<<blocks_for(R, 256), 256, 0, s>>>(ids.data(), R, kPadId);
  B2_CUDA(cudaGetLastError());
}

template <typename T>
void scatter_rows(cudaStream_t s, const T* src, int64_t n, int64_t width, const int64_t* dst_rows, T* dst)
{
  if (n == 0) return;
  count_launch();
  scatter_rows_kernel<<<blocks_for(n * width, 256), 256, 0, s>>>(src, n, width, dst_rows, dst);
  B2_CUDA(cudaGetLastError());
}

template <typename T>
void insert_rows(resources* res, const DLTensor& t, list_layout& lists, owned<T>& payload, int64_t width, owned<int64_t>& ids,
                 const int64_t* new_ids, int64_t id0, const label_chunk_fn& label, const write_chunk_fn<T>& write)
{
  auto s          = res->stream;
  const int64_t n = t.shape[0];
  if (n == 0) return;
  // 1. label every row, count per list
  dbuf<uint32_t> labels(static_cast<size_t>(n), s);
  std::vector<int64_t> sizes = lists.h_sizes;
  std::vector<std::vector<int64_t>> chunk_add;
  for_device_chunks(res, t, [&](const float* x, int64_t rows, int64_t r0) {
    label(x, rows, labels.data() + r0);
    chunk_add.push_back(count_labels(s, labels.data() + r0, rows, lists.n_lists));
    for (int64_t l = 0; l < lists.n_lists; ++l) sizes[l] += chunk_add.back()[l];
  });
  // 2. the new layout; the old rows keep their order at the front of each list
  list_layout nl;
  nl.set_sizes(s, sizes);
  owned<T> npayload;
  owned<int64_t> nids;
  alloc_list_storage(s, nl, width, npayload, nids);
  if (lists.rows_total > 0) {
    dbuf<int64_t> dst_old(static_cast<size_t>(lists.rows_total), s);
    count_launch();
    remap_rows_kernel<<<static_cast<unsigned>(lists.n_lists), 128, 0, s>>>(lists.d_offsets.data(), nl.d_offsets.data(), lists.d_sizes.data(),
                                                                            dst_old.data());
    B2_CUDA(cudaGetLastError());
    scatter_rows(s, payload.data(), lists.rows_total, width, dst_old.data(), npayload.data());
    scatter_rows(s, ids.data(), lists.rows_total, int64_t(1), dst_old.data(), nids.data());
  }
  // 3. every chunk behind the rows already placed in its lists
  std::vector<int64_t> fill = lists.h_sizes;
  size_t ci = 0;
  for_device_chunks(res, t, [&](const float* x, int64_t rows, int64_t r0) {
    dbuf<int64_t> dst_new(static_cast<size_t>(rows), s);
    place_rows(s, labels.data() + r0, rows, nl, fill, chunk_add[ci], dst_new.data());
    for (int64_t l = 0; l < nl.n_lists; ++l) fill[l] += chunk_add[ci][l];
    ++ci;
    write(x, rows, labels.data() + r0, dst_new.data(), npayload.data());
    count_launch();
    write_ids_kernel<<<blocks_for(rows, 256), 256, 0, s>>>(dst_new.data(), new_ids ? new_ids + r0 : nullptr, id0 + r0, rows, nids.data());
    B2_CUDA(cudaGetLastError());
  });
  B2_CUDA(cudaStreamSynchronize(s));
  payload = std::move(npayload);
  ids     = std::move(nids);
  lists   = std::move(nl);
}

template void alloc_list_storage<float>(cudaStream_t, const list_layout&, int64_t, owned<float>&, owned<int64_t>&);
template void alloc_list_storage<uint8_t>(cudaStream_t, const list_layout&, int64_t, owned<uint8_t>&, owned<int64_t>&);
template void scatter_rows<float>(cudaStream_t, const float*, int64_t, int64_t, const int64_t*, float*);
template void scatter_rows<uint8_t>(cudaStream_t, const uint8_t*, int64_t, int64_t, const int64_t*, uint8_t*);
template void insert_rows<float>(resources*, const DLTensor&, list_layout&, owned<float>&, int64_t, owned<int64_t>&, const int64_t*, int64_t,
                                 const label_chunk_fn&, const write_chunk_fn<float>&);
template void insert_rows<uint8_t>(resources*, const DLTensor&, list_layout&, owned<uint8_t>&, int64_t, owned<int64_t>&, const int64_t*,
                                   int64_t, const label_chunk_fn&, const write_chunk_fn<uint8_t>&);

const int64_t* device_ids(resources* res, DLManagedTensor* new_indices, int64_t n, dbuf<int64_t>& buf)
{
  if (!new_indices) return nullptr;
  const DLTensor& it = new_indices->dl_tensor;
  B2_EXPECTS(dl_is(it, kDLInt, 64) && it.shape[0] == n, "new_indices must be int64 [n]");
  if (dl_is_device(it) && it.device.device_type != kDLCUDAHost) return dl_ptr<int64_t>(it);
  buf.alloc(static_cast<size_t>(n), res->stream);
  B2_CUDA(cudaMemcpyAsync(buf.data(), dl_ptr<int64_t>(it), sizeof(int64_t) * n, cudaMemcpyHostToDevice, res->stream));
  return buf.data();
}

}  // namespace b200
