// List storage shared by IVF-Flat and IVF-PQ: rows grouped by list, every list padded to a whole
// number of 128-row tiles so that a (list, query-group) work item is tile aligned for the wgmma scan.
//
// The reference keeps one allocation per list with rows interleaved in groups of 32
// (cpp/include/cuvs/neighbors/ivf_flat.hpp:184-201, ivf_pq.hpp:235-296) because its scan kernel
// assigns one warp lane per row.  Here the scan is a dense tile contraction fed by TMA, so the natural
// layout is one flat K-major [rows, dim] array with lists back to back (a list tile is a single
// 2-D TMA box; no per-list pointer table, no interleaving).
#pragma once
#include "common.hpp"
#include "scan_tc.cuh"  // kPadId

#include <functional>
#include <vector>

namespace b200 {

struct list_layout {
  int64_t n_lists = 0;
  std::vector<int64_t> h_sizes;    // rows per list
  std::vector<int64_t> h_offsets;  // padded start row of each list (n_lists + 1 entries, multiples of 128)
  owned<int64_t> d_offsets;
  owned<uint32_t> d_sizes;
  int64_t rows_total = 0;  // = h_offsets[n_lists]
  int64_t size       = 0;  // sum of sizes

  void set_sizes(cudaStream_t s, const std::vector<int64_t>& sizes);
};

/** Storage for `lists`: payload [rows_total, width] zeroed, ids [rows_total] set to kPadId (at least one row of each). */
template <typename T>
void alloc_list_storage(cudaStream_t s, const list_layout& lists, int64_t width, owned<T>& payload, owned<int64_t>& ids);

/** dst[dst_rows[i]] = src[i] for rows of `width` elements; rows with dst_rows[i] < 0 are skipped. */
template <typename T>
void scatter_rows(cudaStream_t s, const T* src, int64_t n, int64_t width, const int64_t* dst_rows, T* dst);

/** labels[i] = list of row i of the fp32 chunk x [n, dim] (device). */
using label_chunk_fn = std::function<void(const float* x, int64_t n, uint32_t* labels)>;
/** Writes the payload of row i of the chunk x [n, dim] (list labels[i]) to row dst_rows[i] of `payload`. */
template <typename T>
using write_chunk_fn = std::function<void(const float* x, int64_t n, uint32_t* labels, const int64_t* dst_rows, T* payload)>;

/**
 * Appends the rows of `t` ([n, dim], device or host: fp32, or int8 / uint8 widened one chunk at a time) to the lists, with ids new_ids[i] (device; null: id0 + i), and
 * replaces `lists`, `payload` [rows_total, width] and `ids` with the grown storage.  The rows go through the device in
 * chunks of at most 512 MiB (host rows are staged through one buffer), twice, so that the lists are laid out once for the
 * whole insertion: (1) `label` names each row's list and the rows are counted per list; (2) the old rows move to the new
 * layout and every chunk is placed behind them, `write` filling its payload rows.  Inside a list the order is the input
 * order: the old rows in their order, then the new ones in the order of `t`.  The caller refreshes its derived data.
 */
template <typename T>
void insert_rows(resources* res, const DLTensor& t, list_layout& lists, owned<T>& payload, int64_t width, owned<int64_t>& ids,
                 const int64_t* new_ids, int64_t id0, const label_chunk_fn& label, const write_chunk_fn<T>& write);

/** The ids a C-ABI extend was given (int64 [n], device or host) as a device pointer, host ids staged into `buf`; null when
 *  `new_indices` is null. */
const int64_t* device_ids(resources* res, DLManagedTensor* new_indices, int64_t n, dbuf<int64_t>& buf);

}  // namespace b200
