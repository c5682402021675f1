// Optional CUDA-event timing of named kernel sections + launch counting (see include/cuvs_b200/ext.h).
#pragma once
#include <cuda_runtime.h>

namespace b200 {

bool timing_enabled();
void timing_begin(const char* name, cudaStream_t stream, cudaEvent_t* ev_start);
void timing_end(const char* name, cudaStream_t stream, cudaEvent_t ev_start);
void count_launch(int n = 1);
void set_last_flagged(int n);
/** Same, for a count the device has yet to write at dev_count: a copy to pinned memory is enqueued on `stream`, and
 *  cuvsB200LastFlagged waits for it only when it is called, so the search needs no host round trip. */
void set_last_flagged_async(const int* dev_count, cudaStream_t stream);

/** RAII: records start/stop events around a section when timing is enabled. */
struct timed_section {
  const char* name;
  cudaStream_t stream;
  cudaEvent_t start = nullptr;
  bool on;
  timed_section(const char* n, cudaStream_t s) : name(n), stream(s), on(timing_enabled())
  {
    if (on) timing_begin(name, stream, &start);
  }
  ~timed_section()
  {
    if (on) timing_end(name, stream, start);
  }
};

}  // namespace b200
