// Timing / introspection extensions (include/cuvs_b200/ext.h).
#include "common.hpp"
#include "timing.hpp"

#include <cuvs_b200/ext.h>

#include <atomic>
#include <map>
#include <mutex>
#include <string>
#include <vector>

namespace b200 {
namespace {
std::atomic<int> g_timing{0};
std::atomic<long long> g_launches{0};
thread_local int g_last_flagged = 0;
// set_last_flagged_async: one pinned int and event per thread (for the device it was last used on), released when the thread
// exits or moves to another device, after the copy into the int has landed.  Errors are ignored there: at process exit the
// runtime may already be gone, and nothing is left to report to.
struct pending_count {
  int device        = -1;
  int* host         = nullptr;
  cudaEvent_t done  = nullptr;
  bool pending      = false;
  void release()
  {
    if (host == nullptr) return;
    cudaEventSynchronize(done);
    cudaEventDestroy(done);
    cudaFreeHost(host);
    host    = nullptr;
    done    = nullptr;
    device  = -1;
    pending = false;
  }
  ~pending_count() { release(); }
};
thread_local pending_count g_pending;
std::mutex g_mu;
std::map<std::string, std::vector<std::pair<cudaEvent_t, cudaEvent_t>>> g_events;
}  // namespace

bool timing_enabled() { return g_timing.load(std::memory_order_relaxed) != 0; }
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
void set_last_flagged(int n)
{
  g_last_flagged    = n;
  g_pending.pending = false;
}
void set_last_flagged_async(const int* dev_count, cudaStream_t stream)
{
  int dev = 0;
  B2_CUDA(cudaGetDevice(&dev));
  auto& p = g_pending;
  if (p.device != dev) {
    if (p.pending) {  // the count of the search on the old device stays readable
      B2_CUDA(cudaEventSynchronize(p.done));
      g_last_flagged = *p.host;
    }
    p.release();
    B2_CUDA(cudaMallocHost(&p.host, sizeof(int)));
    B2_CUDA(cudaEventCreateWithFlags(&p.done, cudaEventDisableTiming));
    p.device = dev;
  }
  B2_CUDA(cudaMemcpyAsync(p.host, dev_count, sizeof(int), cudaMemcpyDeviceToHost, stream));
  B2_CUDA(cudaEventRecord(p.done, stream));
  p.pending = true;
}

void timing_begin(const char*, cudaStream_t stream, cudaEvent_t* ev_start)
{
  cudaEventCreate(ev_start);
  cudaEventRecord(*ev_start, stream);
}
void timing_end(const char* name, cudaStream_t stream, cudaEvent_t ev_start)
{
  cudaEvent_t stop;
  cudaEventCreate(&stop);
  cudaEventRecord(stop, stream);
  std::lock_guard<std::mutex> lk(g_mu);
  g_events[name].emplace_back(ev_start, stop);
}
}  // namespace b200

using namespace b200;

extern "C" {
void cuvsB200TimingEnable(int on) { g_timing.store(on); }
void cuvsB200TimingReset(void)
{
  std::lock_guard<std::mutex> lk(g_mu);
  for (auto& kv : g_events)
    for (auto& p : kv.second) { cudaEventDestroy(p.first); cudaEventDestroy(p.second); }
  g_events.clear();
}
double cuvsB200TimingTotalMs(const char* name, int* count)
{
  std::lock_guard<std::mutex> lk(g_mu);
  double total = 0;
  int n        = 0;
  auto it      = g_events.find(name ? name : "");
  if (it != g_events.end()) {
    for (auto& p : it->second) {
      float ms = 0;
      if (cudaEventSynchronize(p.second) == cudaSuccess && cudaEventElapsedTime(&ms, p.first, p.second) == cudaSuccess) {
        total += ms;
        ++n;
      }
    }
  }
  if (count) *count = n;
  return total;
}
int cuvsB200LastFlagged(void)
{
  if (g_pending.pending && cudaEventSynchronize(g_pending.done) == cudaSuccess) {
    g_last_flagged    = *g_pending.host;
    g_pending.pending = false;
  }
  return g_last_flagged;
}
long long cuvsB200KernelLaunches(void) { return g_launches.load(); }
}
