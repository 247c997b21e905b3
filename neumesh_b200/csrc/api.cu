// Library-wide state of the neumesh_b200 C ABI: error string, launch counter, device queries.
#include <atomic>
#include <mutex>
#include <vector>

#include "../../include/neumesh_b200.h"
#include "common.cuh"

namespace nmb {
static thread_local std::string g_error;
static std::atomic<int64_t> g_launches{0};
static std::atomic<int64_t> g_allocs{0};
static std::atomic<int> g_deterministic{0};
bool deterministic() { return g_deterministic.load(std::memory_order_relaxed) != 0; }
void set_error(const std::string& msg) { g_error = msg; }
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
void count_alloc() { g_allocs.fetch_add(1, std::memory_order_relaxed); }
int sm_count() {
  static std::atomic<int> cached[NMB_MAX_DEVICES];   // per device of this process; 0 = not queried yet
  int dev = 0;
  cudaGetDevice(&dev);
  std::atomic<int>& c = cached[dev % NMB_MAX_DEVICES];
  int n = c.load(std::memory_order_relaxed);
  if (n == 0) {
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;   // H100 SXM
    c.store(n, std::memory_order_relaxed);
  }
  return n;
}

cudaError_t ensure_scratch_pool() {
  static DeviceOnce once;
  return once.run([] {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    cudaMemPool_t pool;
    e = cudaDeviceGetDefaultMemPool(&pool, dev);
    if (e != cudaSuccess) return e;
    uint64_t cur = 0;
    e = cudaMemPoolGetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &cur);
    if (e != cudaSuccess) return e;
    uint64_t want = 1ull << 30;
    return cur >= want ? cudaSuccess : cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &want);
  });
}

// ---- profiling ----
struct ProfRec {
  cudaEvent_t a, b;
  int tag;
  int64_t units;
};
static bool g_prof = false;
static std::vector<ProfRec> g_recs;
static std::vector<ProfRec> g_open;
static std::mutex g_prof_mu;
bool prof_enabled() { return g_prof; }
void prof_begin(int tag, int64_t units, cudaStream_t stream) {
  ProfRec r;
  cudaEventCreate(&r.a);
  cudaEventCreate(&r.b);
  r.tag = tag;
  r.units = units;
  cudaEventRecord(r.a, stream);
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_open.push_back(r);
}
void prof_end(int tag, cudaStream_t stream) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  for (size_t i = g_open.size(); i-- > 0;) {
    if (g_open[i].tag == tag) {
      cudaEventRecord(g_open[i].b, stream);
      g_recs.push_back(g_open[i]);
      g_open.erase(g_open.begin() + i);
      return;
    }
  }
}
}  // namespace nmb

extern "C" {
void nmb_profile_enable(int on) {
  std::lock_guard<std::mutex> lk(nmb::g_prof_mu);
  nmb::g_prof = on != 0;
}
int nmb_profile_collect(double* ms, int64_t* launches, int64_t* units, int n_tags) {
  std::lock_guard<std::mutex> lk(nmb::g_prof_mu);
  for (int i = 0; i < n_tags; ++i) {
    ms[i] = 0;
    launches[i] = 0;
    units[i] = 0;
  }
  for (auto& r : nmb::g_recs) {
    cudaEventSynchronize(r.b);
    float t = 0.f;
    cudaEventElapsedTime(&t, r.a, r.b);
    if (r.tag < n_tags) {
      ms[r.tag] += t;
      launches[r.tag] += 1;
      units[r.tag] += r.units;
    }
    cudaEventDestroy(r.a);
    cudaEventDestroy(r.b);
  }
  nmb::g_recs.clear();
  return 0;
}
void nmb_set_deterministic(int on) { nmb::g_deterministic.store(on != 0, std::memory_order_relaxed); }
int nmb_deterministic(void) { return nmb::deterministic() ? 1 : 0; }
const char* nmb_last_error(void) { return nmb::g_error.c_str(); }
int nmb_version(void) { return NMB_VERSION; }
int64_t nmb_launch_count(void) { return nmb::g_launches.load(); }
int64_t nmb_alloc_count(void) { return nmb::g_allocs.load(); }
}
