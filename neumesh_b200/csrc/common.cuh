// Shared helpers for the neumesh_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <mutex>
#include <string>

namespace nmb {

void set_error(const std::string& msg);
void count_launch(int n = 1);
void count_alloc();   // one cudaMalloc by a DevBuf (nmb_alloc_count)

#define NMB_CUDA_OK(expr)                                                                               \
  do {                                                                                                  \
    cudaError_t _e = (expr);                                                                            \
    if (_e != cudaSuccess) {                                                                            \
      ::nmb::set_error(std::string(#expr) + " failed: " + cudaGetErrorString(_e) + " (" + __FILE__ +  \
                       ":" + std::to_string(__LINE__) + ")");                                           \
      return 1;                                                                                         \
    }                                                                                                   \
  } while (0)

#define NMB_CHECK(cond, msg)                                                \
  do {                                                                      \
    if (!(cond)) {                                                          \
      ::nmb::set_error(std::string(msg) + " [" #cond "]");                  \
      return 2;                                                             \
    }                                                                       \
  } while (0)

#define NMB_LAUNCH_OK()                                      \
  do {                                                       \
    ::nmb::count_launch();                                   \
    NMB_CUDA_OK(cudaGetLastError());                         \
  } while (0)

// Keeps up to 1 GiB of freed stream-ordered scratch cached in the device's default memory pool (the default
// threshold of 0 hands every block back to the driver at the next synchronisation).  Once per device.
cudaError_t ensure_scratch_pool();

// Stream-ordered scratch (cudaMallocAsync) that is returned to the pool on every exit path of an API call.
struct StreamBuf {
  void* p = nullptr;
  cudaStream_t stream = nullptr;
  StreamBuf() = default;
  StreamBuf(const StreamBuf&) = delete;
  StreamBuf& operator=(const StreamBuf&) = delete;
  ~StreamBuf() {
    if (p) cudaFreeAsync(p, stream);
  }
  cudaError_t alloc(size_t bytes, cudaStream_t s) {
    stream = s;
    cudaError_t e = ensure_scratch_pool();
    if (e != cudaSuccess) return e;
    return cudaMallocAsync(&p, bytes ? bytes : 1, s);
  }
  template <typename T>
  T* as() const { return static_cast<T*>(p); }
};

// Run `f` (-> cudaError_t) until it has succeeded once per CUDA device of this process (kernel attributes are per
// device); thread-safe.
constexpr int NMB_MAX_DEVICES = 64;
struct DeviceOnce {
  std::mutex mu;
  bool done[NMB_MAX_DEVICES] = {};
  template <typename F>
  cudaError_t run(F&& f) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    std::lock_guard<std::mutex> lock(mu);
    bool& d = done[dev % NMB_MAX_DEVICES];
    if (d) return cudaSuccess;
    e = f();               // a failed attempt is reported AND retried by the next call (the flag is only set on success)
    if (e == cudaSuccess) d = true;
    return e;
  }
};

// torch.sum over a contiguous fp32 row of n elements as ATen's CPU kernel computes it (SumKernel.cpp, the path
// `weights.sum(dim=-1)` of rend_util.py:281 takes; checked against torch 2.11 for every n <= 255, AVX2 and AVX512
// builds alike): the row is read as 8-lane vectors; four vector accumulators take vectors 4i, 4i+1, 4i+2, 4i+3, leftover
// vectors go to accumulator 0, the accumulators are folded 0 += 1, 2, 3; then a scalar starts from 0, adds the tail
// elements (n % 8) in order and finally the 8 lanes in order.  Rows shorter than 8 use four scalar accumulators in the
// same pattern.  sample_pdf's u = 1 sample (searchsorted against a cdf that saturates at 1.0 or not) depends on these
// bits, so the normalisation constant is reproduced exactly rather than summed sequentially.
__device__ __forceinline__ float torch_row_sum(const float* __restrict__ x, int64_t stride, int n) {
  if (n < 8) {
    float a[4] = {0.f, 0.f, 0.f, 0.f};
    const int q = n / 4;
    if (q) {
#pragma unroll
      for (int k = 0; k < 4; ++k) a[k] = __fadd_rn(a[k], x[k * stride]);
    }
    for (int i = q * 4; i < n; ++i) a[0] = __fadd_rn(x[i * stride], a[0]);
    a[0] = __fadd_rn(a[0], a[1]);
    a[0] = __fadd_rn(a[0], a[2]);
    return __fadd_rn(a[0], a[3]);
  }
  float acc[4][8];
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int l = 0; l < 8; ++l) acc[k][l] = 0.f;
  const int nvec = n / 8, nblk = nvec / 4;
  for (int b = 0; b < nblk; ++b) {
#pragma unroll
    for (int t = 0; t < 32; ++t) acc[t / 8][t % 8] = __fadd_rn(acc[t / 8][t % 8], x[(int64_t)(b * 32 + t) * stride]);
  }
  for (int v = nblk * 4; v < nvec; ++v) {
#pragma unroll
    for (int l = 0; l < 8; ++l) acc[0][l] = __fadd_rn(x[(int64_t)(v * 8 + l) * stride], acc[0][l]);
  }
#pragma unroll
  for (int k = 1; k < 4; ++k)
#pragma unroll
    for (int l = 0; l < 8; ++l) acc[0][l] = __fadd_rn(acc[0][l], acc[k][l]);
  float fin = 0.f;
  for (int i = nvec * 8; i < n; ++i) fin = __fadd_rn(fin, x[(int64_t)i * stride]);
#pragma unroll
  for (int l = 0; l < 8; ++l) fin = __fadd_rn(fin, acc[0][l]);
  return fin;
}

static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline int64_t align_up(int64_t a, int64_t b) { return ceil_div(a, b) * b; }

// Simple owning device buffer (build-time allocations; hot-path scratch comes from the caller's workspace).
template <typename T>
struct DevBuf {
  T* p = nullptr;
  int64_t n = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }
  // (re)allocation; a buffer that already has `count` elements is kept as it is - a field that is re-packed every
  // training step must not pay cudaFree + cudaMalloc (both synchronise the device) for buffers of unchanged size
  cudaError_t alloc(int64_t count) {
    if (p && n == count) return cudaSuccess;
    release();
    n = count;
    if (count <= 0) return cudaSuccess;
    count_alloc();
    return cudaMalloc(reinterpret_cast<void**>(&p), sizeof(T) * static_cast<size_t>(count));
  }
  // at least `count` elements: a buffer that is already large enough is kept (n stays its capacity); otherwise
  // `count + count * headroom_pct / 100` are allocated, so that a slowly varying size settles after one reallocation
  cudaError_t reserve(int64_t count, int headroom_pct = 0) {
    if (p && n >= count) return cudaSuccess;
    return alloc(count + count * headroom_pct / 100);
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    n = 0;
  }
};

int sm_count();

// nmb_set_deterministic's process-wide mode: the reducing launchers (csrc/train.cu, nmb_vertex_normals) then take
// summation orders that are a function of their inputs alone (no float atomics, no partition read from sm_count()).
bool deterministic();

// cub::DeviceRadixSort::SortPairs over bits [0, end_bit) of uint32 keys with int32 values (stable: equal keys keep
// their input order); tmp == nullptr queries tmp_bytes.  csrc/sort.cu.
cudaError_t sort_pairs_u32(void* tmp, size_t& tmp_bytes, const uint32_t* key_in, uint32_t* key_out,
                           const int32_t* val_in, int32_t* val_out, int n, int end_bit, cudaStream_t stream);

// Optional per-kernel-class device timing (bench.py's roofline): CUDA events recorded on the launching stream
// around the launches of one class.  Disabled by default (no events, no overhead).
enum ProfTag { PROF_KNN = 0, PROF_BOUND = 1, PROF_GEO = 2, PROF_GEO_JVP = 3, PROF_COLOR = 4, PROF_SAMPLER = 5, PROF_KNN_LIST = 6, PROF_N = 7 };
bool prof_enabled();
void prof_begin(int tag, int64_t units, cudaStream_t stream);
void prof_end(int tag, cudaStream_t stream);
struct ProfScope {
  int tag;
  cudaStream_t stream;
  bool on;
  ProfScope(int t, int64_t units, cudaStream_t s) : tag(t), stream(s), on(prof_enabled()) {
    if (on) prof_begin(tag, units, stream);
  }
  ~ProfScope() {
    if (on) prof_end(tag, stream);
  }
};

}  // namespace nmb
