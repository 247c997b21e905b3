// NeuS surface op (neumesh_b200/neus_ops.py::FusedSurfaceFn): the element-wise primitives around the GEMMs.
//
// The surface is an MLP of softplus(beta = 100) layers over e = PE(x) (models/base.py:139-311).  The op evaluates the
// value chain z_l = W_l h_{l-1} + b_l, h_l = sp(z_l) and the reverse-mode adjoint of sdf = w_o . h_D (u_l = g_l * sp'(z_l),
// g_{l-1} = u_l W_l, starting from the broadcast row g_D = w_o); the input adjoint e_bar gives nabla = J^T e_bar with
// J = de/dx.  Derivation and backward: DESIGN.md section 4.6.  The GEMMs are nmb_tr_gemm / nmb_tr_gemm_tc; the kernels
// below are one thread per output element, with no atomics, so results do not depend on the deterministic mode.
//
//   nmb_ns_pe        out[m, c] = PE(x_m)_c, c < 3 (1 + 2L), into a destination with leading dimension ldo
//   nmb_ns_pe_jt     nabla[m, j] = sum_b e_bar[m, 3b + j] * dPE_b(x_mj)          (J^T e_bar)
//   nmb_ns_pe_j      b_e[m, 3b + j] = b_nabla[m, j] * dPE_b(x_mj)               (J b_nabla)
//   nmb_ns_softplus  h[m, n] = sp(z[m, n]), into a destination with leading dimension ldh
//   nmb_ns_gate      out[m, n] = (g ? g[m, n] : row[n]) * (z ? sp'(z[m, n]) : 1)
#include "../../include/neumesh_b200.h"
#include "common.cuh"
#include "train_common.cuh"

namespace nmb {
namespace ns {

using tr::pe_d1;
using tr::pe_val;
using tr::softplus_terms;

constexpr int THREADS = 256;

__global__ void __launch_bounds__(THREADS)
pe_kernel(int64_t M, int C, const float* __restrict__ x, float* __restrict__ out, int64_t ldo) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= M * C) return;
  const int64_t m = i / C;
  const int c = (int)(i - m * C);
  out[m * ldo + c] = pe_val(x[m * 3 + c % 3], c / 3);
}

__global__ void __launch_bounds__(THREADS)
pe_jt_kernel(int64_t M, int B, const float* __restrict__ x, const float* __restrict__ ebar, float* __restrict__ nabla) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= M * 3) return;
  const int64_t m = i / 3;
  const int j = (int)(i - m * 3);
  const float xj = x[i];
  const float* e = ebar + m * 3 * B + j;
  float s = 0.f;
  for (int b = 0; b < B; ++b) s = fmaf(e[3 * b], pe_d1(xj, b), s);
  nabla[i] = s;
}

__global__ void __launch_bounds__(THREADS)
pe_j_kernel(int64_t M, int C, const float* __restrict__ x, const float* __restrict__ b_nabla, float* __restrict__ b_e) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= M * C) return;
  const int64_t m = i / C;
  const int c = (int)(i - m * C), j = c % 3;
  b_e[i] = b_nabla[m * 3 + j] * pe_d1(x[m * 3 + j], c / 3);
}

__global__ void __launch_bounds__(THREADS)
softplus_kernel(int64_t M, int N, const float* __restrict__ z, float* __restrict__ h, int64_t ldh) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= M * N) return;
  const int64_t m = i / N;
  float sp, s1, s2;
  softplus_terms(z[i], sp, s1, s2);
  h[m * ldh + (i - m * N)] = sp;
}

__global__ void __launch_bounds__(THREADS)
gate_kernel(int64_t M, int N, const float* __restrict__ g, const float* __restrict__ row, const float* __restrict__ z,
            float* __restrict__ out) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= M * N) return;
  float v = g ? g[i] : row[i % N];
  if (z) {
    float sp, s1, s2;
    softplus_terms(z[i], sp, s1, s2);
    v *= s1;
  }
  out[i] = v;
}

static unsigned blocks(int64_t n) { return (unsigned)ceil_div(n, THREADS); }

}  // namespace ns
}  // namespace nmb

extern "C" {

int nmb_ns_pe(const float* x, int64_t M, int32_t L, float* out, int64_t ldo, void* stream) {
  if (M <= 0) return 0;   // an empty torch tensor has no storage: check nothing else
  NMB_CHECK(x && out, "null argument");
  NMB_CHECK(L >= 0 && L <= 30, "frequency bands out of range");
  const int C = 3 * (1 + 2 * L);
  NMB_CHECK(ldo >= C, "leading dimension too small");
  nmb::ns::pe_kernel<<<nmb::ns::blocks(M * C), nmb::ns::THREADS, 0, static_cast<cudaStream_t>(stream)>>>(M, C, x, out,
                                                                                                         ldo);
  NMB_LAUNCH_OK();
  return 0;
}

int nmb_ns_pe_jt(const float* x, int64_t M, int32_t L, const float* ebar, float* nabla, void* stream) {
  if (M <= 0) return 0;
  NMB_CHECK(x && ebar && nabla, "null argument");
  NMB_CHECK(L >= 0 && L <= 30, "frequency bands out of range");
  nmb::ns::pe_jt_kernel<<<nmb::ns::blocks(M * 3), nmb::ns::THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      M, 1 + 2 * L, x, ebar, nabla);
  NMB_LAUNCH_OK();
  return 0;
}

int nmb_ns_pe_j(const float* x, int64_t M, int32_t L, const float* b_nabla, float* b_e, void* stream) {
  if (M <= 0) return 0;
  NMB_CHECK(x && b_nabla && b_e, "null argument");
  NMB_CHECK(L >= 0 && L <= 30, "frequency bands out of range");
  const int C = 3 * (1 + 2 * L);
  nmb::ns::pe_j_kernel<<<nmb::ns::blocks(M * C), nmb::ns::THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      M, C, x, b_nabla, b_e);
  NMB_LAUNCH_OK();
  return 0;
}

int nmb_ns_softplus(const float* z, int64_t M, int64_t N, float* h, int64_t ldh, void* stream) {
  if (M <= 0 || N <= 0) return 0;
  NMB_CHECK(z && h, "null argument");
  NMB_CHECK(N < (int64_t(1) << 31) && ldh >= N, "bad width or leading dimension");
  nmb::ns::softplus_kernel<<<nmb::ns::blocks(M * N), nmb::ns::THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      M, (int)N, z, h, ldh);
  NMB_LAUNCH_OK();
  return 0;
}

int nmb_ns_gate(const float* g, const float* row, const float* z, int64_t M, int64_t N, float* out, void* stream) {
  if (M <= 0 || N <= 0) return 0;
  NMB_CHECK(out && (g || row), "null argument");
  NMB_CHECK(N < (int64_t(1) << 31), "width too large");
  nmb::ns::gate_kernel<<<nmb::ns::blocks(M * N), nmb::ns::THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      M, (int)N, g, row, z, out);
  NMB_LAUNCH_OK();
  return 0;
}

}  // extern "C"
