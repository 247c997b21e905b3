// Device helpers shared by the training-path kernels (train.cu: NeuMesh field op; train_neus.cu: NeuS surface op).
#pragma once

namespace nmb {
namespace tr {

// ------------------------------------------------------------------------------------------------------------
// positional encodings (models/base.py:52-70): [x, sin(2^0 x), cos(2^0 x), sin(2^1 x), cos(2^1 x), ...]; for a
// D-vector every block spans all D components.  pe_c(x, c): component c of PE of a SCALAR (c = 0: x; c = 1 + 2b: sin;
// c = 2 + 2b: cos), its first and second derivatives.
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float pe_val(float x, int c) {
  if (c == 0) return x;
  const float f = (float)(1 << ((c - 1) >> 1));
  return ((c - 1) & 1) ? cosf(x * f) : sinf(x * f);
}
__device__ __forceinline__ float pe_d1(float x, int c) {
  if (c == 0) return 1.f;
  const float f = (float)(1 << ((c - 1) >> 1));
  return ((c - 1) & 1) ? -f * sinf(x * f) : f * cosf(x * f);
}
__device__ __forceinline__ float pe_d2(float x, int c) {
  if (c == 0) return 0.f;
  const float f = (float)(1 << ((c - 1) >> 1));
  return ((c - 1) & 1) ? -f * f * cosf(x * f) : -f * f * sinf(x * f);
}

// softplus(beta = 100, threshold = 20) and its derivatives (torch.nn.Softplus semantics)
__device__ __forceinline__ void softplus_terms(float z, float& sp, float& s1, float& s2) {
  if (z * 100.f > 20.f) {
    sp = z;
    s1 = 1.f;
    s2 = 0.f;
  } else {
    const float e = expf(100.f * z);
    sp = log1pf(e) * 0.01f;
    s1 = e / (1.f + e);
    s2 = 100.f * s1 * (1.f - s1);
  }
}

}  // namespace tr
}  // namespace nmb
