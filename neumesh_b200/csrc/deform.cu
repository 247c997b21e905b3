// Geometry editing (editing/render_geometry_editing.py:37-67, deform_model): the rotation of every vertex's indicator
// vector by the rotation that takes its old vertex normal to the new one, restated in oracle/deform.py.
//
// One thread per vertex, fp32, every operation rounded on its own (no contraction) in the order the oracle states:
//   axis = cross(n_old, n_new)                                  torch.cross
//   c    = clamp(dot(n_old, n_new) / (|n_old| |n_new|), -1, 1) cos_between_vectors
//   aa   = axis * acos(c)                                       |aa| = theta |axis|, not theta: the reference's quirk
//   R    = kornia angle_axis_to_rotation_matrix(aa)             Rodrigues above theta^2 = 1e-6, I + [aa]x below
//   out  = R @ ind, negated where c == -1 exactly
#include "../../include/neumesh_b200.h"
#include "common.cuh"

namespace nmb {

__device__ __forceinline__ float dot3_rn(float ax, float ay, float az, float bx, float by, float bz) {
  return __fadd_rn(__fadd_rn(__fmul_rn(ax, bx), __fmul_rn(ay, by)), __fmul_rn(az, bz));
}

__global__ void indicator_rotate_kernel(const float* __restrict__ n_old, const float* __restrict__ n_new,
                                        const float* ind_in, int64_t V, float* ind_out /* may alias ind_in */) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= V) return;
  const float ax = n_old[i * 3], ay = n_old[i * 3 + 1], az = n_old[i * 3 + 2];
  const float bx = n_new[i * 3], by = n_new[i * 3 + 1], bz = n_new[i * 3 + 2];
  const float vx = ind_in[i * 3], vy = ind_in[i * 3 + 1], vz = ind_in[i * 3 + 2];
  // render_geometry_editing.py:46-52
  const float cx = __fsub_rn(__fmul_rn(ay, bz), __fmul_rn(az, by));
  const float cy = __fsub_rn(__fmul_rn(az, bx), __fmul_rn(ax, bz));
  const float cz = __fsub_rn(__fmul_rn(ax, by), __fmul_rn(ay, bx));
  const float na = __fsqrt_rn(dot3_rn(ax, ay, az, ax, ay, az));
  const float nb = __fsqrt_rn(dot3_rn(bx, by, bz, bx, by, bz));
  float c = __fdiv_rn(dot3_rn(ax, ay, az, bx, by, bz), __fmul_rn(na, nb));
  if (c == c) c = fminf(fmaxf(c, -1.f), 1.f);   // torch.clamp keeps a NaN (zero-length normal); fmaxf would not
  const bool flip = (c == -1.f);     // :53
  const float ang = acosf(c);
  const float rx = __fmul_rn(cx, ang), ry = __fmul_rn(cy, ang), rz = __fmul_rn(cz, ang);
  // kornia angle_axis_to_rotation_matrix (:54-56)
  const float theta2 = dot3_rn(rx, ry, rz, rx, ry, rz);
  float R[9];
  if (theta2 > 1e-6f) {
    const float theta = __fsqrt_rn(theta2);
    const float den = __fadd_rn(theta, 1e-6f);
    const float wx = __fdiv_rn(rx, den), wy = __fdiv_rn(ry, den), wz = __fdiv_rn(rz, den);
    const float ct = cosf(theta), st = sinf(theta);
    const float omc = __fsub_rn(1.f, ct);
    R[0] = __fadd_rn(ct, __fmul_rn(__fmul_rn(wx, wx), omc));
    R[1] = __fsub_rn(__fmul_rn(__fmul_rn(wx, wy), omc), __fmul_rn(wz, st));
    R[2] = __fadd_rn(__fmul_rn(wy, st), __fmul_rn(__fmul_rn(wx, wz), omc));
    R[3] = __fadd_rn(__fmul_rn(wz, st), __fmul_rn(__fmul_rn(wx, wy), omc));
    R[4] = __fadd_rn(ct, __fmul_rn(__fmul_rn(wy, wy), omc));
    R[5] = __fadd_rn(__fmul_rn(-wx, st), __fmul_rn(__fmul_rn(wy, wz), omc));
    R[6] = __fadd_rn(__fmul_rn(-wy, st), __fmul_rn(__fmul_rn(wx, wz), omc));
    R[7] = __fadd_rn(__fmul_rn(wx, st), __fmul_rn(__fmul_rn(wy, wz), omc));
    R[8] = __fadd_rn(ct, __fmul_rn(__fmul_rn(wz, wz), omc));
  } else {
    R[0] = 1.f; R[1] = -rz; R[2] = ry;
    R[3] = rz;  R[4] = 1.f; R[5] = -rx;
    R[6] = -ry; R[7] = rx;  R[8] = 1.f;
  }
  // torch.matmul(rot_matrix, ind[..., None]) (:59-61), then deform_indicator[rot_180_mask] *= -1 (:62)
  float ox = dot3_rn(R[0], R[1], R[2], vx, vy, vz);
  float oy = dot3_rn(R[3], R[4], R[5], vx, vy, vz);
  float oz = dot3_rn(R[6], R[7], R[8], vx, vy, vz);
  if (flip) {
    ox = -ox;
    oy = -oy;
    oz = -oz;
  }
  ind_out[i * 3] = ox;
  ind_out[i * 3 + 1] = oy;
  ind_out[i * 3 + 2] = oz;
}

}  // namespace nmb

extern "C" {

int nmb_indicator_rotate(const float* n_old, const float* n_new, const float* ind_in, int64_t V, float* ind_out,
                         void* stream) {
  NMB_CHECK(n_old && n_new && ind_in && ind_out, "null argument");
  NMB_CHECK(V >= 0, "negative vertex count");
  if (V == 0) return 0;
  nmb::indicator_rotate_kernel<<<(unsigned)nmb::ceil_div(V, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      n_old, n_new, ind_in, V, ind_out);
  NMB_LAUNCH_OK();
  return 0;
}

}  // extern "C"
