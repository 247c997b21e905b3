// volume_render (models/renderer.py:105-368) for a NeuMesh field: per-ray sample placement, field evaluation and
// alpha compositing, un-batched, perturb = False, no grad.
//
// Data layout: every per-sample array of a ray chunk is SAMPLE-MAJOR, element (sample s, ray r) at [s * R + r].
// A warp therefore holds 32 neighbouring rays at one sample index: the per-ray kernels (one thread per ray) read
// and write fully coalesced, and the per-point kernels (KNN walk, MLP tiles) see spatially coherent points.
//
// Per chunk:  rays -> sphere near/far -> [256-sample mesh-distance scan -> bounded near/far]
//             -> 64 coarse samples -> 4 x { slope/alpha/cdf -> 16 inverse-cdf samples -> sdf -> merge }
//             -> sdf(+nabla) at the 128 samples, sdf+nabla+colour at the 127 mid-points -> composite.
#include <cub/cub.cuh>
#include <math_constants.h>

#include "edit.cuh"

namespace nmb {

constexpr int RT = 128;  // threads per block of the per-ray kernels

__device__ __forceinline__ float sigmoid_t(float x) { return __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-x))); }

// renderer.py:150-153 (normalise directions) + rend_util.py:179-199 (sphere near/far)
// Spatial sort key of a ray: 30-bit Morton code of its closest point to the origin (the scene centre).  Rays are
// rendered in key order so that the 32 rays of a warp form a compact patch: their octree walks then share nodes
// (coalesced loads) and hit / miss rays are not mixed inside a warp.  Outputs are written back in caller order.
__global__ void ray_key_kernel(const float* __restrict__ rays_o, const float* __restrict__ rays_d, int64_t N,
                               float radius, uint32_t* __restrict__ key, int32_t* __restrict__ idx) {
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r >= N) return;
  const float ox = rays_o[r * 3], oy = rays_o[r * 3 + 1], oz = rays_o[r * 3 + 2];
  float dx = rays_d[r * 3], dy = rays_d[r * 3 + 1], dz = rays_d[r * 3 + 2];
  const float n = fmaxf(sqrtf(dx * dx + dy * dy + dz * dz), 1e-12f);
  dx /= n; dy /= n; dz /= n;
  const float t = -(ox * dx + oy * dy + oz * dz);
  const float s = 511.5f / (2.f * radius);
  const float m[3] = {ox + t * dx, oy + t * dy, oz + t * dz};
  uint32_t q[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float v = m[c] * s + 511.5f;
    v = fminf(fmaxf(v, 0.f), 1023.f);
    q[c] = (uint32_t)v;
  }
  key[r] = (expand_bits10(q[0]) << 2) | (expand_bits10(q[1]) << 1) | expand_bits10(q[2]);
  idx[r] = (int32_t)r;
}

__global__ void ray_setup_kernel(const float* __restrict__ rays_o_all, const float* __restrict__ rays_d_all,
                                 const int32_t* __restrict__ perm, int64_t R, float radius, int normalize,
                                 float* __restrict__ orig, float* __restrict__ dirs, float* __restrict__ near,
                                 float* __restrict__ far, int32_t* __restrict__ bnear, int32_t* __restrict__ bfar) {
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r >= R) return;
  const int64_t src = perm[r];
  const float* rays_o = rays_o_all + src * 3 - r * 3;   // so that rays_o[r * 3 + c] addresses ray `src`
  const float* rays_d = rays_d_all + src * 3 - r * 3;
  orig[r * 3] = rays_o[r * 3];
  orig[r * 3 + 1] = rays_o[r * 3 + 1];
  orig[r * 3 + 2] = rays_o[r * 3 + 2];
  float dx = rays_d[r * 3], dy = rays_d[r * 3 + 1], dz = rays_d[r * 3 + 2];
  if (normalize) {
    // F.normalize: v / max(||v||, 1e-12)
    const float n = fmaxf(__fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz))), 1e-12f);
    dx = __fdiv_rn(dx, n);
    dy = __fdiv_rn(dy, n);
    dz = __fdiv_rn(dz, n);
  }
  dirs[r * 3] = dx;
  dirs[r * 3 + 1] = dy;
  dirs[r * 3 + 2] = dz;
  const float ox = rays_o[r * 3], oy = rays_o[r * 3 + 1], oz = rays_o[r * 3 + 2];
  const float mid = -__fadd_rn(__fadd_rn(__fmul_rn(ox, dx), __fmul_rn(oy, dy)), __fmul_rn(oz, dz));
  near[r] = fmaxf(__fsub_rn(mid, radius), 0.f);
  far[r] = fmaxf(__fadd_rn(mid, radius), radius);
  bnear[r] = 0x7f800000;  // +inf as ordered int (depths are >= 0)
  bfar[r] = -1;
}

// renderer.py:91-101
__global__ void bound_finish_kernel(int64_t R, const int32_t* __restrict__ bnear, const int32_t* __restrict__ bfar,
                                    float* __restrict__ near, float* __restrict__ far) {
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r >= R) return;
  float n = near[r], f = far[r];
  if (bfar[r] >= 0) {  // at least one sample inside the shell: both extrema exist
    n = __int_as_float(bnear[r]);
    f = __int_as_float(bfar[r]);
  }
  if (__fsub_rn(f, n) < 0.1f) {
    f = __fadd_rn(f, 0.05f);
    n = __fsub_rn(n, 0.05f);
  }
  near[r] = n;
  far[r] = f;
}

__global__ void bypass_kernel(int64_t R, int use_near, float nb, int use_far, float fb, float* __restrict__ near,
                              float* __restrict__ far) {
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r >= R) return;
  if (use_near) near[r] = nb;
  if (use_far) far[r] = fb;
}

// renderer.py:193-194: z[s][r] = near * (1 - t_s) + far * t_s
__global__ void coarse_z_kernel(int64_t R, int S, const float* __restrict__ near, const float* __restrict__ far,
                                float* __restrict__ z, int32_t* __restrict__ origin) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= R * S) return;
  const int64_t r = i % R;
  const int s = (int)(i / R);
  const float t = linspace01(s, S);
  z[i] = __fadd_rn(__fmul_rn(near[r], __fsub_rn(1.0f, t)), __fmul_rn(far[r], t));
  if (origin) origin[i] = s;   // sample s of ray r was evaluated as entry s of the neighbour arrays
}

// One up-sampling iteration for one ray (renderer.py:209-245 + rend_util.py:276-319 with det=True).
// n = current number of samples; writes n_new new depths (ascending) to znew[i][r].
__global__ void __launch_bounds__(RT)
upsample_kernel(int64_t R, int n, int n_new, float inv_s, const float* __restrict__ z, const float* __restrict__ sdf,
                float* __restrict__ wbuf, float* __restrict__ znew, const float* __restrict__ u_arr /*[n_new][Nu] or null*/,
                int64_t Nu, const int32_t* __restrict__ perm /*chunk ray -> caller ray (u_arr's column), or null*/) {
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r >= R) return;
  // pass 1: weights (sequential cumprod, as torch's CPU cumprod); their sum afterwards in torch's order
  float z0 = z[r], s0 = sdf[r];
  float prev_raw = 0.f;  // "prev_dot_val": raw slope of the previous interval, 0 for the first
  // torch's CPU cumprod / cumsum accumulate fp32 rows in DOUBLE (at::acc_type<float, false>) and round every output
  // element to fp32: the running product / sum below are kept in double exactly like that
  double T = 1.0;
  for (int j = 0; j + 1 < n; ++j) {
    const float z1 = z[(int64_t)(j + 1) * R + r], s1 = sdf[(int64_t)(j + 1) * R + r];
    const float mid = __fmul_rn(__fadd_rn(s0, s1), 0.5f);
    const float raw = __fdiv_rn(__fsub_rn(s1, s0), __fadd_rn(__fsub_rn(z1, z0), 1e-5f));
    float slope = fminf(prev_raw, raw);
    slope = fminf(fmaxf(slope, -10.0f), 0.0f);
    prev_raw = raw;
    const float dist = __fsub_rn(z1, z0);
    const float half = __fmul_rn(__fmul_rn(slope, dist), 0.5f);
    const float c0 = sigmoid_t(__fmul_rn(__fsub_rn(mid, half), inv_s));
    const float c1 = sigmoid_t(__fmul_rn(__fadd_rn(mid, half), inv_s));
    const float alpha = __fdiv_rn(__fadd_rn(__fsub_rn(c0, c1), 1e-5f), __fadd_rn(c0, 1e-5f));
    const float w = __fadd_rn(__fmul_rn(alpha, (float)T), 1e-5f);  // alpha_to_w, then sample_pdf's "+ 1e-5"
    T = __dmul_rn(T, (double)__fadd_rn(__fsub_rn(1.0f, alpha), 1e-10f));
    wbuf[(int64_t)j * R + r] = w;
    z0 = z1;
    s0 = s1;
  }
  const float total = torch_row_sum(wbuf + r, R, n - 1);
  // pass 2: inverse CDF at u_i = linspace(0,1,n_new); searchsorted(right=False): first j with cdf[j] >= u
  int i = 0;
  const int64_t ucol = u_arr ? (perm ? (int64_t)perm[r] : r) : 0;
  auto u_at = [&](int k) { return u_arr ? u_arr[(int64_t)k * Nu + ucol] : linspace01(k, n_new); };
  float u = u_at(0);
  float cdf_prev = 0.f;           // cdf[j-1]
  float bin_prev = z[r];          // bins[j-1]
  float cdf_j = 0.f;              // cdf[0] = 0
  double cdf_acc = 0.0;           // torch.cumsum's double accumulator
  float bin_j = bin_prev;
  for (int j = 0; j < n && i < n_new; ++j) {
    if (j > 0) {
      cdf_prev = cdf_j;
      bin_prev = bin_j;
      cdf_acc = __dadd_rn(cdf_acc, (double)__fdiv_rn(wbuf[(int64_t)(j - 1) * R + r], total));
      cdf_j = (float)cdf_acc;
      bin_j = z[(int64_t)j * R + r];
    }
    while (i < n_new && cdf_j >= u) {
      // inds = j: below = max(j-1, 0), above = min(j, n-1) = j
      const float cb = (j > 0) ? cdf_prev : cdf_j;
      const float bb = (j > 0) ? bin_prev : bin_j;
      float denom = __fsub_rn(cdf_j, cb);
      if (denom < 1e-5f) denom = 1.0f;
      const float t = __fdiv_rn(__fsub_rn(u, cb), denom);
      znew[(int64_t)i * R + r] = __fadd_rn(bb, __fmul_rn(t, __fsub_rn(bin_j, bb)));
      ++i;
      if (i < n_new) u = u_at(i);
    }
  }
  // u above the last cdf entry: inds = n -> below = above = n-1 -> denom = 0 -> 1 -> sample = bins[n-1]
  for (; i < n_new; ++i) znew[(int64_t)i * R + r] = bin_j;
}

// Merge the n_new ascending new samples into the n sorted ones (renderer.py:246,256-258: cat + sort + gather),
// in place, from the back.  Ties: either order is equivalent (tied depths carry bit-identical sdf values).
__global__ void __launch_bounds__(RT)
merge_kernel(int64_t R, int n, int n_new, float* __restrict__ z, float* __restrict__ sdf,
             const float* __restrict__ znew, const float* __restrict__ sdfnew, float* __restrict__ nab,
             const float* __restrict__ nabnew, int64_t nstride, int32_t* __restrict__ origin, int origin_new, int dup0) {
  // dup0: new sample 0 was NOT evaluated - it is the ray's current first sample again (deterministic up-sampling:
  // u = 0 returns bins[0] exactly), so its sdf / nabla / origin are copied from sample 0, which is still in place when
  // new sample 0 is merged (z[0] == znew[0] is never taken before it)
  // origin (nullable): [P][R] index of the evaluation pass entry a sample came from (the KNN results of every pass
  // stay in place: entry e of ray r lives at position e * R + r); new sample b gets origin_new + b
  // nab / nabnew (nullable): [3][nstride] SoA payload (nabla at the samples) carried through the merge
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r >= R) return;
  int a = n - 1, b = n_new - 1;
  float za = z[(int64_t)a * R + r], zb = znew[(int64_t)b * R + r];
  for (int o = n + n_new - 1; o >= 0 && b >= 0; --o) {
    const int64_t dst = (int64_t)o * R + r;
    if (a >= 0 && za > zb) {
      const int64_t src = (int64_t)a * R + r;
      z[dst] = za;
      sdf[dst] = sdf[src];
      if (origin) origin[dst] = origin[src];
      if (nab) {
        nab[dst] = nab[src];
        nab[nstride + dst] = nab[nstride + src];
        nab[2 * nstride + dst] = nab[2 * nstride + src];
      }
      --a;
      if (a >= 0) za = z[(int64_t)a * R + r];
    } else {
      const int64_t src = (int64_t)b * R + r;
      const bool copy0 = dup0 && b == 0;
      z[dst] = zb;
      sdf[dst] = copy0 ? sdf[r] : sdfnew[src];
      if (origin) origin[dst] = copy0 ? origin[r] : origin_new + b;
      if (nab) {
        nab[dst] = copy0 ? nab[r] : nabnew[src];
        nab[nstride + dst] = copy0 ? nab[nstride + r] : nabnew[nstride + src];
        nab[2 * nstride + dst] = copy0 ? nab[2 * nstride + r] : nabnew[2 * nstride + src];
      }
      --b;
      if (b >= 0) zb = znew[(int64_t)b * R + r];
    }
  }
}

// renderer.py:266: d_mid = 0.5 * (d_all[1:] + d_all[:-1])
__global__ void midpoints_kernel(int64_t R, int P, const float* __restrict__ z, float* __restrict__ zmid) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= R * (P - 1)) return;
  zmid[i] = __fmul_rn(0.5f, __fadd_rn(z[i + R], z[i]));
}

// ---- compositing ---------------------------------------------------------------------------------------------
// The reference multiplies every mid-point colour, depth and point normal by its visibility weight
// (renderer.py:304-333).  Where that weight is exactly 0.0f - in front of the shell (sigmoid saturates to 1), behind
// the surface (transmittance underflows), on rays that miss - the colour MLP, the mid-point nabla and the KNN walk
// feeding them cannot influence any composited output.  The live-sample path (cfg.skip_dead_samples) therefore
// computes the weights first, compacts the samples with a non-zero weight and evaluates only those; the composite
// then adds exactly the same non-zero terms in the same order, so rgb / depth / acc / normals are bit-identical to
// evaluating everything.  Both paths composite from the weights of weights_kernel.

// renderer.py:17-24 (sdf_to_alpha), :49-63 (alpha_to_w): weights + number of live (non-zero weight) samples per ray
__global__ void __launch_bounds__(RT)
weights_kernel(int64_t R, int P, float s, const float* __restrict__ sdf, float* __restrict__ wbuf,
               int32_t* __restrict__ nlive) {
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r >= R) return;
  float c0 = sigmoid_t(__fmul_rn(sdf[r], s));
  double T = 1.0;   // torch.cumprod on the CPU accumulates in double (see upsample_kernel)
  int n = 0;
  for (int j = 0; j + 1 < P; ++j) {
    const int64_t q = (int64_t)j * R + r;
    const float c1 = sigmoid_t(__fmul_rn(sdf[q + R], s));
    const float alpha = fmaxf(__fdiv_rn(__fsub_rn(c0, c1), __fadd_rn(c0, 1e-10f)), 0.f);
    const float w = __fmul_rn(alpha, (float)T);
    T = __dmul_rn(T, (double)__fadd_rn(__fsub_rn(1.0f, alpha), 1e-10f));
    wbuf[q] = w;
    n += (w != 0.f) ? 1 : 0;
    c0 = c1;
  }
  nlive[r] = n;
}

// compact the live samples of every ray: mid-point position + view direction (+ sample position for the normals)
__global__ void __launch_bounds__(RT)
compact_live_kernel(int64_t R, int P, const int32_t* __restrict__ off, const float* __restrict__ wbuf,
                    const float* __restrict__ z, const float* __restrict__ zmid, const float* __restrict__ orig,
                    const float* __restrict__ dirs, float* __restrict__ xyz_mid, float* __restrict__ dir_live,
                    float* __restrict__ xyz_pt /*nullable*/, const int32_t* __restrict__ origin /*nullable*/,
                    int32_t* __restrict__ live_src /*nullable: position of the live point's neighbour data*/) {
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r >= R) return;
  const float ox = orig[r * 3], oy = orig[r * 3 + 1], oz = orig[r * 3 + 2];
  const float dx = dirs[r * 3], dy = dirs[r * 3 + 1], dz = dirs[r * 3 + 2];
  int64_t k = off[r];
  for (int j = 0; j + 1 < P; ++j) {
    const int64_t q = (int64_t)j * R + r;
    if (wbuf[q] != 0.f) {
      const float zm = zmid[q];
      xyz_mid[k * 3 + 0] = __fadd_rn(ox, __fmul_rn(zm, dx));
      xyz_mid[k * 3 + 1] = __fadd_rn(oy, __fmul_rn(zm, dy));
      xyz_mid[k * 3 + 2] = __fadd_rn(oz, __fmul_rn(zm, dz));
      dir_live[k * 3 + 0] = dx;
      dir_live[k * 3 + 1] = dy;
      dir_live[k * 3 + 2] = dz;
      if (xyz_pt) {
        const float zp = z[q];
        xyz_pt[k * 3 + 0] = __fadd_rn(ox, __fmul_rn(zp, dx));
        xyz_pt[k * 3 + 1] = __fadd_rn(oy, __fmul_rn(zp, dy));
        xyz_pt[k * 3 + 2] = __fadd_rn(oz, __fmul_rn(zp, dz));
      }
      if (live_src) live_src[k] = (int32_t)((int64_t)origin[q] * R + r);
      ++k;
    }
  }
}

// renderer.py:299-333 (integration, white background, normals) from the weights of weights_kernel.
// off == nullptr: every sample adds its term, as the reference does (0 * NaN stays NaN); colour and nabla of mid-point
//   j are read sample-major at [c * stride + j * R + r].
// off != nullptr (live path): only the terms with a non-zero weight; colour and nabla of the i-th live sample of ray r
//   are read from the compacted list at [c * stride + off[r] + i].
__global__ void __launch_bounds__(RT)
composite_kernel(int64_t R, int P, int white_bkgd, const float* __restrict__ wbuf, const float* __restrict__ zmid,
                 const int32_t* __restrict__ off, const float* __restrict__ rgb /*[3][cstride]*/, int64_t cstride,
                 const float* __restrict__ nabla /*[3][nstride] or null*/, int64_t nstride,
                 const int32_t* __restrict__ perm, float* __restrict__ rgb_out, float* __restrict__ depth_out,
                 float* __restrict__ acc_out, float* __restrict__ normals_out) {
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r >= R) return;
  const int64_t dst = perm[r];   // caller's ray index
  float acc = 0.f, cr = 0.f, cg = 0.f, cb = 0.f, nx = 0.f, ny = 0.f, nz = 0.f;
  int64_t k = off ? off[r] : 0;  // next live-list entry
  for (int j = 0; j + 1 < P; ++j) {
    const int64_t q = (int64_t)j * R + r;
    const float w = wbuf[q];
    if (off && w == 0.f) continue;
    const int64_t i = off ? k++ : q;
    acc = __fadd_rn(acc, w);
    cr = __fadd_rn(cr, __fmul_rn(w, rgb[i]));
    cg = __fadd_rn(cg, __fmul_rn(w, rgb[cstride + i]));
    cb = __fadd_rn(cb, __fmul_rn(w, rgb[2 * cstride + i]));
    if (nabla) {
      const float gx = nabla[i], gy = nabla[nstride + i], gz = nabla[2 * nstride + i];
      const float nn = fmaxf(__fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)), __fmul_rn(gz, gz))), 1e-12f);
      nx = __fadd_rn(nx, __fmul_rn(__fdiv_rn(gx, nn), w));
      ny = __fadd_rn(ny, __fmul_rn(__fdiv_rn(gy, nn), w));
      nz = __fadd_rn(nz, __fmul_rn(__fdiv_rn(gz, nn), w));
    }
  }
  const float den = __fadd_rn(acc, 1e-10f);
  float depth = 0.f;
  for (int j = 0; j + 1 < P; ++j) {
    const int64_t q = (int64_t)j * R + r;
    const float w = wbuf[q];
    if (!off || w != 0.f) depth = __fadd_rn(depth, __fmul_rn(__fdiv_rn(w, den), zmid[q]));
  }
  if (white_bkgd) {
    const float bg = __fsub_rn(1.0f, acc);
    cr = __fadd_rn(cr, bg);
    cg = __fadd_rn(cg, bg);
    cb = __fadd_rn(cb, bg);
  }
  rgb_out[dst * 3] = cr;
  rgb_out[dst * 3 + 1] = cg;
  rgb_out[dst * 3 + 2] = cb;
  depth_out[dst] = depth;
  acc_out[dst] = acc;
  if (normals_out) {
    normals_out[dst * 3] = nx;
    normals_out[dst * 3 + 1] = ny;
    normals_out[dst * 3 + 2] = nz;
  }
}

// [S][R] sample-major -> [R,S] row-major (detail outputs); C channels with source stride cstride: out [R,S,C]
__global__ void export_samples_kernel(int64_t R, int S, int C, const float* __restrict__ src, int64_t cstride,
                                      const int32_t* __restrict__ perm, float* __restrict__ dst) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= R * S * C) return;
  const int c = (int)(i % C);
  const int64_t t = i / C;
  const int s = (int)(t % S);
  const int64_t r = t / S;
  dst[((int64_t)perm[r] * S + s) * C + c] = src[c * cstride + (int64_t)s * R + r];
}

__global__ void export_near_far_kernel(int64_t R, const float* __restrict__ near, const float* __restrict__ far,
                                       const int32_t* __restrict__ perm, float* __restrict__ dst) {
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r >= R) return;
  dst[(int64_t)perm[r] * 2] = near[r];
  dst[(int64_t)perm[r] * 2 + 1] = far[r];
}

// utils/rend_util.py:97-176: pixel (x, y) -> K^-1 -> normalise -> rotate
__global__ void get_rays_kernel(int H, int W, float fx, float fy, float cx, float cy, float sk, float r00, float r01,
                                float r02, float r10, float r11, float r12, float r20, float r21, float r22, float tx,
                                float ty, float tz, float* __restrict__ rays_o, float* __restrict__ rays_d) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)H * W) return;
  const float x = (float)(i % W), y = (float)(i / W);
  // lift(): x_lift = (x - cx + cy*sk/fy - sk*y/fy) / fx * z ; y_lift = (y - cy) / fy * z ; z = 1
  const float xl = __fdiv_rn(__fsub_rn(__fadd_rn(__fsub_rn(x, cx), __fdiv_rn(__fmul_rn(cy, sk), fy)),
                                        __fdiv_rn(__fmul_rn(sk, y), fy)), fx);
  const float yl = __fdiv_rn(__fsub_rn(y, cy), fy);
  const float n = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(xl, xl), __fmul_rn(yl, yl)), 1.0f));
  const float dx = __fdiv_rn(xl, n), dy = __fdiv_rn(yl, n), dz = __fdiv_rn(1.0f, n);
  rays_d[i * 3 + 0] = r00 * dx + r01 * dy + r02 * dz;
  rays_d[i * 3 + 1] = r10 * dx + r11 * dy + r12 * dz;
  rays_d[i * 3 + 2] = r20 * dx + r21 * dy + r22 * dz;
  rays_o[i * 3 + 0] = tx;
  rays_o[i * 3 + 1] = ty;
  rays_o[i * 3 + 2] = tz;
}

__global__ void pack_bgr8_kernel(const float* __restrict__ rgb, int64_t N, uint8_t* __restrict__ out) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= N) return;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float v = fminf(fmaxf(rgb[i * 3 + c], 0.f), 1.f) * 255.f;
    out[i * 3 + (2 - c)] = (uint8_t)v;
  }
}

// models/ray_casting.py:96-160 (root_finding_surface_points): per ray, the first sign change of val - tau along the
// N_steps proposals; kept only if it goes from positive (outside) to negative (inside) and the first proposal is not
// occupied.  Outputs the bracket of the secant search.  val is row-major [N, n_steps].
__global__ void first_crossing_kernel(int64_t N, int n_steps, float tau, const float* __restrict__ val,
                                      const float* __restrict__ near, const float* __restrict__ far,
                                      float* __restrict__ d_low, float* __restrict__ f_low, float* __restrict__ d_high,
                                      float* __restrict__ f_high, uint8_t* __restrict__ mask,
                                      uint8_t* __restrict__ mask_sign_change, uint8_t* __restrict__ first_free) {
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r >= N) return;
  const float* v = val + r * n_steps;
  const float v0 = v[0] - tau;
  int idx = -1;
  float prev = v0;
  for (int i = 0; i + 1 < n_steps; ++i) {
    const float cur = v[i + 1] - tau;
    if (prev * cur < 0.f) {   // torch.sign(val[i] * val[i+1]) == -1: the minimum of sign * (N_steps - i) picks the first
      idx = i;
      break;
    }
    prev = cur;
  }
  const bool change = idx >= 0;
  const bool pos_to_neg = change && (v[idx] - tau) > 0.f;
  const bool free0 = v0 > 0.f;
  const bool m = change && pos_to_neg && free0;
  mask[r] = m ? 1 : 0;
  mask_sign_change[r] = change ? 1 : 0;
  first_free[r] = free0 ? 1 : 0;
  const int i0 = change ? idx : 0, i1 = change ? min(idx + 1, n_steps - 1) : 0;
  const float n = near[r], f = far[r];
  const float t0 = linspace01(i0, n_steps), t1 = linspace01(i1, n_steps);
  d_high[r] = __fadd_rn(__fmul_rn(n, __fsub_rn(1.0f, t0)), __fmul_rn(f, t0));   // the proposal BEFORE the crossing
  f_high[r] = v[i0] - tau;
  d_low[r] = __fadd_rn(__fmul_rn(n, __fsub_rn(1.0f, t1)), __fmul_rn(f, t1));
  f_low[r] = v[i1] - tau;
}

__global__ void face_normals_kernel(const float* __restrict__ v, const int32_t* __restrict__ tri, int64_t T,
                                    float* __restrict__ acc) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= T) return;
  const int32_t a = tri[t * 3], b = tri[t * 3 + 1], c = tri[t * 3 + 2];
  const float ax = v[a * 3], ay = v[a * 3 + 1], az = v[a * 3 + 2];
  const float ux = v[b * 3] - ax, uy = v[b * 3 + 1] - ay, uz = v[b * 3 + 2] - az;
  const float wx = v[c * 3] - ax, wy = v[c * 3 + 1] - ay, wz = v[c * 3 + 2] - az;
  const float nx = uy * wz - uz * wy, ny = uz * wx - ux * wz, nz = ux * wy - uy * wx;
  const int32_t ids[3] = {a, b, c};
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    atomicAdd(acc + (int64_t)ids[k] * 3 + 0, nx);
    atomicAdd(acc + (int64_t)ids[k] * 3 + 1, ny);
    atomicAdd(acc + (int64_t)ids[k] * 3 + 2, nz);
  }
}

// Deterministic vertex normals: the corner list (key = vertex id, value = corner 3 t + j) sorted stably by vertex; the
// first corner of every vertex's run adds the run's face normals in triangle order.
__global__ void corner_list_kernel(const int32_t* __restrict__ tri, int64_t n, uint32_t* __restrict__ key,
                                   int32_t* __restrict__ corner) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  key[i] = (uint32_t)tri[i];
  corner[i] = (int32_t)i;
}

__global__ void vertex_normal_runs_kernel(const float* __restrict__ v, const int32_t* __restrict__ tri, int64_t n,
                                          const uint32_t* __restrict__ key, const int32_t* __restrict__ corner,
                                          float* __restrict__ acc) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n || (i > 0 && key[i] == key[i - 1])) return;
  float sx = 0.f, sy = 0.f, sz = 0.f;
  for (int64_t j = i; j < n && key[j] == key[i]; ++j) {
    const int64_t t = corner[j] / 3;
    const int32_t a = tri[t * 3], b = tri[t * 3 + 1], c = tri[t * 3 + 2];
    const float ax = v[a * 3], ay = v[a * 3 + 1], az = v[a * 3 + 2];
    const float ux = v[b * 3] - ax, uy = v[b * 3 + 1] - ay, uz = v[b * 3 + 2] - az;
    const float wx = v[c * 3] - ax, wy = v[c * 3 + 1] - ay, wz = v[c * 3 + 2] - az;
    sx += uy * wz - uz * wy;
    sy += uz * wx - ux * wz;
    sz += ux * wy - uy * wx;
  }
  const int64_t k = key[i];
  acc[k * 3] = sx;
  acc[k * 3 + 1] = sy;
  acc[k * 3 + 2] = sz;
}

__global__ void normalize_rows_kernel(float* __restrict__ n, int64_t V) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= V) return;
  const float x = n[i * 3], y = n[i * 3 + 1], z = n[i * 3 + 2];
  float l = sqrtf(x * x + y * y + z * z);
  if (l == 0.f) l = 1.f;
  n[i * 3] = x / l;
  n[i * 3 + 1] = y / l;
  n[i * 3 + 2] = z / l;
}

}  // namespace nmb

namespace {

struct Workspace {
  // all sizes in floats
  float *orig, *dirs, *near, *far;
  int32_t *bnear, *bfar;
  float *z, *sdf, *znew, *sdfnew, *wbuf, *zmid;
  float *k_ds, *k_w, *k_grad;
  int32_t* k_slot;
  float *nabla_pts, *nabla_mid, *sdf_mid, *rgb;
  float *live_mid, *live_dir, *live_pt;   // [M,3] positions / directions of the live samples (M <= (P-1) R)
  int32_t *nlive, *live_off;
  int32_t *origin, *live_src;             // [P][R] pass entry of every final sample; [M] neighbour-data position of a live point
  void* scan_tmp;
  int64_t scan_bytes;
  int64_t total;
};

Workspace carve(void* base, int64_t R, int P, int n_new) {
  Workspace w{};
  float* p = static_cast<float*>(base);
  int64_t off = 0;
  auto take = [&](int64_t n) {
    float* q = p ? p + off : nullptr;
    off += nmb::align_up(n, 64);
    return q;
  };
  const int64_t PR = (int64_t)P * R;
  w.orig = take(3 * R);
  w.dirs = take(3 * R);
  w.near = take(R);
  w.far = take(R);
  w.bnear = reinterpret_cast<int32_t*>(take(R));
  w.bfar = reinterpret_cast<int32_t*>(take(R));
  w.z = take(PR);
  w.sdf = take(PR);
  w.znew = take((int64_t)n_new * R);
  w.sdfnew = take((int64_t)n_new * R);
  w.wbuf = take(PR);
  w.zmid = take(PR);
  w.k_ds = take(PR);
  w.k_slot = reinterpret_cast<int32_t*>(take(8 * PR));
  w.k_w = take(8 * PR);
  w.k_grad = take(3 * PR);
  w.nabla_pts = take(3 * PR);
  w.nabla_mid = take(3 * PR);
  w.sdf_mid = take(PR);
  w.rgb = take(3 * PR);
  w.live_mid = take(3 * PR);
  w.live_dir = take(3 * PR);
  w.live_pt = take(3 * PR);
  w.nlive = reinterpret_cast<int32_t*>(take(R));
  w.live_off = reinterpret_cast<int32_t*>(take(R + 1));
  w.origin = reinterpret_cast<int32_t*>(take(PR));
  w.live_src = reinterpret_cast<int32_t*>(take(PR));
  w.scan_bytes = 16 * 1024 + R / 32;   // cub::DeviceScan temp storage (a few KB; generous)
  w.scan_tmp = take(w.scan_bytes / 4 + 1);
  w.total = off;
  return w;
}

}  // namespace

extern "C" {

int64_t nmb_render_workspace_bytes(const nmb_render_cfg* cfg, int64_t rays_per_chunk) {
  if (!cfg || rays_per_chunk <= 0) return 0;
  const int P = cfg->N_samples + cfg->N_importance;
  const int n_new = cfg->N_upsample_iters > 0 ? cfg->N_importance / cfg->N_upsample_iters : 0;
  return carve(nullptr, rays_per_chunk, P, n_new > 0 ? n_new : 1).total * (int64_t)sizeof(float) + 256;
}

int64_t nmb_render_edit_workspace_bytes(const nmb_render_cfg* cfg, const nmb_edit* edit, int64_t rays_per_chunk) {
  const int64_t base = nmb_render_workspace_bytes(cfg, rays_per_chunk);
  if (!edit || base == 0) return base;
  // the edit pass runs over at most every mid-point of a chunk
  const int64_t points = (int64_t)(cfg->N_samples + cfg->N_importance - 1) * rays_per_chunk;
  return base + nmb::edit_carve(nullptr, points).total * (int64_t)sizeof(float);
}

}  // extern "C"

namespace {

using namespace nmb;

// What every stage of a chunk reads.  The chunk's rays are perm[0..R): chunk-local ray r is the caller's ray perm[r].
struct Chunk {
  const nmb_field* f;
  const nmb_edit* edit;      // nullable
  const nmb_render_cfg* cfg;
  int64_t N;                 // rays of the call (columns of cfg->perturb_u)
  int64_t R;
  int P, n_new;
  const int32_t* perm;
  Workspace w;
  EditScratch es;
  cudaStream_t stream;
  unsigned rb;               // blocks of the per-ray kernels
};

// rays -> origin, direction, near / far (renderer.py:150-191): sphere, [bounded mesh-distance scan], [bypass]
int setup_rays(const Chunk& c, const float* rays_o, const float* rays_d) {
  const nmb_render_cfg* cfg = c.cfg;
  const Workspace& w = c.w;
  ray_setup_kernel<<<c.rb, RT, 0, c.stream>>>(rays_o, rays_d, c.perm, c.R, cfg->obj_bounding_radius,
                                              cfg->normalize_dirs, w.orig, w.dirs, w.near, w.far, w.bnear, w.bfar);
  NMB_LAUNCH_OK();
  if (cfg->bounded_near_far) {
    ShellGrid shell{};
    if (c.R >= 65536) {   // the certificate costs ~0.1-0.3 s to build: only worth it for frame-sized renders
      int rc = ensure_shell_grid(c.f, c.stream);
      if (rc) return rc;
      shell = c.f->shell;
    }
    int rc = launch_bound_scan(c.f->grid, c.f->indicator.p, c.f->w1, w.orig, w.dirs, w.near, w.far, c.R, 256, 0.1f,
                               w.bnear, w.bfar, shell, c.stream);
    if (rc) return rc;
    bound_finish_kernel<<<c.rb, RT, 0, c.stream>>>(c.R, w.bnear, w.bfar, w.near, w.far);
    NMB_LAUNCH_OK();
  }
  if (cfg->use_near_bypass || cfg->use_far_bypass) {
    bypass_kernel<<<c.rb, RT, 0, c.stream>>>(c.R, cfg->use_near_bypass, cfg->near_bypass, cfg->use_far_bypass,
                                             cfg->far_bypass, w.near, w.far);
    NMB_LAUNCH_OK();
  }
  return 0;
}

// The field at n points whose neighbours `in` describes: sdf, and nabla where non-null; with colour also the colour
// MLP and the edit's blend, into w.rgb ([3][in.stride] SoA) at the view directions in.dirs or in.rays_d.
int eval_field(const Chunk& c, FieldIn in, int64_t n, float* sdf, float* nabla, bool color) {
  int rc = launch_geo(c.f, in, n, sdf, nabla, c.stream);
  if (rc || !color) return rc;
  in.nabla = nabla;
  rc = launch_color(c.f, in, n, c.w.rgb, c.stream);
  if (rc || !c.edit) return rc;
  return apply_edit(c.edit, in, n, c.w.rgb, c.es, c.stream);
}

// The field at S samples z [S][R] of every ray.  Their neighbours are stored as pass entries entry0.. of the
// neighbour arrays (entry e of ray r at position e * R + r).
int eval_samples(const Chunk& c, const float* z, int S, float* sdf, float* nabla, bool color, int64_t entry0) {
  const Workspace& w = c.w;
  const int64_t o = entry0 * c.R;   // first position of this pass in the neighbour arrays
  KnnOut ko{w.k_ds + o, w.k_slot + o, w.k_w + o, w.k_grad + o, (int64_t)c.P * c.R};
  PointSrc src{nullptr, w.orig, w.dirs, z, c.R};
  if (entry0 > 0) {
    // an up-sampling pass: the first new sample of a ray (u = 0 reproduces the ray's first sample exactly) starts
    // from the stored neighbours of the ray's current first sample instead of a cold walk
    src.seed_slot = w.k_slot;
    src.seed_entry = w.origin;        // row 0 of origin: pass entry of sample 0 of every ray
    src.seed_stride = (int64_t)c.P * c.R;
  }
  int rc = launch_knn_distance(c.f->grid, c.f->indicator.p, c.f->w1, src, (int64_t)S * c.R, ko, c.stream);
  if (rc) return rc;
  FieldIn in(ko);
  in.rays_d = w.dirs;
  in.R = c.R;
  return eval_field(c, in, (int64_t)S * c.R, sdf, nabla, color);
}

// The sampling cascade (renderer.py:193-259): coarse samples, then N_upsample_iters x {inverse-cdf samples -> sdf ->
// merge}.  Leaves the P sorted depths and their sdf in w.z / w.sdf, and the nabla at them in nab_pts if non-null.
int sample_cascade(const Chunk& c, float* nab_pts) {
  const Workspace& w = c.w;
  const int64_t R = c.R;
  int n = c.cfg->N_samples;
  // The live path with normals needs sdf' and the neighbours of its live sample points again at the end.  Every pass
  // therefore leaves its KNN results in place (coarse samples are entries 0..N_samples-1, iteration `it` adds
  // N_samples + it * n_new ...) and an `origin` index is carried through the merges, so that pass GATHERS instead of
  // walking the octree again (cheap: pointer offsets + one int32 per sample through the merges).
  coarse_z_kernel<<<(unsigned)ceil_div(R * n, 256), 256, 0, c.stream>>>(R, n, w.near, w.far, w.z, w.origin);
  NMB_LAUNCH_OK();
  // The reference evaluates the P final samples a second time (renderer.py:271-274: forward_with_nablas when
  // calc_normal, forward_density_only otherwise).  They are the very points of the coarse / up-sampling passes, so
  // their sdf is already known (same point, same kernel => same bits) and the nabla, when carried, is obtained in
  // those passes too (tangent rows) and carried through the merges: no second KNN walk, no second MLP pass.
  float* nab_new = nab_pts ? w.nabla_mid : nullptr;   // free until the mid-point pass
  int rc = eval_samples(c, w.z, n, w.sdf, nab_pts, false, 0);
  if (rc) return rc;
  const float* u = c.cfg->perturb_u;
  for (int it = 0; it < c.cfg->N_upsample_iters; ++it) {
    upsample_kernel<<<c.rb, RT, 0, c.stream>>>(R, n, c.n_new, 256.0f * (float)(1 << it), w.z, w.sdf, w.wbuf, w.znew,
                                               u ? u + (int64_t)it * c.n_new * c.N : nullptr, c.N, c.perm);
    NMB_LAUNCH_OK();
    // deterministic up-sampling: u_0 = 0 returns the ray's first sample again, bit for bit (upsample_kernel: j = 0,
    // denom -> 1, t = 0) - the same point through the same kernels gives the same sdf, so it is not evaluated twice
    const int dup0 = (u == nullptr && c.n_new > 1) ? 1 : 0;
    rc = eval_samples(c, w.znew + dup0 * R, c.n_new - dup0, w.sdfnew + dup0 * R, nab_new ? nab_new + dup0 * R : nullptr,
                      false, n + dup0);
    if (rc) return rc;
    merge_kernel<<<c.rb, RT, 0, c.stream>>>(R, n, c.n_new, w.z, w.sdf, w.znew, w.sdfnew, nab_pts, nab_new,
                                            (int64_t)c.P * R, w.origin, n, dup0);
    NMB_LAUNCH_OK();
    n += c.n_new;
  }
  return 0;
}

// Live path: compact the mid-points with a non-zero weight (*M of them) and evaluate only those; with normals also
// the nabla at the live sample points, into w.nabla_pts.
int eval_live(const Chunk& c, float* mid_nabla, int64_t* M) {
  const Workspace& w = c.w;
  const int64_t R = c.R;
  size_t need = 0;
  NMB_CUDA_OK(cub::DeviceScan::ExclusiveSum(nullptr, need, w.nlive, w.live_off, (int)R, c.stream));
  NMB_CHECK((int64_t)need <= w.scan_bytes, "scan scratch too small");
  size_t sb = (size_t)w.scan_bytes;
  NMB_CUDA_OK(cub::DeviceScan::ExclusiveSum(w.scan_tmp, sb, w.nlive, w.live_off, (int)R, c.stream));
  count_launch(2);
  int32_t last_off = 0, last_n = 0;   // the live count sizes every launch below
  NMB_CUDA_OK(cudaMemcpyAsync(&last_off, w.live_off + (R - 1), 4, cudaMemcpyDeviceToHost, c.stream));
  NMB_CUDA_OK(cudaMemcpyAsync(&last_n, w.nlive + (R - 1), 4, cudaMemcpyDeviceToHost, c.stream));
  NMB_CUDA_OK(cudaStreamSynchronize(c.stream));
  *M = (int64_t)last_off + last_n;
  if (*M == 0) return 0;
  const bool normals = c.cfg->calc_normal;
  compact_live_kernel<<<c.rb, RT, 0, c.stream>>>(R, c.P, w.live_off, w.wbuf, w.z, w.zmid, w.orig, w.dirs, w.live_mid,
                                                 w.live_dir, nullptr, normals ? w.origin : nullptr,
                                                 normals ? w.live_src : nullptr);
  NMB_LAUNCH_OK();
  if (normals) {
    // sdf' * grad ds at the live sample POINTS, from the neighbours the sampling passes found (no second walk);
    // must run before the mid-point pass below re-uses the neighbour arrays
    FieldIn in(KnnOut{w.k_ds, w.k_slot, w.k_w, w.k_grad, (int64_t)c.P * R});
    in.index = w.live_src;
    int rc = eval_field(c, in, *M, w.sdf_mid, w.nabla_pts, false);
    if (rc) return rc;
  }
  KnnOut ko{w.k_ds, w.k_slot, w.k_w, w.k_grad, *M};
  int rc;
  if (R >= RAY_KERNEL_MIN_RAYS) {   // warm-started per-ray lists
    rc = launch_knn_lists(c.f->grid, c.f->indicator.p, c.f->w1, w.live_mid, w.live_off, w.nlive, R, *M, c.P - 1, ko,
                          c.stream);
  } else {
    PointSrc src{w.live_mid, nullptr, nullptr, nullptr, 0};
    rc = launch_knn_distance(c.f->grid, c.f->indicator.p, c.f->w1, src, *M, ko, c.stream);
  }
  if (rc) return rc;
  FieldIn in(ko);
  in.dirs = w.live_dir;
  return eval_field(c, in, *M, w.sdf_mid, mid_nabla, true);
}

// Mid-points, visibility weights, colour at the mid-points (every one, or the live ones only) and the composite into
// the caller's per-ray outputs.
int shade(const Chunk& c, bool live, float* rgb, float* depth, float* acc, float* normals) {
  const Workspace& w = c.w;
  const int64_t R = c.R, PR = (int64_t)c.P * R;
  midpoints_kernel<<<(unsigned)ceil_div(R * (c.P - 1), 256), 256, 0, c.stream>>>(R, c.P, w.z, w.zmid);
  NMB_LAUNCH_OK();
  weights_kernel<<<c.rb, RT, 0, c.stream>>>(R, c.P, c.f->s, w.sdf, w.wbuf, w.nlive);
  NMB_LAUNCH_OK();
  // the colour MLPs of the main model or of an edit's reference models may take the mid-point nabla as an input
  const bool need_mid_nabla = c.f->lay.use_nabla != 0 || (c.edit && edit_needs_nabla(c.edit));
  float* mid_nabla = need_mid_nabla ? w.nabla_mid : nullptr;
  int64_t M = 0;   // live path: length of the compacted list, the stride of its colours
  int rc = live ? eval_live(c, mid_nabla, &M) : eval_samples(c, w.zmid, c.P - 1, w.sdf_mid, mid_nabla, true, 0);
  if (rc) return rc;
  composite_kernel<<<c.rb, RT, 0, c.stream>>>(R, c.P, c.cfg->white_bkgd, w.wbuf, w.zmid, live ? w.live_off : nullptr,
                                              w.rgb, live ? M : PR, c.cfg->calc_normal ? w.nabla_pts : nullptr, PR,
                                              c.perm, rgb, depth, acc, normals);
  NMB_LAUNCH_OK();
  return 0;
}

// [S][R] chunk arrays -> the caller's per-ray detail outputs, each skipped when null.  A sampling_only render has
// computed the samples, their sdf and near / far only, and exports only those.
int export_detail(const Chunk& c, const nmb_render_detail* d) {
  const Workspace& w = c.w;
  const int P = c.P;
  const int64_t PR = (int64_t)P * c.R;
  auto ex = [&](float* dst, const float* src, int S, int C, int64_t cstride) -> int {
    if (!dst) return 0;
    export_samples_kernel<<<(unsigned)ceil_div(c.R * S * C, 256), 256, 0, c.stream>>>(c.R, S, C, src, cstride, c.perm,
                                                                                      dst);
    NMB_LAUNCH_OK();
    return 0;
  };
  int rc;
  if ((rc = ex(d->d_all, w.z, P, 1, 0))) return rc;
  if ((rc = ex(d->implicit_surface, w.sdf, P, 1, 0))) return rc;
  if (!c.cfg->sampling_only) {
    if (c.cfg->calc_normal && (rc = ex(d->implicit_nablas, w.nabla_pts, P, 3, PR))) return rc;
    if ((rc = ex(d->radiance, w.rgb, P - 1, 3, PR))) return rc;
    if ((rc = ex(d->sdf_mid, w.sdf_mid, P - 1, 1, 0))) return rc;
  }
  if (d->near_far) {
    export_near_far_kernel<<<c.rb, RT, 0, c.stream>>>(c.R, w.near, w.far, c.perm, d->near_far);
    NMB_LAUNCH_OK();
  }
  return 0;
}

}  // namespace

static int render_impl(const nmb_field* f, const nmb_edit* edit, const nmb_render_cfg* cfg, const float* rays_o,
                       const float* rays_d, int64_t N, int64_t rays_per_chunk, float* rgb, float* depth, float* acc,
                       float* normals, const nmb_render_detail* detail, void* workspace, int64_t workspace_bytes,
                       void* stream_) {
  using namespace nmb;
  if (N <= 0) return 0;   // an empty shard: nothing to do (the output pointers of empty tensors are null)
  NMB_CHECK(f && cfg && rays_o && rays_d, "null argument");
  NMB_CHECK_FRESH(f);
  NMB_CHECK(!edit || edit_grid(edit) == f->grid, "the edit was created for another main model's mesh grid");
  NMB_CHECK(!edit || edit_fresh(edit),
            "the edit was packed before its main mesh grid was last updated (nmb_grid_update): re-pack it with "
            "nmb_edit_update");
  NMB_CHECK(!edit || !cfg->sampling_only, "an edit changes colour only: sampling_only renders take nmb_render");
  NMB_CHECK(cfg->sampling_only ? (detail != nullptr) : (rgb && depth && acc), "null output");
  NMB_CHECK(rays_per_chunk > 0, "rays_per_chunk must be positive");
  NMB_CHECK(cfg->N_samples >= 2, "N_samples must be >= 2");
  NMB_CHECK(cfg->N_upsample_iters >= 0 && (cfg->N_upsample_iters == 0 || cfg->N_importance % cfg->N_upsample_iters == 0),
            "N_importance must be a multiple of N_upsample_iters");
  NMB_CHECK(!cfg->calc_normal || normals || cfg->sampling_only, "calc_normal needs a normals output");
  NMB_CHECK(workspace_bytes >= nmb_render_edit_workspace_bytes(cfg, edit, rays_per_chunk), "workspace too small");
  NMB_CHECK(N < (int64_t(1) << 31), "at most 2^31 - 1 rays per call (32-bit ray permutation)");
  NMB_CHECK(rays_per_chunk * (int64_t)(cfg->N_samples + cfg->N_importance) < (int64_t(1) << 31),
            "rays_per_chunk x samples per ray must stay below 2^31 (32-bit live-sample offsets)");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int n_iters = cfg->N_upsample_iters;
  const int n_new = n_iters > 0 ? cfg->N_importance / n_iters : 0;
  const int P = cfg->N_samples + n_new * n_iters;
  void* ws_aligned = reinterpret_cast<void*>(align_up(reinterpret_cast<int64_t>(workspace), 256));

  // ---- render order: rays sorted by the Morton key of their closest point to the scene centre ----
  uint32_t *key_in = nullptr, *key_out = nullptr;
  int32_t *idx_in = nullptr, *perm_all = nullptr;
  void* sort_tmp = nullptr;
  size_t sort_bytes = 0;
  NMB_CUDA_OK(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, key_in, key_out, idx_in, perm_all, (int)N, 0, 30, stream));
  StreamBuf b_key_in, b_key_out, b_idx_in, b_perm, b_sort;   // returned to the pool on every exit path
  NMB_CUDA_OK(b_key_in.alloc(sizeof(uint32_t) * N, stream));
  NMB_CUDA_OK(b_key_out.alloc(sizeof(uint32_t) * N, stream));
  NMB_CUDA_OK(b_idx_in.alloc(sizeof(int32_t) * N, stream));
  NMB_CUDA_OK(b_perm.alloc(sizeof(int32_t) * N, stream));
  NMB_CUDA_OK(b_sort.alloc(sort_bytes, stream));
  key_in = b_key_in.as<uint32_t>();
  key_out = b_key_out.as<uint32_t>();
  idx_in = b_idx_in.as<int32_t>();
  perm_all = b_perm.as<int32_t>();
  sort_tmp = b_sort.p;
  ray_key_kernel<<<(unsigned)ceil_div(N, 256), 256, 0, stream>>>(rays_o, rays_d, N, cfg->obj_bounding_radius, key_in, idx_in);
  NMB_LAUNCH_OK();
  NMB_CUDA_OK(cub::DeviceRadixSort::SortPairs(sort_tmp, sort_bytes, key_in, key_out, idx_in, perm_all, (int)N, 0, 30, stream));
  count_launch(3);

  // live path: only the mid-points with a non-zero weight are evaluated (per-sample detail outputs need them all)
  const bool live = cfg->skip_dead_samples && !detail;
  // full path with normals: the nabla at every sample is carried through the sampling passes
  const bool carry_nabla = cfg->calc_normal && !live && !cfg->sampling_only;
  for (int64_t c0 = 0; c0 < N; c0 += rays_per_chunk) {
    const int64_t R = (N - c0 < rays_per_chunk) ? (N - c0) : rays_per_chunk;
    const Workspace w = carve(ws_aligned, R, P, n_new > 0 ? n_new : 1);
    const EditScratch es = edit ? edit_carve(static_cast<float*>(ws_aligned) + w.total, (int64_t)(P - 1) * R)
                                : EditScratch{};
    const Chunk c{f, edit, cfg, N, R, P, n_new, perm_all + c0, w, es, stream, (unsigned)ceil_div(R, RT)};
    int rc = setup_rays(c, rays_o, rays_d);
    if (!rc) rc = sample_cascade(c, carry_nabla ? w.nabla_pts : nullptr);
    if (!rc && !cfg->sampling_only) rc = shade(c, live, rgb, depth, acc, normals);
    if (!rc && detail) rc = export_detail(c, detail);
    if (rc) return rc;
  }
  return 0;
}

extern "C" {

int nmb_render(const nmb_field* f, const nmb_render_cfg* cfg, const float* rays_o, const float* rays_d, int64_t N,
               int64_t rays_per_chunk, float* rgb, float* depth, float* acc, float* normals,
               const nmb_render_detail* detail, void* workspace, int64_t workspace_bytes, void* stream) {
  return render_impl(f, nullptr, cfg, rays_o, rays_d, N, rays_per_chunk, rgb, depth, acc, normals, detail, workspace,
                     workspace_bytes, stream);
}

int nmb_render_edit(const nmb_field* f, const nmb_edit* edit, const nmb_render_cfg* cfg, const float* rays_o,
                    const float* rays_d, int64_t N, int64_t rays_per_chunk, float* rgb, float* depth, float* acc,
                    float* normals, const nmb_render_detail* detail, void* workspace, int64_t workspace_bytes,
                    void* stream) {
  NMB_CHECK(edit != nullptr, "null edit (plain renders take nmb_render)");
  return render_impl(f, edit, cfg, rays_o, rays_d, N, rays_per_chunk, rgb, depth, acc, normals, detail, workspace,
                     workspace_bytes, stream);
}

int nmb_upsample_step(const float* z, const float* sdf, int64_t N, int32_t n, int32_t n_new, float inv_s, float* z_new,
                      float* scratch, void* stream) {
  NMB_CHECK(z && sdf && z_new && scratch && n >= 2 && n_new >= 1, "bad argument");
  if (N <= 0) return 0;
  nmb::upsample_kernel<<<(unsigned)nmb::ceil_div(N, nmb::RT), nmb::RT, 0, static_cast<cudaStream_t>(stream)>>>(
      N, n, n_new, inv_s, z, sdf, scratch, z_new, nullptr, 0, nullptr);
  NMB_LAUNCH_OK();
  return 0;
}

int nmb_first_crossing(const float* val, int64_t N, int32_t n_steps, float tau, const float* near, const float* far,
                       float* d_low, float* f_low, float* d_high, float* f_high, uint8_t* mask,
                       uint8_t* mask_sign_change, uint8_t* first_free, void* stream) {
  NMB_CHECK(val && near && far && d_low && f_low && d_high && f_high && mask && mask_sign_change && first_free && n_steps >= 2,
            "bad argument");
  if (N <= 0) return 0;
  nmb::first_crossing_kernel<<<(unsigned)nmb::ceil_div(N, 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(
      N, n_steps, tau, val, near, far, d_low, f_low, d_high, f_high, mask, mask_sign_change, first_free);
  NMB_LAUNCH_OK();
  return 0;
}

int nmb_pack_bgr8(const float* rgb, int64_t N, uint8_t* bgr8, void* stream) {
  NMB_CHECK(rgb && bgr8, "null argument");
  if (N <= 0) return 0;
  nmb::pack_bgr8_kernel<<<(unsigned)nmb::ceil_div(N, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(rgb, N, bgr8);
  NMB_LAUNCH_OK();
  return 0;
}

int nmb_vertex_normals(const float* vertices, int64_t V, const int32_t* triangles, int64_t T, float* normals,
                       void* stream_) {
  NMB_CHECK(vertices && triangles && normals && V > 0, "bad argument");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  NMB_CUDA_OK(cudaMemsetAsync(normals, 0, sizeof(float) * 3 * V, stream));
  if (T > 0 && nmb::deterministic()) {
    NMB_CHECK(T < (int64_t(1) << 31) / 3 && V <= (int64_t(1) << 31), "mesh too large for the deterministic normals");
    const int64_t n = 3 * T;
    int bits = 1;
    while ((int64_t(1) << bits) < V) ++bits;
    size_t sort_bytes = 0;
    NMB_CUDA_OK(nmb::sort_pairs_u32(nullptr, sort_bytes, nullptr, nullptr, nullptr, nullptr, (int)n, bits, stream));
    const int64_t n_al = nmb::align_up(n, 64);
    nmb::StreamBuf buf;   // key, key_sorted, corner, corner_sorted [3T] | sort temporaries
    NMB_CUDA_OK(buf.alloc(4 * sizeof(uint32_t) * n_al + sort_bytes, stream));
    uint32_t* key = buf.as<uint32_t>();
    uint32_t* key_sorted = key + n_al;
    int32_t* corner = reinterpret_cast<int32_t*>(key_sorted + n_al);
    int32_t* corner_sorted = corner + n_al;
    nmb::corner_list_kernel<<<(unsigned)nmb::ceil_div(n, 256), 256, 0, stream>>>(triangles, n, key, corner);
    NMB_LAUNCH_OK();
    NMB_CUDA_OK(nmb::sort_pairs_u32(corner_sorted + n_al, sort_bytes, key, key_sorted, corner, corner_sorted, (int)n,
                                    bits, stream));
    nmb::count_launch();
    nmb::vertex_normal_runs_kernel<<<(unsigned)nmb::ceil_div(n, 256), 256, 0, stream>>>(vertices, triangles, n,
                                                                                       key_sorted, corner_sorted, normals);
    NMB_LAUNCH_OK();
  } else if (T > 0) {
    nmb::face_normals_kernel<<<(unsigned)nmb::ceil_div(T, 256), 256, 0, stream>>>(vertices, triangles, T, normals);
    NMB_LAUNCH_OK();
  }
  nmb::normalize_rows_kernel<<<(unsigned)nmb::ceil_div(V, 256), 256, 0, stream>>>(normals, V);
  NMB_LAUNCH_OK();
  return 0;
}

int nmb_get_rays(const float* c2w, const float* intr, int32_t H, int32_t W, float* rays_o, float* rays_d,
                 void* stream) {
  NMB_CHECK(c2w && intr && rays_o && rays_d && H > 0 && W > 0, "bad argument");
  nmb::get_rays_kernel<<<(unsigned)nmb::ceil_div((int64_t)H * W, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      H, W, intr[0], intr[1], intr[2], intr[3], intr[4], c2w[0], c2w[1], c2w[2], c2w[4], c2w[5], c2w[6], c2w[8],
      c2w[9], c2w[10], c2w[3], c2w[7], c2w[11], rays_o, rays_d);
  NMB_LAUNCH_OK();
  return 0;
}

}  // extern "C"
