// "Shell-free" certificate grid for compute_bounded_near_far (models/renderer.py:66-102).
//
// The reference evaluates the mesh distance ds at 256 samples of every ray only to test `ds < 0.1` (:86-87).  More
// than half of the rays of a frame never enter that shell, and the others spend most samples outside it.  This file
// proves, per cell of a G^3 grid, that EVERY point x of the cell has ds(x) >= 0.1 + margin; the scan kernel skips such
// samples (their mask would be false).  A cell that cannot be certified is simply evaluated as before, so the
// near / far values are exactly those of the full scan.
//
// Certificate.  ds(x) = sum_k w_k f(x - p_k, n_k) over the 8 nearest vertices with w_k >= 0, sum w_k = 1
// (mesh_grid.py:123-142), f(v, n) = (w1 n.v + |v|^3) / (w1 + |v|).  Hence ds(x) >= min over ALL vertices p of
// f(x - p, n_p).  For a set of vertices inside a sphere (m, r) whose indicator vectors satisfy |n_p - nb| <= dn, and a
// cell with centre c and half-diagonal delta, with rho = |x - p| in [rlo, rhi] = [|c-m| - r - delta, |c-m| + r + delta]:
//     n_p.(x - p) >= nb.(c - m) - |nb| (r + delta) - dn * rhi  =: nv_lo
//     f >= N / (w1 + rhi) if N := w1 nv_lo + rlo^3 >= 0, else N / (w1 + rlo).
// Independently f >= g(rho) = rho (rho^2 - w1 nmax) / (w1 + rho); beyond rho_safe, g >= 0.1 + margin.
// The octree is walked per cell with these node-level bounds (descending only where they fail); leaves are checked
// point by point; the first vertex that cannot be bounded above the threshold makes the cell "uncertain".
#include <math_constants.h>

#include <cmath>

#include "field.cuh"
#include "knn_walk.cuh"

namespace nmb {

constexpr int SHELL_G = 128;               // cells per axis
constexpr float SHELL_B = 1.001f;          // grid covers [-B, B]^3 (the unit bounding sphere of the reference's scenes)
constexpr float SHELL_THR = 0.1f + 2e-3f;  // certificate threshold: renderer.py:73 distance_thresh + rounding margin
constexpr float SHELL_THR_IN = 0.1f - 2e-3f;  // "inside" certificate: every point of the cell has ds < 0.1

// per-node indicator statistics, bottom-up: {mean vector, max deviation of any vertex below the node from it}
__global__ void node_normals_kernel(int32_t first, int32_t count, const float4* __restrict__ nodes,
                                    const float4* __restrict__ indicator, float4* __restrict__ stats) {
  const int32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= count) return;
  const int32_t n = first + t;
  const int32_t link = __float_as_int(nodes[NODE_F4 * n].w);
  const int32_t cnt = __float_as_int(nodes[NODE_F4 * n + 1].w);
  float mx = 0.f, my = 0.f, mz = 0.f, dn = 0.f;
  if (cnt < 0) {
    const int32_t k = -cnt;
    for (int32_t i = link; i < link + k; ++i) {
      const float4 v = indicator[i];
      mx += v.x; my += v.y; mz += v.z;
    }
    mx /= k; my /= k; mz /= k;
    for (int32_t i = link; i < link + k; ++i) {
      const float4 v = indicator[i];
      const float ex = v.x - mx, ey = v.y - my, ez = v.z - mz;
      dn = fmaxf(dn, sqrtf(ex * ex + ey * ey + ez * ez));
    }
  } else {
    for (int32_t c = link; c < link + cnt; ++c) {
      const float4 s = stats[c];
      mx += s.x; my += s.y; mz += s.z;
    }
    mx /= cnt; my /= cnt; mz /= cnt;
    for (int32_t c = link; c < link + cnt; ++c) {
      const float4 s = stats[c];
      const float ex = s.x - mx, ey = s.y - my, ez = s.z - mz;
      dn = fmaxf(dn, sqrtf(ex * ex + ey * ey + ez * ez) + s.w);   // triangle inequality
    }
  }
  stats[n] = make_float4(mx, my, mz, dn * 1.0001f + 1e-6f);
}

__device__ __forceinline__ float f_lower(float w1, float nv_lo, float rlo, float rhi) {
  const float num = w1 * nv_lo + rlo * rlo * rlo;
  return num >= 0.f ? num / (w1 + rhi) : num / (w1 + rlo);
}
__device__ __forceinline__ float f_upper(float w1, float nv_hi, float rlo, float rhi) {
  const float num = w1 * nv_hi + rhi * rhi * rhi;
  return num >= 0.f ? num / (w1 + rlo) : num / (w1 + rhi);
}

// "Inside" certificate: ds(x) <= max_k f(x - p_k, n_k) over the 8 nearest vertices of x, and for x in the cell those
// lie within R_S = d8(c) + 2 delta of the centre c (d8 = distance to the 8th neighbour of c, from an exact walk).
// If f is bounded below the threshold for EVERY vertex inside that ball, every point of the cell is inside the shell.
__device__ bool certify_inside(const float4* __restrict__ nodes, const float4* __restrict__ pts,
                               const float4* __restrict__ indicator, const float4* __restrict__ stats, float w1,
                               float cx, float cy, float cz, float delta) {
  float d2[KNN_K];
  int32_t ix[KNN_K];
  knn_walk<KNN_K, false>(nodes, pts, cx, cy, cz, d2, ix);
  const float RS = sqrtf(d2[KNN_K - 1]) * 1.00001f + 2.f * delta + 1e-6f;
  int32_t stack[STACK_MAX];
  int sp = 1;
  stack[0] = 0;
  while (sp > 0) {
    const int32_t n = stack[--sp];
    const float4 cr = __ldg(&nodes[NODE_F4 * n + 2]);
    const float ex = cx - cr.x, ey = cy - cr.y, ez = cz - cr.z;
    const float D = sqrtf(ex * ex + ey * ey + ez * ez);
    if (D * 0.99999f - cr.w > RS) continue;                       // no vertex of the node can be a neighbour
    const float rlo = fmaxf(D * 0.99999f - cr.w - delta, 0.f);
    const float rhi = D * 1.00001f + cr.w + delta;
    const float4 st = __ldg(&stats[n]);
    const float nbn = sqrtf(st.x * st.x + st.y * st.y + st.z * st.z);
    const float nv_hi = (st.x * ex + st.y * ey + st.z * ez) + nbn * (cr.w + delta) + st.w * rhi + 1e-6f;
    if (f_upper(w1, nv_hi, rlo, rhi) < SHELL_THR_IN) continue;    // whole node bounded
    const int32_t link = __float_as_int(__ldg(&nodes[NODE_F4 * n]).w);
    const int32_t cnt = __float_as_int(__ldg(&nodes[NODE_F4 * n + 1]).w);
    if (cnt < 0) {
      for (int32_t i = link; i < link - cnt; ++i) {
        const float4 p = __ldg(&pts[i]);
        const float vx = cx - p.x, vy = cy - p.y, vz = cz - p.z;
        const float rc = sqrtf(vx * vx + vy * vy + vz * vz);
        if (rc * 0.99999f > RS) continue;
        const float4 nv = __ldg(&indicator[i]);
        const float plo = fmaxf(rc * 0.99999f - delta, 0.f), phi = rc * 1.00001f + delta;
        const float nn = sqrtf(nv.x * nv.x + nv.y * nv.y + nv.z * nv.z);
        const float hi = (nv.x * vx + nv.y * vy + nv.z * vz) + nn * delta + 1e-6f;
        if (!(f_upper(w1, hi, plo, phi) < SHELL_THR_IN)) return false;
      }
    } else {
      for (int32_t c = 0; c < cnt; ++c) {
        if (sp >= STACK_MAX) return false;
        stack[sp++] = link + c;
      }
    }
  }
  return true;
}

__global__ void __launch_bounds__(128)
shell_certify_kernel(const float4* __restrict__ nodes, const float4* __restrict__ pts,
                     const float4* __restrict__ indicator, const float4* __restrict__ stats, float w1, float rho_safe,
                     int G, float B, uint8_t* __restrict__ cells) {
  const int64_t cell = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (cell >= (int64_t)G * G * G) return;
  const int ix = (int)(cell % G), iy = (int)((cell / G) % G), iz = (int)(cell / ((int64_t)G * G));
  const float hs = B / (float)G;   // half cell size
  const float cx = -B + (2 * ix + 1) * hs, cy = -B + (2 * iy + 1) * hs, cz = -B + (2 * iz + 1) * hs;
  const float delta = hs * 1.7320508f * 1.0001f + 2e-6f;
  int32_t stack[STACK_MAX];
  int sp = 1;
  stack[0] = 0;
  bool ok = true;
  while (sp > 0 && ok) {
    const int32_t n = stack[--sp];
    const float4 cr = __ldg(&nodes[NODE_F4 * n + 2]);
    const float ex = cx - cr.x, ey = cy - cr.y, ez = cz - cr.z;
    const float D = sqrtf(ex * ex + ey * ey + ez * ez);
    const float rlo = fmaxf(D * 0.99999f - cr.w - delta, 0.f);
    if (rlo >= rho_safe) continue;                                  // g(rho) bound certifies the whole node
    const float rhi = D * 1.00001f + cr.w + delta;
    const float4 st = __ldg(&stats[n]);
    const float nbn = sqrtf(st.x * st.x + st.y * st.y + st.z * st.z);
    const float nv_lo = (st.x * ex + st.y * ey + st.z * ez) - nbn * (cr.w + delta) - st.w * rhi - 1e-6f;
    if (f_lower(w1, nv_lo, rlo, rhi) > SHELL_THR) continue;          // node certified
    const int32_t link = __float_as_int(__ldg(&nodes[NODE_F4 * n]).w);
    const int32_t cnt = __float_as_int(__ldg(&nodes[NODE_F4 * n + 1]).w);
    if (cnt < 0) {
      for (int32_t i = link; i < link - cnt; ++i) {
        const float4 p = __ldg(&pts[i]);
        const float4 nv = __ldg(&indicator[i]);
        const float vx = cx - p.x, vy = cy - p.y, vz = cz - p.z;
        const float rc = sqrtf(vx * vx + vy * vy + vz * vz);
        const float plo = fmaxf(rc * 0.99999f - delta, 0.f), phi = rc * 1.00001f + delta;
        if (plo >= rho_safe) continue;
        const float nn = sqrtf(nv.x * nv.x + nv.y * nv.y + nv.z * nv.z);
        const float lo = (nv.x * vx + nv.y * vy + nv.z * vz) - nn * delta - 1e-6f;
        if (!(f_lower(w1, lo, plo, phi) > SHELL_THR)) {
          ok = false;
          break;
        }
      }
    } else {
      for (int32_t c = 0; c < cnt && sp < STACK_MAX; ++c) stack[sp++] = link + c;
      if (sp >= STACK_MAX) ok = false;   // cannot happen (7 * depth + 8 < STACK_MAX); stay conservative
    }
  }
  uint8_t code = ok ? 1 : 0;
  if (!ok && certify_inside(nodes, pts, indicator, stats, w1, cx, cy, cz, delta)) code = 2;
  cells[cell] = code;   // 1: every point has ds >= 0.1; 2: every point has ds < 0.1; 0: not proven either way
}

int ensure_shell_grid(const nmb_field* f, cudaStream_t stream) {
  std::lock_guard<std::mutex> lock(f->shell_mu);
  if (f->shell_valid) return 0;
  const nmb_grid* g = f->grid;
  f->shell = ShellGrid{};
  f->shell_valid = true;   // whatever happens below, do not retry on every frame
  if (g->lvl_off.size() < 2 || !(f->w1 > 0.f)) return 0;
  // the node count changes when the grid is rebuilt over moved vertices (nmb_grid_update): keep 1/8 to spare then, as
  // the grid does for its node array
  const int64_t nn = g->num_nodes;
  NMB_CUDA_OK(g->generation > 0 ? f->node_normals.reserve(nn + nn / 8, 12) : f->node_normals.alloc(nn));
  NMB_CUDA_OK(f->shell_cells.alloc((int64_t)SHELL_G * SHELL_G * SHELL_G));
  for (int l = (int)g->lvl_off.size() - 2; l >= 0; --l) {
    const int32_t first = g->lvl_off[l], cnt = g->lvl_off[l + 1] - g->lvl_off[l];
    if (cnt <= 0) continue;
    node_normals_kernel<<<(unsigned)ceil_div(cnt, 128), 128, 0, stream>>>(first, cnt, g->nodes.p, f->indicator.p,
                                                                        f->node_normals.p);
    NMB_LAUNCH_OK();
  }
  float4 root_stats, root_sphere;
  NMB_CUDA_OK(cudaMemcpyAsync(&root_stats, f->node_normals.p, sizeof(float4), cudaMemcpyDeviceToHost, stream));
  NMB_CUDA_OK(cudaMemcpyAsync(&root_sphere, g->nodes.p + 2, sizeof(float4), cudaMemcpyDeviceToHost, stream));
  NMB_CUDA_OK(cudaStreamSynchronize(stream));
  const double nmax = std::sqrt((double)root_stats.x * root_stats.x + (double)root_stats.y * root_stats.y +
                                (double)root_stats.z * root_stats.z) + root_stats.w;
  if (!(nmax == nmax) || nmax > 1e3) return 0;   // non-finite / absurd indicator vectors: no certificate
  // rho_safe: g(rho) = rho (rho^2 - w1 nmax) / (w1 + rho) >= threshold for every rho >= rho_safe
  const double w1 = f->w1, thr = (double)SHELL_THR + 1e-3;
  // g is increasing once rho^2 > w1 nmax; if it is not yet above the threshold at the start of the search (very large
  // learned indicator vectors, w1 * nmax > ~64) there is no sound rho_safe in range: build no certificate at all
  double rho_safe = 8.0;
  if (rho_safe * (rho_safe * rho_safe - w1 * nmax) / (w1 + rho_safe) < thr) return 0;
  for (double rho = 8.0; rho > 0.0; rho -= 1e-3) {
    const double gval = rho * (rho * rho - w1 * nmax) / (w1 + rho);
    if (gval < thr) break;
    rho_safe = rho;
  }
  rho_safe += 2e-3;
  const int64_t n_cells = (int64_t)SHELL_G * SHELL_G * SHELL_G;
  shell_certify_kernel<<<(unsigned)ceil_div(n_cells, 128), 128, 0, stream>>>(
      g->nodes.p, g->pts.p, f->indicator.p, f->node_normals.p, f->w1, (float)rho_safe, SHELL_G, SHELL_B,
      f->shell_cells.p);
  NMB_LAUNCH_OK();
  ShellGrid sg;
  sg.cells = f->shell_cells.p;
  sg.G = SHELL_G;
  sg.B = SHELL_B;
  sg.cx = root_sphere.x;
  sg.cy = root_sphere.y;
  sg.cz = root_sphere.z;
  sg.far_r = root_sphere.w + (float)rho_safe + 1e-3f;   // beyond this every vertex is farther than rho_safe
  // one-off build: complete it before publishing, so that renders on OTHER streams may use the cells right away
  NMB_CUDA_OK(cudaStreamSynchronize(stream));
  f->shell = sg;
  return 0;
}

}  // namespace nmb
