// Spatial index over mesh vertices: Morton-ordered sparse octree with tight node boxes.
#pragma once
#include <vector>

#include "common.cuh"

struct nmb_grid {
  int64_t V = 0;
  int levels = 0;          // octree depth L (codes have 3*L bits)
  int num_nodes = 0;
  // incremented by every nmb_grid_update: fields and edits record the value they were packed against (their vertex
  // tables are in this grid's slot order, which an update changes) and are refused while it is behind
  int64_t generation = 0;
  float bmin[3] = {0, 0, 0};
  float inv_cell = 0.f;    // 2^L / cube side
  nmb::DevBuf<float4> pts;     // [V] sorted by Morton code: x, y, z, __int_as_float(original index)
  nmb::DevBuf<int32_t> order;  // [V] sorted slot -> original index
  nmb::DevBuf<int32_t> inv;    // [V] original index -> sorted slot
  nmb::DevBuf<float4> nodes;   // [NODE_F4*num_nodes]: box + disc bounds and child / point links; see grid.cu
  std::vector<int32_t> lvl_off; // first node id of every octree level (+ end sentinel); children ids > parent ids
};

namespace nmb {

constexpr int KNN_K = 8;          // neighbours used by the field (mesh_grid.py:77 default K=8)
constexpr int LEAF_MAX = 32;      // nodes with <= LEAF_MAX points are leaves (measured: 8 -> 169 ms, 16 -> 145, 32 -> 137 per frame)
constexpr int NODE_F4 = 4;        // float4 per node: {lo, link}, {hi, count}, {centre, r}, {axis, t}
constexpr int DISC_MAX_POINTS = 8192;  // nodes larger than this get the trivial disc (sphere) bound
constexpr int STACK_MAX = 96;     // traversal stack entries (7 * depth + 8 <= 78 for depth 10)
// from this many rays on, one thread per ray (or ray segment) fills the GPU; below it the per-point kernels expose more
// parallelism
constexpr int64_t RAY_KERNEL_MIN_RAYS = 32768;

// the 10 bits of v spread to every third bit: one axis of a 30-bit Morton code
__device__ __forceinline__ uint32_t expand_bits10(uint32_t v) {
  v = (v * 0x00010001u) & 0xFF0000FFu;
  v = (v * 0x00000101u) & 0x0F00F00Fu;
  v = (v * 0x00000011u) & 0xC30C30C3u;
  v = (v * 0x00000005u) & 0x49249249u;
  return v;
}

// Per-point outputs of the fused KNN + mesh-distance kernel, structure-of-arrays with stride `stride`
// (element (k, p) at [k * stride + p]) so that a warp of consecutive points reads/writes coalesced.
struct KnnOut {
  float* ds;        // [P]
  int32_t* slot;    // [8][P] neighbour slots in SORTED order
  float* w;         // [8][P]
  float* grad;      // [3][P] d ds / d xyz (nullable)
  int64_t stride;
};

// points given explicitly (xyz [P,3] row-major) or as rays: xyz = o[r] + z[p] * d[r], p = s * R + r
struct PointSrc {
  const float* xyz;     // explicit points, or nullptr
  const float* rays_o;  // [R,3]
  const float* rays_d;  // [R,3]
  const float* z;       // [S][R] sample-major depths
  int64_t R;
  // optional warm start of the FIRST sample of every ray (ray-ordered kernel, segment 0): the 8 neighbour slots of an
  // earlier query of that ray, stored SoA at seed_slot[k * seed_stride + seed_pos[r]].  Any 8 distinct real points are
  // a valid warm start (the walk is exact for every starting list), so this only removes a cold walk.
  const int32_t* seed_slot = nullptr;
  const int32_t* seed_entry = nullptr;   // [R]: pass entry e of the seed query; its data sits at e * R + r
  int64_t seed_stride = 0;
};

// torch.linspace(0, 1, n)[i] in fp32: step * i below the midpoint, fma(-step, n-1-i, 1) above (ATen's CPU kernel)
__device__ __forceinline__ float linspace01(int i, int n) {
  const float step = __fdiv_rn(1.0f, (float)(n - 1));
  return (i < n / 2) ? __fmul_rn(step, (float)i) : fmaf(-step, (float)(n - 1 - i), 1.0f);
}

// Shell certificate grid (csrc/shell.cu) over [-B,B]^3: cell value 1 = EVERY point of the cell provably has mesh distance
// ds >= 0.1 (the bounded-near/far scan skips it), 2 = every point provably has ds < 0.1 (a hit without evaluation),
// 0 = not proven either way (evaluated exactly).
struct ShellGrid {
  const uint8_t* cells = nullptr;   // nullptr = no certificate available
  int G = 0;
  float B = 0.f;
  float cx = 0.f, cy = 0.f, cz = 0.f, far_r = 0.f;   // |x - c| >= far_r  =>  certified as well (outside the grid)
};

int launch_bound_scan(const nmb_grid* g, const float4* indicator, float w1, const float* rays_o, const float* dirs,
                      const float* near, const float* far, int64_t R, int n_grid, float thresh, int32_t* bnear,
                      int32_t* bfar, ShellGrid shell, cudaStream_t stream);

int launch_knn_lists(const nmb_grid* g, const float4* indicator_sorted, float w1, const float* xyz, const int32_t* off,
                     const int32_t* cnt, int64_t R, int64_t M, int max_list, KnnOut out, cudaStream_t stream);

int launch_knn_distance(const nmb_grid* g, const float4* indicator_sorted, float w1, PointSrc src, int64_t P,
                        KnnOut out, cudaStream_t stream);

// SoA neighbour data (sorted slots) -> the reference's row-major outputs in original vertex order; any output may be null
int launch_export_knn(const nmb_grid* g, KnnOut in, int64_t M, float* ds, int64_t* idx, float* w, float* grad,
                      cudaStream_t stream);

}  // namespace nmb
