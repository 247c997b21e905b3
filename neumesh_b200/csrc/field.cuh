// Packed NeuMesh field (vertex tables in Morton order + MLP weights in the layouts the two MLP engines consume).
#pragma once
#include "../../include/neumesh_b200.h"
#include "grid.cuh"

namespace nmb {

constexpr int MLP_W = 256;     // hidden width the fused kernels are specialised for
constexpr int FEAT = 32;       // feature block: vertex codes are processed 32 columns at a time (code width = 32 n)
constexpr int MAX_LAYERS = 8;
// fp16 engine: the tangent seed of PE(ds) band b is 2^b cos(2^b ds), an fp16 A operand, so the highest band
// (2^(multires_d - 1)) must stay below fp16's largest finite value 65504
constexpr int F16_MAX_MULTIRES_D = 16;

// Column layout of the first-layer inputs (our own order; weights are permuted to match at pack time).
//   geometry: [PE(ds) | 0-pad to 16 | fg, sin fg, cos fg, sin 2fg, cos 2fg, ...]            K0g (multiple of 16)
//   colour  : [PE(ds) | nabla(3) | PE(view) | 0-pad to 16 | ft, sin ft, cos ft, ...]         K0c (multiple of 16)
struct FieldLayout {
  int Ld, Lfg, Lft, Lv;      // number of frequency bands
  int ch_d, ch_v;            // 1+2Ld, 3(1+2Lv)
  int off_fg, K0g;           // geometry
  int off_nabla, off_view, off_ft, K0c;
  int n_geo, n_col;          // hidden layer counts
  int use_nabla;
  int Fg, Fc;                // vertex code widths (multiples of FEAT; the fp32 engine handles 32 only)
};

struct MlpFfma {            // fp32 engine: W^T per layer, [K][256] row-major (k-major), zero rows for padding
  DevBuf<float> w;          // all layers back to back
  DevBuf<float> b;          // [n_layers][256]
  DevBuf<float> w_out;      // [n_out][256]
  DevBuf<float> b_out;      // [n_out]
  DevBuf<int32_t> cm0, cmi; // packing only: first-layer column map, identity map (kept: re-packing allocates nothing)
  int64_t w_off[MAX_LAYERS];
  int K[MAX_LAYERS];
  int n_layers = 0, n_out = 0;
};

struct MlpTc {              // tensor-core engine: per layer, per 16-column K-slab: [hi | lo] x [K/4][256][4] tf32 images
  DevBuf<float> w;
  DevBuf<int32_t> kmap[MAX_LAYERS];   // packing only: source column of every packed K column (kept between re-packs)
  int64_t slab_off[MAX_LAYERS];  // in floats
  int n_slabs[MAX_LAYERS];
  int total_slabs = 0;
};

}  // namespace nmb

struct nmb_field {
  const nmb_grid* grid = nullptr;
  int64_t grid_generation = 0;    // grid->generation the vertex tables were permuted for (stale when behind)
  int engine = 0;
  nmb::FieldLayout lay{};
  float w1 = 0.1f, s = 1.f;
  nmb::DevBuf<float4> indicator;  // [V] sorted
  nmb::DevBuf<float> fg;          // [V,Fg] sorted
  nmb::DevBuf<float> fc;          // [V,Fc] sorted
  nmb::MlpFfma geo_f, col_f;
  nmb::MlpTc geo_t, col_t;
  // shell-free certificate grid (built lazily by the first large render after a (re)pack; csrc/shell.cu)
  mutable nmb::DevBuf<uint8_t> shell_cells;
  mutable nmb::DevBuf<float4> node_normals;   // per octree node: mean indicator vector, max deviation
  mutable bool shell_valid = false;
  mutable nmb::ShellGrid shell{};
  mutable std::mutex shell_mu;                // serialises the lazy build when several host threads share the field
};

namespace nmb {

// Inputs of a field evaluation over P points whose neighbours are known (SoA from the KNN kernel).
struct FieldIn {
  FieldIn() = default;
  // the neighbours a KNN kernel found; every other member null
  explicit FieldIn(const KnnOut& k)
      : ds(k.ds), slot(k.slot), w(k.w), grad(k.grad), stride(k.stride), nabla(nullptr), dirs(nullptr), rays_d(nullptr),
        R(0), color_table(nullptr), index(nullptr) {}
  const float* ds;        // [P]
  const int32_t* slot;    // [8][P]
  const float* w;         // [8][P]
  const float* grad;      // [3][P] d ds/d xyz
  int64_t stride;
  // colour only:
  const float* nabla;     // [3][P] (SoA) d sdf / d xyz
  const float* dirs;      // explicit [P,3] row-major view directions, or nullptr -> rays_d[p % R]
  const float* rays_d;    // [R,3]
  int64_t R;
  const float* color_table;   // colour only: [rows, Fc] table indexed by `slot` instead of the field's own (nullable)
  const int32_t* index;       // geometry only (nullable): point p reads ds / slot / w / grad at position index[p] of the
                              // SoA arrays instead of p (nmb_render: the live sample points re-use the neighbours found
                              // in the sampling passes instead of walking the octree again); outputs are written at p
};

__device__ __forceinline__ int64_t field_src(const FieldIn& in, int64_t p) { return in.index ? (int64_t)in.index[p] : p; }

// geometry: sdf [P]; if nabla != nullptr also nabla [3][P] (SoA, stride = in.stride)
int launch_geo_ffma(const nmb_field* f, const FieldIn& in, int64_t P, float* sdf, float* nabla, cudaStream_t stream);
int launch_color_ffma(const nmb_field* f, const FieldIn& in, int64_t P, float* rgb /*[3][P] SoA*/, cudaStream_t stream);
int launch_geo_tc(const nmb_field* f, const FieldIn& in, int64_t P, float* sdf, float* nabla, cudaStream_t stream);
int launch_color_tc(const nmb_field* f, const FieldIn& in, int64_t P, float* rgb, cudaStream_t stream);

inline int launch_geo(const nmb_field* f, const FieldIn& in, int64_t P, float* sdf, float* nabla, cudaStream_t s) {
  return f->engine != 1 ? launch_geo_tc(f, in, P, sdf, nabla, s) : launch_geo_ffma(f, in, P, sdf, nabla, s);
}
inline int launch_color(const nmb_field* f, const FieldIn& in, int64_t P, float* rgb, cudaStream_t s) {
  return f->engine != 1 ? launch_color_tc(f, in, P, rgb, s) : launch_color_ffma(f, in, P, rgb, s);
}

// refuses a field packed before its grid's last nmb_grid_update (its tables are in the old slot order)
#define NMB_CHECK_FRESH(f)                                                                                          \
  NMB_CHECK((f)->grid_generation == (f)->grid->generation,                                                          \
            "the field was packed before its mesh grid was last updated (nmb_grid_update): re-pack it with "         \
            "nmb_field_update")

int permute_indicator(const nmb_grid* g, const float* indicator, float4* dst, cudaStream_t stream);
int pack_mlp_tc(const nmb_field_desc* d, const FieldLayout& lay, nmb_field* f, cudaStream_t stream);
// builds f->shell if it is not valid; on any failure leaves it empty (the scan then evaluates every sample)
int ensure_shell_grid(const nmb_field* f, cudaStream_t stream);

}  // namespace nmb
