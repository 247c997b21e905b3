// Texture edit (editing/texture_neumesh/texture_neumesh.py:81-121, restated in oracle/texture.py) inside nmb_render:
// the nmb_edit handle (masks and transferred codes permuted to the main grid's slot order, rotations) and the pass
// that runs after the main colour MLP at every colour call site of the renderer.
//
// Per reference model i, in order:
//   select  one thread per colour point: w_paint = sum_k w_k m_k, painted iff w_paint > 0 (flag)
//   compact order-preserving stream compaction of the painted points (cub::DeviceSelect::Flagged: the list, and so
//           the output bits, depend neither on scheduling nor on the chunk size)
//   gather  a_paint, a_rest, w_ref, R_i nabla, R_i v, ds, slots of the painted points, SoA
//   colour  the reference's own colour MLP (launch_color) on the edited code table, main-mesh slots, w_ref
//   blend   rgb = rgb * a_rest + c_ref * a_paint, multiply and add rounded separately as the reference does
#include <vector>

#include <cub/cub.cuh>

#include "edit.cuh"

struct nmb_edit {
  const nmb_field* main = nullptr;
  const nmb_grid* grid = nullptr;
  int64_t grid_generation = 0;  // grid->generation the masks and codes were permuted for
  int n_ref = 0;
  int Fc = 0;
  std::vector<const nmb_field*> refs;
  nmb::DevBuf<uint8_t> masks;   // [n_ref][V] slot order
  nmb::DevBuf<float> codes;     // [V][Fc] slot order
  bool has_rot = false;
  std::vector<float> rot;       // [n_ref][9] row-major
};

namespace nmb {

namespace {

constexpr int ET = 128;

// masks [n_ref][V] (original order) -> [n_ref][V] slot order
__global__ void permute_masks_kernel(const uint8_t* __restrict__ src, const int32_t* __restrict__ order, int64_t V,
                                     int n_ref, uint8_t* __restrict__ dst) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= V * n_ref) return;
  const int64_t i = t / V, s = t % V;
  dst[t] = src[i * V + order[s]] ? 1 : 0;
}

// codes [V][F] (original order) -> slot order, F = 32 n: one warp per row
__global__ void permute_codes_kernel(const float* __restrict__ src, const int32_t* __restrict__ order, int64_t V, int F,
                                     float* __restrict__ dst) {
  const int64_t row = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= V) return;
  const float* s = src + (int64_t)order[row] * F;
  for (int c = lane; c < F; c += 32) dst[row * F + c] = s[c];
}

// (w * m).sum(-1) and (w * ~m).sum(-1) over a row of 8: torch_row_sum's n = 8 case (common.cuh)
__device__ __forceinline__ void paint_sums(const FieldIn& in, int64_t p, const uint8_t* __restrict__ mask,
                                           float (&wm)[KNN_K], float (&wr)[KNN_K], float& w_paint, float& w_rest) {
#pragma unroll
  for (int k = 0; k < KNN_K; ++k) {
    const float w = in.w[k * in.stride + p];
    const bool m = mask[in.slot[k * in.stride + p]] != 0;
    wm[k] = m ? w : __fmul_rn(w, 0.f);   // w * True = w, w * False = 0 * w (keeps the sign torch gives)
    wr[k] = m ? __fmul_rn(w, 0.f) : w;
  }
  w_paint = torch_row_sum(wm, 1, KNN_K);
  w_rest = torch_row_sum(wr, 1, KNN_K);
}

__global__ void __launch_bounds__(ET)
edit_select_kernel(FieldIn in, int64_t n, const uint8_t* __restrict__ mask, int32_t* __restrict__ flag) {
  const int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (p >= n) return;
  float wm[KNN_K], wr[KNN_K], w_paint, w_rest;
  paint_sums(in, p, mask, wm, wr, w_paint, w_rest);
  flag[p] = w_paint > 0.f ? 1 : 0;
}

struct Rot {
  float r[9];
};

// torch.matmul(R, v[..., None]): row j = R[j,0] v0 + R[j,1] v1 + R[j,2] v2
__device__ __forceinline__ void rotate(const Rot& R, float x, float y, float z, float& ox, float& oy, float& oz) {
  ox = __fadd_rn(__fadd_rn(__fmul_rn(R.r[0], x), __fmul_rn(R.r[1], y)), __fmul_rn(R.r[2], z));
  oy = __fadd_rn(__fadd_rn(__fmul_rn(R.r[3], x), __fmul_rn(R.r[4], y)), __fmul_rn(R.r[5], z));
  oz = __fadd_rn(__fadd_rn(__fmul_rn(R.r[6], x), __fmul_rn(R.r[7], y)), __fmul_rn(R.r[8], z));
}

__global__ void __launch_bounds__(ET)
edit_gather_kernel(FieldIn in, int64_t n_sel, const int32_t* __restrict__ src, const uint8_t* __restrict__ mask,
                   int has_rot, Rot R, int64_t so /*stride of the outputs*/, float* __restrict__ ds,
                   int32_t* __restrict__ slot, float* __restrict__ w_ref, float* __restrict__ nabla,
                   float* __restrict__ dirs, float* __restrict__ a_paint, float* __restrict__ a_rest) {
  const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (j >= n_sel) return;
  const int64_t p = src[j];
  float wm[KNN_K], wr[KNN_K], w_paint, w_rest;
  paint_sums(in, p, mask, wm, wr, w_paint, w_rest);
  const float total = __fadd_rn(w_paint, w_rest);
  a_paint[j] = __fdiv_rn(w_paint, total);
  a_rest[j] = __fdiv_rn(w_rest, total);
  // w_ref.sum(-1) is the same row sum as w_paint
  const float den = __fadd_rn(w_paint, 1e-8f);
#pragma unroll
  for (int k = 0; k < KNN_K; ++k) {
    slot[k * so + j] = in.slot[k * in.stride + p];
    w_ref[k * so + j] = __fdiv_rn(wm[k], den);
  }
  ds[j] = in.ds[p];
  const float* d = in.dirs ? (in.dirs + p * 3) : (in.rays_d + (p % in.R) * 3);
  float dx = d[0], dy = d[1], dz = d[2];
  if (has_rot) rotate(R, dx, dy, dz, dx, dy, dz);
  dirs[j * 3 + 0] = dx;
  dirs[j * 3 + 1] = dy;
  dirs[j * 3 + 2] = dz;
  if (in.nabla) {
    float gx = in.nabla[p], gy = in.nabla[in.stride + p], gz = in.nabla[2 * in.stride + p];
    if (has_rot) rotate(R, gx, gy, gz, gx, gy, gz);
    nabla[j] = gx;
    nabla[so + j] = gy;
    nabla[2 * so + j] = gz;
  }
}

__global__ void __launch_bounds__(ET)
edit_blend_kernel(int64_t n_sel, const int32_t* __restrict__ src, const float* __restrict__ a_paint,
                  const float* __restrict__ a_rest, const float* __restrict__ c_ref, int64_t so, float* __restrict__ rgb,
                  int64_t stride) {
  const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (j >= n_sel) return;
  const int64_t p = src[j];
  const float ap = a_paint[j], ar = a_rest[j];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float* o = rgb + c * stride + p;
    *o = __fadd_rn(__fmul_rn(*o, ar), __fmul_rn(c_ref[c * so + j], ap));
  }
}

size_t select_temp_bytes(int64_t n) {
  size_t bytes = 0;
  cub::DeviceSelect::Flagged(nullptr, bytes, cub::CountingInputIterator<int32_t>(0), (const int32_t*)nullptr,
                             (int32_t*)nullptr, (int32_t*)nullptr, (int)n);
  return bytes;
}

int upload(nmb_edit* e, const uint8_t* masks, const float* codes, const float* rotations, cudaStream_t stream) {
  const int64_t V = e->grid->V;
  NMB_CUDA_OK(e->masks.alloc(V * e->n_ref));
  NMB_CUDA_OK(e->codes.alloc(V * e->Fc));
  permute_masks_kernel<<<(unsigned)ceil_div(V * e->n_ref, 256), 256, 0, stream>>>(masks, e->grid->order.p, V, e->n_ref,
                                                                                  e->masks.p);
  NMB_LAUNCH_OK();
  permute_codes_kernel<<<(unsigned)ceil_div(V * 32, 256), 256, 0, stream>>>(codes, e->grid->order.p, V, e->Fc,
                                                                            e->codes.p);
  NMB_LAUNCH_OK();
  e->has_rot = rotations != nullptr;
  e->rot.assign(rotations ? rotations : nullptr, rotations ? rotations + 9 * e->n_ref : nullptr);
  NMB_CUDA_OK(cudaStreamSynchronize(stream));   // the caller may free or overwrite its inputs when this returns
  e->grid_generation = e->grid->generation;
  return 0;
}

}  // namespace

EditScratch edit_carve(void* base, int64_t n) {
  EditScratch s{};
  float* p = static_cast<float*>(base);
  int64_t off = 0;
  auto take = [&](int64_t k) {
    float* q = p ? p + off : nullptr;
    off += align_up(k, 64);
    return q;
  };
  s.flag = reinterpret_cast<int32_t*>(take(n));
  s.src = reinterpret_cast<int32_t*>(take(n));
  s.count = reinterpret_cast<int32_t*>(take(1));
  s.ds = take(n);
  s.slot = reinterpret_cast<int32_t*>(take(8 * n));
  s.w_ref = take(8 * n);
  s.nabla = take(3 * n);
  s.dirs = take(3 * n);
  s.a_paint = take(n);
  s.a_rest = take(n);
  s.rgb = take(3 * n);
  s.select_bytes = select_temp_bytes(n);
  s.select_tmp = take((int64_t)(s.select_bytes / 4 + 1));
  s.total = off;
  return s;
}

bool edit_needs_nabla(const nmb_edit* e) {
  for (const nmb_field* r : e->refs)
    if (r->lay.use_nabla) return true;
  return false;
}

const nmb_grid* edit_grid(const nmb_edit* e) { return e->grid; }

bool edit_fresh(const nmb_edit* e) { return e->grid_generation == e->grid->generation; }

int apply_edit(const nmb_edit* e, const FieldIn& in, int64_t n, float* rgb, const EditScratch& s, cudaStream_t stream) {
  if (n <= 0) return 0;
  const unsigned nb = (unsigned)ceil_div(n, ET);
  const int64_t V = e->grid->V;
  for (int i = 0; i < e->n_ref; ++i) {
    const nmb_field* ref = e->refs[i];
    NMB_CHECK(!ref->lay.use_nabla || in.nabla != nullptr, "a reference model takes nabla but none was computed");
    const uint8_t* mask = e->masks.p + (int64_t)i * V;
    edit_select_kernel<<<nb, ET, 0, stream>>>(in, n, mask, s.flag);
    NMB_LAUNCH_OK();
    size_t bytes = s.select_bytes;
    NMB_CUDA_OK(cub::DeviceSelect::Flagged(s.select_tmp, bytes, cub::CountingInputIterator<int32_t>(0), s.flag, s.src,
                                           s.count, (int)n, stream));
    count_launch(1);
    int32_t n_sel = 0;
    NMB_CUDA_OK(cudaMemcpyAsync(&n_sel, s.count, 4, cudaMemcpyDeviceToHost, stream));
    NMB_CUDA_OK(cudaStreamSynchronize(stream));
    if (n_sel == 0) continue;
    Rot R{};
    if (e->has_rot)
      for (int k = 0; k < 9; ++k) R.r[k] = e->rot[(size_t)i * 9 + k];
    const unsigned sb = (unsigned)ceil_div(n_sel, ET);
    edit_gather_kernel<<<sb, ET, 0, stream>>>(in, n_sel, s.src, mask, e->has_rot ? 1 : 0, R, n, s.ds, s.slot, s.w_ref,
                                              s.nabla, s.dirs, s.a_paint, s.a_rest);
    NMB_LAUNCH_OK();
    FieldIn ri{};
    ri.ds = s.ds;
    ri.slot = s.slot;
    ri.w = s.w_ref;
    ri.stride = n;
    ri.nabla = s.nabla;
    ri.dirs = s.dirs;
    ri.color_table = e->codes.p;
    int rc = launch_color(ref, ri, n_sel, s.rgb, stream);
    if (rc) return rc;
    edit_blend_kernel<<<sb, ET, 0, stream>>>(n_sel, s.src, s.a_paint, s.a_rest, s.rgb, n, rgb, in.stride);
    NMB_LAUNCH_OK();
  }
  return 0;
}

}  // namespace nmb

extern "C" {

static int edit_check(const nmb_field* main_field, int32_t n_ref, const nmb_field* const* ref_fields,
                      const uint8_t* masks, const float* codes, int64_t V, int32_t color_dim) {
  NMB_CHECK(main_field != nullptr && masks != nullptr && codes != nullptr, "null argument");
  NMB_CHECK(n_ref >= 1 && ref_fields != nullptr, "an edit needs at least one reference field");
  NMB_CHECK(V == main_field->grid->V, "masks / codes must have one row per vertex of the main model's mesh");
  NMB_CHECK(color_dim >= nmb::FEAT && color_dim % nmb::FEAT == 0, "the code table width must be a multiple of 32");
  for (int i = 0; i < n_ref; ++i) {
    const nmb_field* r = ref_fields[i];
    NMB_CHECK(r != nullptr, "null reference field");
    NMB_CHECK(r->lay.Fc == color_dim, "every reference field's color_dim must equal the code table width");
  }
  return 0;
}

int nmb_edit_create(const nmb_field* main_field, int32_t n_ref, const nmb_field* const* ref_fields,
                    const uint8_t* masks, const float* codes, int64_t V, int32_t color_dim, const float* rotations,
                    void* stream, nmb_edit** out) {
  if (!out) return 2;
  *out = nullptr;
  int rc = edit_check(main_field, n_ref, ref_fields, masks, codes, V, color_dim);
  if (rc) return rc;
  nmb_edit* e = new nmb_edit();
  e->main = main_field;
  e->grid = main_field->grid;
  e->n_ref = n_ref;
  e->Fc = color_dim;
  e->refs.assign(ref_fields, ref_fields + n_ref);
  rc = nmb::upload(e, masks, codes, rotations, static_cast<cudaStream_t>(stream));
  if (rc) {
    delete e;
    return rc;
  }
  *out = e;
  return 0;
}

int nmb_edit_update(nmb_edit* e, const uint8_t* masks, const float* codes, const float* rotations, void* stream) {
  NMB_CHECK(e != nullptr && masks != nullptr && codes != nullptr, "null argument");
  return nmb::upload(e, masks, codes, rotations, static_cast<cudaStream_t>(stream));
}

void nmb_edit_destroy(nmb_edit* e) { delete e; }

}  // extern "C"
