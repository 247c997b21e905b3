// Field packing (tables -> Morton order, weight-norm folding, weight layouts) and the point-query C ABI.
#include <vector>

#include "field.cuh"

namespace nmb {

__global__ void permute_table_kernel(const float* __restrict__ src, const int32_t* __restrict__ order, int64_t V, int F,
                                     float* __restrict__ dst) {
  // F = 32 n floats per row: one warp per row, coalesced both ways
  const int64_t row = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= V) return;
  const float* s = src + (int64_t)order[row] * F;
  for (int c = lane; c < F; c += 32) dst[row * F + c] = s[c];
}

// One block per output unit n: W_eff[n][:] = g[n] * v[n][:] / ||v[n]||  (or v itself when g == nullptr), written
// transposed and column-permuted: wt[k * n_out_stride + n] = W_eff[n][colmap[k]] (0 where colmap[k] < 0).
__global__ void fold_transpose_kernel(const float* __restrict__ v, const float* __restrict__ g, int in_dim,
                                      const int32_t* __restrict__ colmap, int K, int n_stride,
                                      float* __restrict__ wt) {
  const int n = blockIdx.x;
  __shared__ float red[32];
  __shared__ float scale_s;
  float scale = 1.f;
  if (g) {
    float s = 0.f;
    for (int i = threadIdx.x; i < in_dim; i += blockDim.x) {
      const float x = v[(int64_t)n * in_dim + i];
      s += x * x;
    }
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f;
      for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i];
      scale_s = g[n] / sqrtf(t);
    }
    __syncthreads();
    scale = scale_s;
  }
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const int c = colmap[k];
    wt[(int64_t)k * n_stride + n] = c >= 0 ? v[(int64_t)n * in_dim + c] * scale : 0.f;
  }
}

static FieldLayout make_layout(const nmb_field_desc* d) {
  FieldLayout L{};
  L.Ld = d->multires_d;
  L.Lfg = d->multires_fg;
  L.Lft = d->multires_ft;
  L.Lv = d->multires_view;
  L.ch_d = 1 + 2 * L.Ld;
  L.ch_v = 3 * (1 + 2 * L.Lv);
  L.use_nabla = d->enable_nablas_input ? 1 : 0;
  L.Fg = d->geometry_dim;
  L.Fc = d->color_dim;
  L.off_fg = (int)align_up(L.ch_d, 16);
  L.K0g = (int)align_up(L.off_fg + L.Fg * (1 + 2 * L.Lfg), 16);
  L.off_nabla = L.ch_d;
  L.off_view = L.ch_d + (L.use_nabla ? 3 : 0);
  L.off_ft = (int)align_up(L.off_view + L.ch_v, 16);
  L.K0c = (int)align_up(L.off_ft + L.Fc * (1 + 2 * L.Lft), 16);
  L.n_geo = d->D_density;
  L.n_col = d->D_color;
  return L;
}

// Every configuration limit of the fused kernels, from the descriptor's integer fields and the engine only (no CUDA
// call).  A packed field has passed it, so the launchers do not check again.
static int check_field(const nmb_field_desc* d, int engine) {
  NMB_CHECK(engine >= 0 && engine <= 2, "mlp_engine must be 0 (tensor-core 3xTF32), 1 (fp32) or 2 (tensor-core fp16x3)");
  NMB_CHECK(d->W == MLP_W, "fused kernels are specialised for W = 256");
  NMB_CHECK(d->geometry_dim >= FEAT && d->geometry_dim % FEAT == 0 && d->color_dim >= FEAT && d->color_dim % FEAT == 0,
            "fused kernels need vertex code widths that are multiples of 32");
  NMB_CHECK(engine != 1 || (d->geometry_dim == FEAT && d->color_dim == FEAT),
            "the fp32 engine is specialised for 32-d vertex codes (use a tensor-core engine)");
  NMB_CHECK(d->D_density >= 1 && d->D_density < MAX_LAYERS && d->D_color >= 1 && d->D_color < MAX_LAYERS,
            "unsupported MLP depth");
  NMB_CHECK(d->multires_d >= 0 && d->multires_fg >= 0 && d->multires_ft >= 0 && d->multires_view >= 0,
            "identity embedders (multires < 0) are not supported by the fused kernels");
  NMB_CHECK(engine != 2 || d->multires_d <= F16_MAX_MULTIRES_D,
            "multires_d > 16 overflows the fp16 engine's tangent operands (use the 3xTF32 engine)");
  const FieldLayout L = make_layout(d);
  NMB_CHECK(engine != 1 || (L.K0g <= 256 && L.K0c <= 256), "first-layer width exceeds the fp32 engine's 256-column tile");
  NMB_CHECK(engine == 1 || (L.off_fg <= 64 && L.off_ft <= 64),
            "head block wider than 64 columns (the tensor-core engines' limit)");
  return 0;
}

// reference column of each of our first-layer columns (-1 = padding)
static std::vector<int32_t> geo_colmap(const FieldLayout& L) {
  std::vector<int32_t> m(L.K0g, -1);
  for (int i = 0; i < L.ch_d; ++i) m[i] = i;                                            // neumesh.py:214,217
  for (int i = 0; i < L.Fg * (1 + 2 * L.Lfg); ++i) m[L.off_fg + i] = L.ch_d + i;
  return m;
}
static std::vector<int32_t> col_colmap(const FieldLayout& L) {
  // reference order (neumesh.py:249-256): [nabla(3)?, d_emb, view_emb, ft_emb]
  std::vector<int32_t> m(L.K0c, -1);
  const int nb = L.use_nabla ? 3 : 0;
  for (int i = 0; i < L.ch_d; ++i) m[i] = nb + i;
  for (int i = 0; i < nb; ++i) m[L.off_nabla + i] = i;
  for (int i = 0; i < L.ch_v; ++i) m[L.off_view + i] = nb + L.ch_d + i;
  for (int i = 0; i < L.Fc * (1 + 2 * L.Lft); ++i) m[L.off_ft + i] = nb + L.ch_d + L.ch_v + i;
  return m;
}

static int pack_ffma(const float* const* v, const float* const* g, const float* const* b, int n_layers, int n_out,
                     int K0, int in_ref0, const std::vector<int32_t>& colmap0, MlpFfma* out, cudaStream_t stream) {
  out->n_layers = n_layers;
  out->n_out = n_out;
  int64_t total = 0;
  for (int l = 0; l < n_layers; ++l) {
    out->K[l] = (l == 0) ? K0 : MLP_W;
    out->w_off[l] = total;
    total += (int64_t)out->K[l] * MLP_W;
  }
  NMB_CUDA_OK(out->w.alloc(total));
  NMB_CUDA_OK(out->b.alloc((int64_t)n_layers * MLP_W));
  NMB_CUDA_OK(out->w_out.alloc((int64_t)n_out * MLP_W));
  NMB_CUDA_OK(out->b_out.alloc(n_out));
  std::vector<int32_t> ident(MLP_W);
  for (int i = 0; i < MLP_W; ++i) ident[i] = i;
  // the maps live in the field (no allocation and no synchronisation when a field is re-packed); the uploads come from
  // pageable host memory, i.e. they are staged before cudaMemcpyAsync returns, so the vectors may go out of scope
  DevBuf<int32_t>& cm0 = out->cm0;
  DevBuf<int32_t>& cmi = out->cmi;
  NMB_CUDA_OK(cm0.alloc((int64_t)colmap0.size()));
  NMB_CUDA_OK(cmi.alloc(MLP_W));
  NMB_CUDA_OK(cudaMemcpyAsync(cm0.p, colmap0.data(), colmap0.size() * 4, cudaMemcpyHostToDevice, stream));
  NMB_CUDA_OK(cudaMemcpyAsync(cmi.p, ident.data(), MLP_W * 4, cudaMemcpyHostToDevice, stream));
  for (int l = 0; l < n_layers; ++l) {
    fold_transpose_kernel<<<MLP_W, 128, 0, stream>>>(v[l], g ? g[l] : nullptr, l == 0 ? in_ref0 : MLP_W,
                                                     l == 0 ? cm0.p : cmi.p, out->K[l], MLP_W, out->w.p + out->w_off[l]);
    NMB_LAUNCH_OK();
    NMB_CUDA_OK(cudaMemcpyAsync(out->b.p + l * MLP_W, b[l], MLP_W * 4, cudaMemcpyDeviceToDevice, stream));
  }
  // output layer: [n_out][256] row-major == fold_transpose with K = 256 written at stride 1... reuse with n_stride
  // trick: treat each output unit as a "row n" and write wt[k * 1 + n * 256]; do it with one launch per unit.
  for (int o = 0; o < n_out; ++o) {
    fold_transpose_kernel<<<1, 128, 0, stream>>>(v[n_layers] + (int64_t)o * MLP_W, g ? g[n_layers] + o : nullptr, MLP_W,
                                                 cmi.p, MLP_W, 1, out->w_out.p + (int64_t)o * MLP_W);
    NMB_LAUNCH_OK();
  }
  NMB_CUDA_OK(cudaMemcpyAsync(out->b_out.p, b[n_layers], n_out * 4, cudaMemcpyDeviceToDevice, stream));
  return 0;
}

static int pack_field(const nmb_field_desc* d, nmb_field* f, cudaStream_t stream) {
  const nmb_grid* g = f->grid;
  int rc = check_field(d, f->engine);
  if (rc) return rc;
  f->lay = make_layout(d);
  // the certificate depends on the vertex positions and the indicator: rebuilt lazily for the tables packed below
  f->shell_valid = false;
  f->shell = ShellGrid{};
  f->grid_generation = g->generation;
  f->w1 = d->indicator_weight;
  f->s = d->s;
  NMB_CUDA_OK(f->indicator.alloc(g->V));
  NMB_CUDA_OK(f->fg.alloc(g->V * f->lay.Fg));
  NMB_CUDA_OK(f->fc.alloc(g->V * f->lay.Fc));
  rc = permute_indicator(g, d->indicator_vector, f->indicator.p, stream);
  if (rc) return rc;
  const unsigned blocks = (unsigned)ceil_div(g->V * 32, 256);
  permute_table_kernel<<<blocks, 256, 0, stream>>>(d->geometry_features, g->order.p, g->V, f->lay.Fg, f->fg.p);
  NMB_LAUNCH_OK();
  permute_table_kernel<<<blocks, 256, 0, stream>>>(d->color_features, g->order.p, g->V, f->lay.Fc, f->fc.p);
  NMB_LAUNCH_OK();
  const FieldLayout& L = f->lay;
  rc = pack_ffma(d->geo_v, d->geo_g, d->geo_b, L.n_geo, 1, L.K0g, L.ch_d + L.Fg * (1 + 2 * L.Lfg), geo_colmap(L),
                 &f->geo_f, stream);
  if (rc) return rc;
  rc = pack_ffma(d->col_w, nullptr, d->col_b, L.n_col, 3, L.K0c,
                 (L.use_nabla ? 3 : 0) + L.ch_d + L.ch_v + L.Fc * (1 + 2 * L.Lft), col_colmap(L), &f->col_f, stream);
  if (rc) return rc;
  rc = pack_mlp_tc(d, L, f, stream);
  if (rc) return rc;
  NMB_CUDA_OK(cudaStreamSynchronize(stream));
  return 0;
}

// row-major <-> SoA helpers for the point-query API
__global__ void soa3_to_rows_kernel(const float* __restrict__ soa, int64_t stride, int64_t M, float* __restrict__ rows) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= M * 3) return;
  rows[t] = soa[(t % 3) * stride + t / 3];
}

// caller-supplied neighbours (row-major, original vertex order) -> the SoA the field kernels read
__global__ void import_neighbours_kernel(const int64_t* __restrict__ idx /*[M,8]*/, const float* __restrict__ w /*[M,8]*/,
                                         const float* __restrict__ nabla /*[M,3] or null*/,
                                         const int32_t* __restrict__ inv /*vertex -> slot, or null = identity*/,
                                         int64_t rows, int64_t M, int32_t* __restrict__ slot /*[8][M]*/,
                                         float* __restrict__ w_soa /*[8][M]*/, float* __restrict__ nabla_soa /*[3][M]*/) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= M * KNN_K) return;
  const int64_t m = t / KNN_K;
  const int k = (int)(t % KNN_K);
  int64_t v = idx[t];
  v = v < 0 ? 0 : (v >= rows ? rows - 1 : v);   // never read outside the table, whatever the caller passed
  slot[k * M + m] = inv ? inv[v] : (int32_t)v;
  w_soa[k * M + m] = w[t];
  if (k < 3 && nabla) nabla_soa[k * M + m] = nabla[m * 3 + k];
}

}  // namespace nmb

extern "C" {

int nmb_field_create(const nmb_grid* g, const nmb_field_desc* desc, int mlp_engine, void* stream, nmb_field** out) {
  if (!out) return 2;
  *out = nullptr;
  NMB_CHECK(g != nullptr && desc != nullptr, "null grid / descriptor");
  nmb_field* f = new nmb_field();
  f->grid = g;
  f->engine = mlp_engine;   // pack_field validates it with the descriptor
  int rc = nmb::pack_field(desc, f, static_cast<cudaStream_t>(stream));
  if (rc) {
    delete f;
    return rc;
  }
  *out = f;
  return 0;
}

int nmb_field_check(const nmb_field_desc* desc, int mlp_engine) {
  NMB_CHECK(desc != nullptr, "null descriptor");
  return nmb::check_field(desc, mlp_engine);
}

void nmb_field_destroy(nmb_field* f) { delete f; }

int nmb_field_update(nmb_field* f, const nmb_field_desc* desc, void* stream) {
  NMB_CHECK(f != nullptr && desc != nullptr, "null field / descriptor");
  return nmb::pack_field(desc, f, static_cast<cudaStream_t>(stream));
}

static int field_query(const nmb_field* f, const float* xyz, const float* dirs, int64_t M, float* sdf, float* rgb,
                       float* nabla, bool want_color, cudaStream_t stream, float* ds_out = nullptr,
                       int64_t* idx_out = nullptr, float* w_out = nullptr) {
  using namespace nmb;
  NMB_CHECK(f != nullptr, "null field");
  NMB_CHECK_FRESH(f);
  if (M <= 0) return 0;
  const bool need_nabla = (nabla != nullptr) || (want_color && f->lay.use_nabla);
  // scratch: ds 1, slot 8, w 8, grad 3, nabla 3, rgb 3, sdf 1 = 27 words per point
  StreamBuf scratch;
  NMB_CUDA_OK(scratch.alloc(sizeof(float) * M * 27, stream));
  float* sc = scratch.as<float>();
  KnnOut ko{sc, reinterpret_cast<int32_t*>(sc + M), sc + 9 * M, sc + 17 * M, M};
  PointSrc src{xyz, nullptr, nullptr, nullptr, 0};
  int rc = launch_knn_distance(f->grid, f->indicator.p, f->w1, src, M, ko, stream);
  if (rc) return rc;
  if (ds_out || idx_out || w_out) {
    rc = launch_export_knn(f->grid, ko, M, ds_out, idx_out, w_out, nullptr, stream);
    if (rc) return rc;
  }
  FieldIn in(ko);
  float* nab = sc + 20 * M;
  float* rgb_soa = sc + 23 * M;
  float* sdf_tmp = sdf ? sdf : sc + 26 * M;
  rc = launch_geo(f, in, M, sdf_tmp, need_nabla ? nab : nullptr, stream);
  if (rc) return rc;
  if (nabla) {
    soa3_to_rows_kernel<<<(unsigned)ceil_div(M * 3, 256), 256, 0, stream>>>(nab, M, M, nabla);
    NMB_LAUNCH_OK();
  }
  if (want_color) {
    in.nabla = nab;
    in.dirs = dirs;
    rc = launch_color(f, in, M, rgb_soa, stream);
    if (rc) return rc;
    soa3_to_rows_kernel<<<(unsigned)ceil_div(M * 3, 256), 256, 0, stream>>>(rgb_soa, M, M, rgb);
    NMB_LAUNCH_OK();
  }
  return 0;
}

int nmb_field_shell_grid(const nmb_field* f, uint8_t* cells, int32_t* G, float* B, void* stream_) {
  NMB_CHECK(f != nullptr && G != nullptr && B != nullptr, "null argument");
  NMB_CHECK_FRESH(f);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc = nmb::ensure_shell_grid(f, stream);
  if (rc) return rc;
  *G = f->shell.G;
  *B = f->shell.B;
  if (cells && f->shell.cells) {
    NMB_CUDA_OK(cudaMemcpyAsync(cells, f->shell.cells, (size_t)f->shell.G * f->shell.G * f->shell.G,
                                cudaMemcpyDeviceToDevice, stream));
  }
  return 0;
}

int nmb_field_sdf(const nmb_field* f, const float* xyz, int64_t M, float* sdf, float* nabla, void* stream) {
  return field_query(f, xyz, nullptr, M, sdf, nullptr, nabla, false, static_cast<cudaStream_t>(stream));
}

int nmb_field_forward(const nmb_field* f, const float* xyz, const float* view_dirs, int64_t M, float* sdf, float* rgb,
                      float* nabla, void* stream) {
  NMB_CHECK(view_dirs != nullptr && rgb != nullptr, "view_dirs and rgb are required");
  return field_query(f, xyz, view_dirs, M, sdf, rgb, nabla, true, static_cast<cudaStream_t>(stream));
}

int nmb_field_forward_ex(const nmb_field* f, const float* xyz, const float* view_dirs, int64_t M, float* sdf, float* rgb,
                         float* nabla, float* ds, int64_t* idx, float* w, void* stream) {
  NMB_CHECK((view_dirs != nullptr) == (rgb != nullptr), "view_dirs and rgb go together (both or neither)");
  return field_query(f, xyz, view_dirs, M, sdf, rgb, nabla, rgb != nullptr, static_cast<cudaStream_t>(stream), ds, idx,
                     w);
}

int nmb_field_color(const nmb_field* f, const float* color_table, int64_t table_rows, const float* ds,
                    const int64_t* idx, const float* w, const float* nabla, const float* view_dirs, int64_t M, float* rgb,
                    void* stream_) {
  using namespace nmb;
  NMB_CHECK(f != nullptr && ds && idx && w && view_dirs && rgb, "null argument");
  NMB_CHECK_FRESH(f);
  NMB_CHECK(!f->lay.use_nabla || nabla != nullptr, "this field's colour network takes nabla as an input");
  NMB_CHECK(color_table == nullptr || table_rows > 0, "table_rows must be positive when a table is given");
  if (M <= 0) return 0;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  // scratch: slot 8, w 8, nabla 3, rgb 3 words per point
  StreamBuf scratch;
  NMB_CUDA_OK(scratch.alloc(sizeof(float) * M * 22, stream));
  float* sc = scratch.as<float>();
  int32_t* slot = reinterpret_cast<int32_t*>(sc);
  float* w_soa = sc + 8 * M;
  float* nab = sc + 16 * M;
  float* rgb_soa = sc + 19 * M;
  import_neighbours_kernel<<<(unsigned)ceil_div(M * KNN_K, 256), 256, 0, stream>>>(
      idx, w, f->lay.use_nabla ? nabla : nullptr, color_table ? nullptr : f->grid->inv.p,
      color_table ? table_rows : f->grid->V, M, slot, w_soa, nab);
  NMB_LAUNCH_OK();
  FieldIn in{};
  in.ds = ds;
  in.slot = slot;
  in.w = w_soa;
  in.stride = M;
  in.nabla = nab;
  in.dirs = view_dirs;
  in.color_table = color_table;
  int rc = launch_color(f, in, M, rgb_soa, stream);
  if (rc) return rc;
  soa3_to_rows_kernel<<<(unsigned)ceil_div(M * 3, 256), 256, 0, stream>>>(rgb_soa, M, M, rgb);
  NMB_LAUNCH_OK();
  return 0;
}

}  // extern "C"
