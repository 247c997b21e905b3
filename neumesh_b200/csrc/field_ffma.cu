// fp32 (FFMA) MLP engine - the verification path of the field kernels (mlp_engine = 1).
//
// One CTA evaluates a tile of 64 rows through the whole MLP with the activations resident in shared memory
// (k-major: act[k][row]) and the weights streamed from L2 in 16-row chunks (cp.async, double-buffered).
//   geometry (neumesh.py:204-218):  [PE8(ds), PE2(fg)] -> D x (Linear + Softplus(100)) -> Linear(1)
//   nabla    (neumesh.py:223-232):  forward-mode: rows 32..63 of the tile carry the tangents d/d(ds) of rows 0..31
//                                   and nabla = (d sdf / d ds) * grad_xyz(ds)   (idx, w are detached in the reference)
//   colour   (neumesh.py:239-260):  [PE8(ds), nabla, PE4(view), PE2(ft)] -> D x (Linear + ReLU) -> Linear(3) + Sigmoid
#include <cuda_pipeline.h>

#include "field_build.cuh"

namespace nmb {

constexpr int TM = 64;     // rows per tile
constexpr int KC = 16;     // weight rows per chunk
constexpr int FT = 256;    // threads

struct FfmaParams {
  FieldLayout lay;
  FieldIn in;
  FieldTables tab;
  const float* w;        // layers back to back, each [K][256]
  const float* b;        // [n_layers][256]
  const float* w_out;    // [n_out][256]
  const float* b_out;    // [n_out]
  int64_t w_off[MAX_LAYERS];
  int K[MAX_LAYERS];
  int n_layers;
  int64_t P;
  float* out0;           // geo: sdf [P]; colour: rgb [3][P] SoA (stride in.stride)
  float* out1;           // geo: nabla [3][P] SoA or nullptr
};

__device__ __forceinline__ void load_w_chunk(float* dst, const float* __restrict__ src) {
  // KC*256 floats = 1024 float4; 4 per thread
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int v = threadIdx.x + i * FT;
    __pipeline_memcpy_async(reinterpret_cast<float4*>(dst) + v, reinterpret_cast<const float4*>(src) + v, 16);
  }
  __pipeline_commit();
}

// MODE 0: geometry, value rows only (64 points / tile)
// MODE 1: geometry + tangent rows (32 points / tile)
// MODE 2: colour (64 points / tile)
template <int MODE>
__global__ void __launch_bounds__(FT, 2) mlp_ffma_kernel(const FfmaParams prm) {
  extern __shared__ __align__(16) float smem[];
  float* act = smem;                    // [256][TM]
  float* wbuf = smem + 256 * TM;        // [2][KC][256]
  constexpr int PTS = (MODE == 1) ? 32 : 64;
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const FieldLayout& L = prm.lay;
  const int K0 = (MODE == 2) ? L.K0c : L.K0g;
  const int64_t n_tiles = (prm.P + PTS - 1) / PTS;

  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t p0 = tile * PTS;
    // ---------------- build the first-layer input ----------------
    for (int i = tid; i < K0 * TM; i += FT) act[i] = 0.f;
    __syncthreads();
    {
      const int m = tid & 63, q = tid >> 6;  // 4 threads per row, 8 features each
      const int pm = (MODE == 1) ? (m & 31) : m;
      const int64_t p = p0 + pm;
      const bool valid = p < prm.P;
      auto st = [&](int col, float v) { act[col * TM + m] = v; };
      if (valid) {
        const int64_t ps = (MODE == 2) ? p : field_src(prm.in, p);   // where this point's neighbour data lives
        if (MODE == 1 && m >= 32) {
          if (q == 0) store_scalar_pe_tangent(prm.in.ds[ps], 0, L.Ld, st);
        } else {
          float x[8];
          blend8(MODE == 2 ? prm.tab.fc : prm.tab.fg, prm.in, ps, q, x);
          store_feat_pe(x, q, MODE == 2 ? L.off_ft : L.off_fg, MODE == 2 ? L.Lft : L.Lfg, st);
          if (q == 0) store_scalar_pe(prm.in.ds[ps], 0, L.Ld, st);
          if (MODE == 2 && q == 1) {
            float dx, dy, dz;
            load_dir(prm.in, p, dx, dy, dz);
            store_vec3_pe(dx, dy, dz, L.off_view, L.Lv, st);
          }
          if (MODE == 2 && q == 2 && L.use_nabla) {
            st(L.off_nabla + 0, prm.in.nabla[0 * prm.in.stride + p]);
            st(L.off_nabla + 1, prm.in.nabla[1 * prm.in.stride + p]);
            st(L.off_nabla + 2, prm.in.nabla[2 * prm.in.stride + p]);
          }
        }
      }
    }
    __syncthreads();

    // ---------------- hidden layers ----------------
    for (int l = 0; l < prm.n_layers; ++l) {
      const int K = prm.K[l];
      const float* __restrict__ wl = prm.w + prm.w_off[l];
      float acc[4][16];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 16; ++j) acc[i][j] = 0.f;
      const int n_chunks = K / KC;
      load_w_chunk(wbuf, wl);
      for (int c = 0; c < n_chunks; ++c) {
        if (c + 1 < n_chunks) {
          load_w_chunk(wbuf + ((c + 1) & 1) * KC * 256, wl + (int64_t)(c + 1) * KC * 256);
          __pipeline_wait_prior(1);
        } else {
          __pipeline_wait_prior(0);
        }
        __syncthreads();
        const float* wc = wbuf + (c & 1) * KC * 256;
        const float* ac = act + (c * KC) * TM + ty * 4;
#pragma unroll
        for (int kk = 0; kk < KC; ++kk) {
          const float4 a = *reinterpret_cast<const float4*>(ac + kk * TM);
          const float av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float4 b = *reinterpret_cast<const float4*>(wc + kk * 256 + j * 64 + tx * 4);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              acc[i][j * 4 + 0] = fmaf(av[i], b.x, acc[i][j * 4 + 0]);
              acc[i][j * 4 + 1] = fmaf(av[i], b.y, acc[i][j * 4 + 1]);
              acc[i][j * 4 + 2] = fmaf(av[i], b.z, acc[i][j * 4 + 2]);
              acc[i][j * 4 + 3] = fmaf(av[i], b.w, acc[i][j * 4 + 3]);
            }
          }
        }
        __syncthreads();
      }
      // epilogue: every thread has finished reading act (barrier above)
      const float* bl = prm.b + l * 256;
      const bool tangent_rows = (MODE == 1) && (ty >= 8);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int n = j * 64 + tx * 4 + jj;
          const float bias = bl[n];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int m = ty * 4 + i;
            const float z = acc[i][j * 4 + jj] + bias;
            if (MODE == 2) {
              act[n * TM + m] = fmaxf(z, 0.f);
            } else if (!tangent_rows) {
              act[n * TM + m] = softplus100(z);
              if (MODE == 1) act[n * TM + m + 32] = softplus100_grad(z);
            }
          }
        }
      }
      if (MODE == 1) {
        __syncthreads();
        if (tangent_rows) {
#pragma unroll
          for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const int n = j * 64 + tx * 4 + jj;
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const int m = ty * 4 + i;
                act[n * TM + m] = act[n * TM + m] * acc[i][j * 4 + jj];  // sigma'(z) * (W t)
              }
            }
        }
      }
      __syncthreads();
    }

    // ---------------- output layer ----------------
    if (MODE == 2) {
      if (tid < 192) {
        const int m = tid & 63, c = tid >> 6;
        const float* wo = prm.w_out + c * 256;
        float s = 0.f;
        for (int n = 0; n < 256; ++n) s = fmaf(act[n * TM + m], wo[n], s);
        s += prm.b_out[c];
        const int64_t p = p0 + m;
        if (p < prm.P) prm.out0[c * prm.in.stride + p] = sigmoid_acc(s);
      }
    } else {
      float s = 0.f;
      if (tid < 64) {
        for (int n = 0; n < 256; ++n) s = fmaf(act[n * TM + tid], prm.w_out[n], s);
      }
      if (MODE == 0) {
        if (tid < 64 && p0 + tid < prm.P) prm.out0[p0 + tid] = s + prm.b_out[0];
      } else {
        const int64_t p = p0 + (tid & 31);
        if (tid < 32 && p < prm.P) prm.out0[p] = s + prm.b_out[0];
        if (tid >= 32 && tid < 64 && p < prm.P && prm.out1) {
          // nabla = (d sdf / d ds) * grad_xyz ds
          const int64_t ps = field_src(prm.in, p);
          prm.out1[0 * prm.in.stride + p] = s * prm.in.grad[0 * prm.in.stride + ps];
          prm.out1[1 * prm.in.stride + p] = s * prm.in.grad[1 * prm.in.stride + ps];
          prm.out1[2 * prm.in.stride + p] = s * prm.in.grad[2 * prm.in.stride + ps];
        }
      }
    }
    __syncthreads();
  }
}

template <int MODE>
static int launch_ffma(const nmb_field* f, const MlpFfma& mlp, const FieldIn& in, int64_t P, float* out0, float* out1,
                       cudaStream_t stream) {
  if (P <= 0) return 0;
  FfmaParams prm;
  prm.lay = f->lay;
  prm.in = in;
  prm.tab = FieldTables{f->fg.p, in.color_table ? in.color_table : f->fc.p};
  prm.w = mlp.w.p;
  prm.b = mlp.b.p;
  prm.w_out = mlp.w_out.p;
  prm.b_out = mlp.b_out.p;
  for (int i = 0; i < MAX_LAYERS; ++i) {
    prm.w_off[i] = mlp.w_off[i];
    prm.K[i] = mlp.K[i];
  }
  prm.n_layers = mlp.n_layers;
  prm.P = P;
  prm.out0 = out0;
  prm.out1 = out1;
  constexpr int PTS = (MODE == 1) ? 32 : 64;
  const size_t smem = (256 * TM + 2 * KC * 256) * sizeof(float);
  static DeviceOnce attr_once;
  NMB_CUDA_OK(attr_once.run([&] {
    return cudaFuncSetAttribute(mlp_ffma_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  }));
  const int64_t tiles = ceil_div(P, PTS);
  const int64_t grid = tiles < (int64_t)2 * sm_count() ? tiles : (int64_t)2 * sm_count();
  ProfScope prof(MODE == 2 ? PROF_COLOR : (MODE == 1 ? PROF_GEO_JVP : PROF_GEO), P, stream);
  mlp_ffma_kernel<MODE><<<(unsigned)grid, FT, smem, stream>>>(prm);
  NMB_LAUNCH_OK();
  return 0;
}

int launch_geo_ffma(const nmb_field* f, const FieldIn& in, int64_t P, float* sdf, float* nabla, cudaStream_t stream) {
  if (nabla) return launch_ffma<1>(f, f->geo_f, in, P, sdf, nabla, stream);
  return launch_ffma<0>(f, f->geo_f, in, P, sdf, nullptr, stream);
}

int launch_color_ffma(const nmb_field* f, const FieldIn& in, int64_t P, float* rgb, cudaStream_t stream) {
  return launch_ffma<2>(f, f->col_f, in, P, rgb, nullptr, stream);
}

}  // namespace nmb
