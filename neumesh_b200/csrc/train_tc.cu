// 3xTF32 tensor-core GEMM of the training path (train_engine = "tf32x3"): nmb_tr_gemm's contract - C[M,N] (+)= A.B
// (+ bias, relu | mask), A and B each K-contiguous or not, any leading dimensions, split-K for long reductions - on
// Hopper's wgmma.
//
// Precision.  Every operand x is split into x_hi = tf32(x) and x_lo = tf32(x - x_hi) and each product is issued as
// D += A_lo.B_hi + A_hi.B_lo + A_hi.B_hi with fp32 accumulation (the render path's mlp_engine = "tcgen05" scheme).
// TF32 keeps fp32's 8-bit exponent, so the tiny upstream gradients of a training step (loss / M, eikonal and colour
// terms) are represented as in fp32; the dropped A_lo.B_lo term and the rounding of the lo parts cost about 2^-20
// |A|.|B| per product on top of the fp32 accumulation error.  The tensor core's own accumulation into D truncates
// (rounds toward zero); over a whole K = 256 chain of 96 MMAs that bias reached ~1e-5 relative on the NeuS teacher and
// 3e-3 on a colour-code gradient of the training step.  So each K step's 6 MMAs go to a fresh accumulator that is added
// to the running sum with an fp32 FADD (round to nearest): truncation acts on 6-MMA chains only.
//
// Tiles.  A CTA computes a 128 x 128 tile of C with two warpgroups (rows 0-63 and 64-127, wgmma m64n128k8, 64
// accumulator registers per thread), K in steps of 16.  Operands are staged through registers: coalesced scalar global
// loads (any stride, ragged K and M / N edges read as zeros), the hi / lo split, then 16-byte stores into the
// no-swizzle K-major core-matrix layout of wgmma.cuh ([k/4][row][k%4], one hi and one lo image per operand).  The same
// step does the transposition of a non-K-contiguous operand, so all four layouts share one pipeline.  Two shared-memory
// stages (64 KB) and one __syncthreads per K step: while step t's MMAs run, the threads stage step t + 1 into the other
// buffer and issue the global loads of step t + 2; then they wait for the MMAs and add the step's products.  The two
// 64-register accumulators need more than 128 registers per thread: one CTA per SM.
//
// Split-K.  When the output has fewer than SPLIT_CTAS tiles, K >= 4096 and the epilogue is plain (the weight-gradient
// products, K = number of points), K is cut into equal BK-aligned chunks, each CTA writes its chunk's partial product to
// scratch and reduce_splits_kernel (train.cu) adds the partials in split order.  The plan depends on (M, N, K) alone,
// never on the device, so the result is bit-reproducible with or without torch.use_deterministic_algorithms.
#include "../../include/neumesh_b200.h"
#include "common.cuh"
#include "wgmma.cuh"

namespace nmb {
namespace tr {

// C (+)= sum_z part[z * split_stride + m * N + n] in z order (train.cu: reduce_splits_kernel)
int reduce_splits(const float* part, int splits, int64_t split_stride, int64_t M, int64_t N, float* C, int64_t ldc,
                  int accumulate, cudaStream_t stream);

namespace tf32x3 {

constexpr int BM = 128, BN = 128, BK = 16, THREADS = 256;
constexpr int A_HALF = BM * BK * 4;                    // 8 KB: the hi (or lo) image of a 128 x 16 A tile
constexpr int B_HALF = BN * BK * 4;
constexpr int STAGE = 2 * A_HALF + 2 * B_HALF;         // 32 KB
constexpr int SMEM = 2 * STAGE;                        // 64 KB: two stages
constexpr int SPLIT_CTAS = 264;                        // CTAs a split-K product aims for (two waves on a 132-SM H100)

// Staging unit: 4 consecutive K-columns [4 kc, 4 kc + 4) of one tile row (one 16-byte core-matrix row).  A tile is
// 128 rows x 4 kc = 512 units, two per thread.  K-contiguous operands: a warp takes 8 rows x 4 kc (each row's 64 bytes
// are read together; the 8 threads of a quarter warp store 8 consecutive rows of one kc, 128 contiguous bytes).
// Row-contiguous operands: a warp takes 32 consecutive rows of one kc (128-byte loads per k, 512 contiguous bytes stored).
template <bool KC>
__device__ __forceinline__ void unit_pos(int u, int& row, int& kc) {
  if (KC) {
    row = (u & 7) | ((u >> 5) << 3);
    kc = (u >> 3) & 3;
  } else {
    row = u & (BM - 1);
    kc = u >> 7;
  }
}

// X(r, k) = KC ? X[r * ld + k] : X[k * ld + r] for r < rows, k < k_end; 0 elsewhere
template <bool KC>
__device__ __forceinline__ void load_units(const float* __restrict__ X, int64_t ld, int rows, int r0, int k0, int k_end,
                                           float (&v)[2][4]) {
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    int row, kc;
    unit_pos<KC>(threadIdx.x + i * THREADS, row, kc);
    const int gr = r0 + row;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gk = k0 + 4 * kc + j;
      float x = 0.f;
      if (gr < rows && gk < k_end) x = KC ? X[(int64_t)gr * ld + gk] : X[(int64_t)gk * ld + gr];
      v[i][j] = x;
    }
  }
}

template <bool KC>
__device__ __forceinline__ void store_units(char* img, int half_bytes, const float (&v)[2][4]) {
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    int row, kc;
    unit_pos<KC>(threadIdx.x + i * THREADS, row, kc);
    float4 hi, lo;
    hi.x = tc::tf32_rna(v[i][0]);
    hi.y = tc::tf32_rna(v[i][1]);
    hi.z = tc::tf32_rna(v[i][2]);
    hi.w = tc::tf32_rna(v[i][3]);
    lo.x = tc::tf32_rna(v[i][0] - hi.x);
    lo.y = tc::tf32_rna(v[i][1] - hi.y);
    lo.z = tc::tf32_rna(v[i][2] - hi.z);
    lo.w = tc::tf32_rna(v[i][3] - hi.w);
    char* dst = img + kc * (BM * 16) + row * 16;
    *reinterpret_cast<float4*>(dst) = hi;
    *reinterpret_cast<float4*>(dst + half_bytes) = lo;
  }
}

__device__ __forceinline__ void fence_acc(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

template <bool A_KC, bool B_KC>
__global__ void __launch_bounds__(THREADS, 1)
gemm_tf32x3_kernel(int M, int N, int K, const float* __restrict__ A, int64_t lda, const float* __restrict__ B,
                   int64_t ldb, float* __restrict__ C, int64_t ldc, const float* __restrict__ bias, int epi,
                   const float* __restrict__ mask, int64_t ldmask, int accumulate, int gn, int k_chunk,
                   int64_t split_stride) {
  extern __shared__ __align__(128) char smem[];
  const int tid = threadIdx.x, wg = tid >> 7;
  const int n0 = (int)(blockIdx.x % gn) * BN, m0 = (int)(blockIdx.x / gn) * BM;
  const int k_begin = blockIdx.z * k_chunk;
  const int k_end = min(K, k_begin + k_chunk);
  const int steps = k_begin < k_end ? (k_end - k_begin + BK - 1) / BK : 0;
  const uint32_t s_base = tc::smem_u32(smem);

  // d: the running sum; acc: one K step's products, added to d by FADD once they are complete
  float d[64], acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) d[i] = 0.f;
  float ra[2][4], rb[2][4];   // the operands of the next step to be staged
  auto load = [&](int t) {
    load_units<A_KC>(A, lda, M, m0, k_begin + t * BK, k_end, ra);
    load_units<B_KC>(B, ldb, N, n0, k_begin + t * BK, k_end, rb);
  };
  auto stage = [&](int t) {
    char* st = smem + (t & 1) * STAGE;
    store_units<A_KC>(st, A_HALF, ra);
    store_units<B_KC>(st + 2 * A_HALF, B_HALF, rb);
    tc::fence_proxy_async();
  };
  if (steps > 0) {
    load(0);
    stage(0);
    if (steps > 1) load(1);
  }
  __syncthreads();
  for (int t = 0; t < steps; ++t) {
    const uint32_t sa = s_base + (t & 1) * STAGE + wg * (64 * 16), sb = s_base + (t & 1) * STAGE + 2 * A_HALF;
    tc::wg_fence();
#pragma unroll
    for (int ks = 0; ks < BK / 8; ++ks) {
      const uint64_t a_hi = tc::make_desc(sa + ks * 2 * (BM * 16), BM * 16, 128);
      const uint64_t a_lo = tc::make_desc(sa + A_HALF + ks * 2 * (BM * 16), BM * 16, 128);
      const uint64_t b_hi = tc::make_desc(sb + ks * 2 * (BN * 16), BN * 16, 128);
      const uint64_t b_lo = tc::make_desc(sb + B_HALF + ks * 2 * (BN * 16), BN * 16, 128);
      tc::mma_tf32_n128(acc, a_lo, b_hi, ks == 0 ? 0u : 1u);   // the step's first MMA overwrites acc
      tc::mma_tf32_n128(acc, a_hi, b_lo, 1u);
      tc::mma_tf32_n128(acc, a_hi, b_hi, 1u);
    }
    tc::wg_commit();
    // under the MMAs: stage step t + 1 into the other buffer (its readers, step t - 1's MMAs, completed before the
    // last __syncthreads) and start the global loads of step t + 2
    if (t + 1 < steps) {
      stage(t + 1);
      if (t + 2 < steps) load(t + 2);
    }
    tc::wg_wait<0>();
    fence_acc(acc);
#pragma unroll
    for (int i = 0; i < 64; ++i) d[i] += acc[i];
    __syncthreads();
  }

  // d[4 n8 + 2 hh + jj] = D(row 16 warp + lane / 4 + 8 hh, col 8 n8 + 2 (lane % 4) + jj) of the warpgroup's 64 rows
  const int lane = tid & 31, warp = (tid >> 5) & 3;
  float* Cz = C + (int64_t)blockIdx.z * split_stride;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int gm = m0 + wg * 64 + warp * 16 + (lane >> 2) + 8 * hh;
    if (gm >= M) continue;
#pragma unroll
    for (int n8 = 0; n8 < BN / 8; ++n8) {
#pragma unroll
      for (int jj = 0; jj < 2; ++jj) {
        const int gn_ = n0 + 8 * n8 + 2 * (lane & 3) + jj;
        if (gn_ >= N) continue;
        float v = d[4 * n8 + 2 * hh + jj];
        if (bias) v += bias[gn_];
        if (epi == 1) v = fmaxf(v, 0.f);
        if (epi == 2) v = (mask[(int64_t)gm * ldmask + gn_] > 0.f) ? v : 0.f;
        float* dst = Cz + (int64_t)gm * ldc + gn_;
        if (accumulate) v += *dst;
        *dst = v;
      }
    }
  }
}

static DeviceOnce g_attr_once;

static cudaError_t set_attributes() {
  return g_attr_once.run([] {
    cudaError_t e = cudaFuncSetAttribute(gemm_tf32x3_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(gemm_tf32x3_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(gemm_tf32x3_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(gemm_tf32x3_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    return e;
  });
}

}  // namespace tf32x3
}  // namespace tr
}  // namespace nmb

extern "C" int nmb_tr_gemm_tc(const float* A, int64_t lda, int a_kcontig, const float* B, int64_t ldb, int b_kcontig,
                              float* C, int64_t ldc, int64_t M, int64_t N, int64_t K, const float* bias, int epilogue,
                              const float* mask, int64_t ldmask, int accumulate, void* stream_) {
  using namespace nmb;
  using namespace nmb::tr::tf32x3;
  NMB_CHECK(A && B && C, "null argument");
  NMB_CHECK(M < (int64_t(1) << 31) && N < (int64_t(1) << 31) && K < (int64_t(1) << 31), "dimension too large");
  NMB_CHECK(epilogue >= 0 && epilogue <= 2 && (epilogue != 2 || mask), "bad epilogue");
  if (M <= 0 || N <= 0) return 0;
  const int64_t gm = ceil_div(M, BM), gn = ceil_div(N, BN);
  NMB_CHECK(gm * gn < (int64_t(1) << 31), "dimension too large");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  NMB_CUDA_OK(set_attributes());
  int splits = 1;
  if (gm * gn < SPLIT_CTAS && K >= 4096 && !bias && epilogue == 0)
    splits = (int)std::min<int64_t>(ceil_div(SPLIT_CTAS, gm * gn), ceil_div(K, 1024));
  const int k_chunk = splits > 1 ? (int)align_up(ceil_div(K, splits), BK) : (int)(K > 0 ? K : 1);
  if (splits > 1) splits = (int)ceil_div(K, k_chunk);
  float* Cdst = C;
  int64_t ldd = ldc, split_stride = 0;
  StreamBuf part;
  if (splits > 1) {
    NMB_CUDA_OK(part.alloc(sizeof(float) * (size_t)splits * M * N, stream));
    Cdst = part.as<float>();
    ldd = N;
    split_stride = M * N;
  }
  const int acc = splits > 1 ? 0 : accumulate;
  dim3 grid((unsigned)(gm * gn), 1, (unsigned)splits);
#define NMB_TC_LAUNCH(AK, BKC)                                                                                     \
  gemm_tf32x3_kernel<AK, BKC><<<grid, THREADS, SMEM, stream>>>((int)M, (int)N, (int)K, A, lda, B, ldb, Cdst, ldd, \
                                                               bias, epilogue, mask, ldmask, acc, (int)gn,        \
                                                               k_chunk, split_stride)
  if (a_kcontig && b_kcontig) NMB_TC_LAUNCH(true, true);
  else if (a_kcontig) NMB_TC_LAUNCH(true, false);
  else if (b_kcontig) NMB_TC_LAUNCH(false, true);
  else NMB_TC_LAUNCH(false, false);
#undef NMB_TC_LAUNCH
  NMB_LAUNCH_OK();
  if (splits > 1) return nmb::tr::reduce_splits(Cdst, splits, split_stride, M, N, C, ldc, accumulate, stream);
  return 0;
}
