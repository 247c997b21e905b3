// Tensor-core MLP engines for Hopper (sm_90a; mlp_engine = 2: fp16x3 split operands, the default; mlp_engine = 0:
// 3xTF32): the NeuMesh geometry / colour MLPs on wgmma.  The Python-side engine names ("tcgen05_f16", "tcgen05") are
// kept for API compatibility.
//
// Why split operands.  The sdf feeds sigmoid(s * sdf) with s ~ 50-300 and a discrete re-sampling cascade; single-pass TF32
// (10-bit mantissa) or BF16 operands miss the 1e-4 / 1e-5 parity bar by 1-3 orders of magnitude, while the split
// x = hi + lo (both TF32), D += A_hi*B_hi + A_hi*B_lo + A_lo*B_hi with fp32 accumulation is fp32-accurate
// (SURVEY.md section 7.3); the fp16 variant (hi = fp16(x), lo = fp16(x - hi), weights pre-scaled by 2^8) is as accurate
// at twice the MMA rate and half the operand bytes.  Every algorithmic MAC is therefore issued three times.
//
// One persistent CTA per SM.  Every consumer warpgroup owns a 64-row tile (points, or their tangent rows d/d(ds) in the
// geometry + tangent mode, see below) and does all the work for it:
//   * layer 0: its threads build the first-layer A slabs (neighbour gather + blend + positional encoding, 2 threads per
//     row) into a 2-step ring inside the warpgroup's shared-memory region; the wgmma of step s runs while step s + 1 is
//     being built;
//   * every layer: wgmma m64n256 (k16 fp16 / k8 tf32) with the 64x256 fp32 accumulator in registers (128 per thread);
//   * epilogue: bias + activation, hi/lo split, the whole next-layer A operand (64 rows x 256 K) written back into the
//     region, or the output layer's dot products (quad shuffles) for the last layer.
// The fp16 engine runs two consumer warpgroups per CTA (two 64 KB regions), the TF32 engine one (its A operand is
// 128 KB).  One producer thread streams the weight slabs L2 -> shared memory with cp.async.bulk into a ring that the
// CTA's warpgroups consume in lock step (mbarrier full / empty pairs).
//
// Geometry + tangent mode (MODE 1).  fp16 engine: warpgroup 0 holds the 64 value rows of a CTA tile, warpgroup 1 the 64
// tangent rows of the same points in the same order, so accumulator fragment i of thread t is the same (point, column)
// in both.  A tangent row's first-layer input is zero outside the head block, so warpgroup 1 builds and multiplies only
// the ring steps holding head columns and just releases the others.  In each epilogue warpgroup 0 hands e = exp(100 z)
// to warpgroup 1 one column eighth at a time through two shared-memory buffers (named-barrier full / empty pairs), so
// the value and tangent formulas run on all four SM sub-partitions and pipeline across eighths.  TF32 engine (one
// consumer warpgroup): rows 32..63 of a tile carry d/d(ds) of rows 0..31, exchanged one column quarter at a time.
//
// Operand layout (no swizzle, K-major canonical layout): a K-slab of 16 columns is stored as [k/4][row][k%4] fp32 (tf32)
// or [k/8][row][k%8] fp16, i.e. 8x16-byte core matrices with SBO = 128 B (next 8 rows) and LBO = rows*16 B (next
// k chunk).  Weights are pre-packed in exactly this image (hi slab then lo slab), so a slab is one contiguous copy.
#include <cuda_fp16.h>

#include <type_traits>
#include <vector>

#include "field_build.cuh"

namespace nmb {

namespace tc {

constexpr int ROWS = 64;                      // rows of a warpgroup tile (wgmma M)
constexpr int SLAB_K = 16;                    // K columns per slab
constexpr int B_HALF32 = MLP_W * SLAB_K * 4;  // 16 KB: one hi (or lo) tf32 weight slab
constexpr int B_SLOT32 = 2 * B_HALF32;        // 32 KB
constexpr int B_HALF16 = MLP_W * SLAB_K * 2;  // 8 KB: one hi (or lo) fp16 weight slab
constexpr int B_SLOT16 = 2 * B_HALF16;        // 16 KB
constexpr float F16_W_SCALE = 256.f;          // weights are packed as 2^8 W (keeps their lo parts out of the subnormals)
// fp16 engine: GR16 = 2 slabs (32 K-columns) per pipeline step, i.e. per weight-ring slot and barrier pair; the first
// layer is padded with zero slabs to whole steps
constexpr int GR16 = 2;
constexpr int NB = 2;                         // weight ring depth (steps)
constexpr int NA0 = 2;                        // first-layer A ring depth (steps) inside a warpgroup's region
constexpr int CONST_FLOATS = (MAX_LAYERS + 3) * MLP_W;   // biases of every hidden layer + up to 3 output rows
// MODE 1 exchange area per consumer warpgroup: exp(100 z) of one column quarter of 32 value rows (TF32 engine), or one
// of the fp16 engine's two column-eighth buffers ([16 values][128 threads])
constexpr int SIG_FLOATS = 64 * 32;
static_assert(SIG_FLOATS == 16 * 128, "an fp16 exchange buffer holds one column eighth of a warpgroup's accumulator");
// fp16 MODE 1 exchange: named barriers (0 is __syncthreads, 1..2 the consumer warpgroups') of buffers 0 / 1
constexpr uint32_t EX_FULL = 3, EX_EMPTY = 5;

template <bool F16>
struct Cfg {
  static constexpr int NWG = F16 ? 2 : 1;                        // consumer warpgroups per CTA
  static constexpr int GR = F16 ? GR16 : 1;                      // slabs per pipeline step
  static constexpr int A_HALF = ROWS * SLAB_K * (F16 ? 2 : 4);   // one hi (or lo) A slab
  static constexpr int A_SUB = 2 * A_HALF;                       // one A slab, hi + lo
  static constexpr int A_REGION = (MLP_W / SLAB_K) * A_SUB;      // a whole 256-column A operand: 64 KB / 128 KB
  static constexpr int B_HALF = F16 ? B_HALF16 : B_HALF32;
  static constexpr int B_SUB = F16 ? B_SLOT16 : B_SLOT32;
  static constexpr int B_STEP = GR * B_SUB;                      // 32 KB
  // + the producer: one warp, or with two consumer warpgroups a whole warpgroup so that setmaxnreg can hand its
  // registers to the consumers (a 288-thread block would cap every thread at 168 registers and spill the accumulator)
  static constexpr int THREADS = NWG * 128 + (NWG > 1 ? 128 : 32);
  static constexpr int REGS_CONSUMER = 232, REGS_PRODUCER = 40;  // NWG > 1: 2 * 128 * 232 + 128 * 40 <= 65536
};

// points per CTA tile: 64 per consumer warpgroup; MODE 1 also needs a tangent row per point, held by the second
// warpgroup in the fp16 engine and by the upper half of the tile in the TF32 engine
template <int MODE, bool F16>
constexpr int tile_points() {
  return MODE != 1 ? Cfg<F16>::NWG * ROWS : (F16 ? ROWS : ROWS / 2);
}

// SIG: the geometry + tangent instantiation exchanges exp(100 z) between value and tangent rows
template <bool F16, bool SIG>
struct SmemLayoutT {
  using C = Cfg<F16>;
  static constexpr int a_off = 0;
  static constexpr int b_off = C::NWG * C::A_REGION;
  static constexpr int sig_off = b_off + NB * C::B_STEP;
  static constexpr int const_off = sig_off + (SIG ? C::NWG * SIG_FLOATS * 4 : 0);
  static constexpr int bar_off = const_off + CONST_FLOATS * 4;
  static constexpr int total = bar_off + 2 * NB * 8;
};
static_assert(SmemLayoutT<true, true>::total <= 232448 && SmemLayoutT<false, true>::total <= 232448,
              "shared memory budget (227 KB per block)");
static_assert(NA0 * Cfg<true>::GR * Cfg<true>::A_SUB <= Cfg<true>::A_REGION &&
              NA0 * Cfg<false>::GR * Cfg<false>::A_SUB <= Cfg<false>::A_REGION, "first-layer ring fits the region");

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
  } while (!done);
}
// the producer thread backs off between polls so its spin does not steal issue slots from the consumer warps
__device__ __forceinline__ void mbar_wait_backoff(uint32_t bar, uint32_t parity) {
  uint32_t done;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (done) break;
    __nanosleep(40);
  }
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}

// wgmma shared-memory matrix descriptor, no swizzle: start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46), layout 0 [62,64)
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  return d;
}

__device__ __forceinline__ void named_sync(uint32_t id, uint32_t threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
__device__ __forceinline__ void named_arrive(uint32_t id, uint32_t threads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator accesses across the asynchronous MMA's issue / wait points
__device__ __forceinline__ void fence_acc(float (&d)[128]) {
#pragma unroll
  for (int i = 0; i < 128; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Accumulator fragment of m64n256: d[4 n8 + 2 hh + jj] = D(row 16 warp + lane / 4 + 8 hh, col 8 n8 + 2 (lane % 4) + jj)
#define NMB_WG_D \
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, " \
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, " \
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, " \
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, " \
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, " \
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, " \
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, " \
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"

#define NMB_WG_OPS \
        "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), \
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), \
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), \
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), \
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), \
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), \
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), \
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), \
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), \
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), \
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), \
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), \
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])

__device__ __forceinline__ void mma_f16(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {" NMB_WG_D "}, %128, %129, p, 1, 1, 0, 0;\n\t}"
      : NMB_WG_OPS
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void mma_tf32(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {" NMB_WG_D "}, %128, %129, p, 1, 1;\n\t}"
      : NMB_WG_OPS
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
#undef NMB_WG_D
#undef NMB_WG_OPS

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ float tf32_rna(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}

// write 8 consecutive K-columns [8h, 8h+8) of row `r` (two 4-column chunks) into a tf32 A slab: hi, then lo
__device__ __forceinline__ void store_a_half(char* a_slot, int r, int h, const float (&v)[8]) {
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    const int kc = 2 * h + c;
    float4 hi, lo;
    hi.x = tf32_rna(v[c * 4 + 0]);
    hi.y = tf32_rna(v[c * 4 + 1]);
    hi.z = tf32_rna(v[c * 4 + 2]);
    hi.w = tf32_rna(v[c * 4 + 3]);
    lo.x = tf32_rna(v[c * 4 + 0] - hi.x);
    lo.y = tf32_rna(v[c * 4 + 1] - hi.y);
    lo.z = tf32_rna(v[c * 4 + 2] - hi.z);
    lo.w = tf32_rna(v[c * 4 + 3] - hi.w);
    *reinterpret_cast<float4*>(a_slot + kc * (ROWS * 16) + r * 16) = hi;
    *reinterpret_cast<float4*>(a_slot + Cfg<false>::A_HALF + kc * (ROWS * 16) + r * 16) = lo;
  }
}

// fp16 variant: the 8 columns [8h, 8h+8) of row `r` are ONE 16-byte chunk ([k/8][row][k%8] halves);
// hi = fp16(x), lo = fp16(x - hi) (lo may be subnormal: absolute error <= 2^-25, see tools/split_precision_study.py)
__device__ __forceinline__ void store_a_half_f16(char* a_slot, int r, int h, const float (&v)[8]) {
  uint32_t hi[4], lo[4];
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const __half2 hp = __floats2half2_rn(v[2 * c], v[2 * c + 1]);   // .x (low 16 bits) = even column
    const float2 hf = __half22float2(hp);
    const __half2 lp = __floats2half2_rn(v[2 * c] - hf.x, v[2 * c + 1] - hf.y);
    hi[c] = *reinterpret_cast<const uint32_t*>(&hp);
    lo[c] = *reinterpret_cast<const uint32_t*>(&lp);
  }
  *reinterpret_cast<uint4*>(a_slot + h * (ROWS * 16) + r * 16) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
  *reinterpret_cast<uint4*>(a_slot + Cfg<true>::A_HALF + h * (ROWS * 16) + r * 16) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
}

// the two adjacent columns (c, c + 1) of row `r` of a whole-layer A operand (epilogue -> next layer)
template <bool F16>
__device__ __forceinline__ void store_a_pair(char* region, int r, int c, float x0, float x1) {
  using C = Cfg<F16>;
  char* slab = region + (c >> 4) * C::A_SUB;
  const int k = c & 15;
  if constexpr (F16) {
    const __half2 hp = __floats2half2_rn(x0, x1);
    const float2 hf = __half22float2(hp);
    const __half2 lp = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
    char* dst = slab + (k >> 3) * (ROWS * 16) + r * 16 + (k & 7) * 2;
    *reinterpret_cast<__half2*>(dst) = hp;
    *reinterpret_cast<__half2*>(dst + C::A_HALF) = lp;
  } else {
    const float h0 = tf32_rna(x0), h1 = tf32_rna(x1);
    char* dst = slab + (k >> 2) * (ROWS * 16) + r * 16 + (k & 3) * 4;
    *reinterpret_cast<float2*>(dst) = make_float2(h0, h1);
    *reinterpret_cast<float2*>(dst + C::A_HALF) = make_float2(tf32_rna(x0 - h0), tf32_rna(x1 - h1));
  }
}

struct Params {
  FieldLayout lay;
  FieldIn in;
  FieldTables tab;
  const float* w;          // packed slabs
  const float* bias;       // [n_layers][256]
  const float* w_out;      // [n_out][256]
  const float* b_out;
  int64_t slab_off[MAX_LAYERS];  // floats
  int n_slabs[MAX_LAYERS];
  int n_layers;
  int64_t P;
  float* out0;
  float* out1;
};

}  // namespace tc

// MODE 0: geometry.  MODE 1: geometry + tangent rows d/d(ds) (fp16: warpgroup 1 holds the tangent rows of warpgroup 0's
// points; TF32: rows 32..63 of the tile carry the tangents of rows 0..31).  MODE 2: colour.
// F16 = false: 3xTF32 operands (mlp_engine 0).  F16 = true: fp16x3 operands (mlp_engine 2).
template <int MODE, bool F16 = false>
__global__ void __launch_bounds__(tc::Cfg<F16>::THREADS, 1) mlp_tc_kernel(const tc::Params prm) {
  using namespace tc;
  using C = Cfg<F16>;
  using SmemLayout = SmemLayoutT<F16, MODE == 1>;
  constexpr int NWG = C::NWG, GR = C::GR, A_SUB = C::A_SUB, B_SUB = C::B_SUB;
  constexpr bool SPLIT = (MODE == 1) && F16;            // value and tangent rows in separate warpgroups
  constexpr bool HALF_ROWS = (MODE == 1) && !SPLIT;     // rows 32..63 of a tile: the tangents of rows 0..31
  constexpr int PTS = HALF_ROWS ? ROWS / 2 : ROWS;      // points per warpgroup tile
  constexpr int TILE_PTS = tile_points<MODE, F16>();    // points per CTA tile
  extern __shared__ __align__(1024) char smem[];
  float* cst = reinterpret_cast<float*>(smem + SmemLayout::const_off);   // [n_layers][256] biases, then output rows
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + SmemLayout::bar_off);
  constexpr int B_FULL = 0, B_EMPTY = NB;
  const uint32_t bar0 = smem_u32(bars);
  auto bar = [&](int i) { return bar0 + 8u * (uint32_t)i; };
  const uint32_t b_base = smem_u32(smem + SmemLayout::b_off);

  const int tid = threadIdx.x;
  const int64_t n_tiles = (prm.P + TILE_PTS - 1) / TILE_PTS;
  const FieldLayout& L = prm.lay;
  const int NL = prm.n_layers;

  if (tid == 0) {
    for (int i = 0; i < NB; ++i) {
      mbar_init(bar(B_FULL + i), 1);
      mbar_init(bar(B_EMPTY + i), 4 * NWG);   // released by lane 0 of every consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  {
    const int n_out = (MODE == 2) ? 3 : 1;
    for (int i = tid; i < prm.n_layers * MLP_W; i += C::THREADS) cst[i] = prm.bias[i];
    for (int i = tid; i < n_out * MLP_W; i += C::THREADS) cst[prm.n_layers * MLP_W + i] = prm.w_out[i];
  }
  __syncthreads();

  if (tid >= NWG * 128) {
    // =========================================== weight producer ====================================
    if constexpr (NWG > 1) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(C::REGS_PRODUCER));
    if (tid == NWG * 128) {
      uint32_t q = 0;
      for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        for (int l = 0; l < NL; ++l) {
          const float* src = prm.w + prm.slab_off[l];
          for (int j = 0; j < prm.n_slabs[l]; j += GR, ++q) {   // GR consecutive slabs are contiguous in the image
            const uint32_t sb = q % NB;
            mbar_wait_backoff(bar(B_EMPTY + sb), ((q / NB) & 1u) ^ 1u);
            mbar_expect_tx(bar(B_FULL + sb), C::B_STEP);
#pragma unroll
            for (int hf = 0; hf < 2; ++hf)
              bulk_load(b_base + sb * C::B_STEP + hf * (C::B_STEP / 2), src + (int64_t)j * (B_SUB / 4) + hf * (C::B_STEP / 8),
                        C::B_STEP / 2, bar(B_FULL + sb));
          }
        }
      }
    }
    return;
  }

  // ============================================= consumer warpgroup =================================
  if constexpr (NWG > 1) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(C::REGS_CONSUMER));
  const int wg = tid >> 7, t = tid & 127, warp = t >> 5, lane = t & 31;
  char* region = smem + SmemLayout::a_off + wg * C::A_REGION;
  const uint32_t a_base = smem_u32(region);
  // SPLIT: the two exchange buffers, shared by both warpgroups
  float* sig = reinterpret_cast<float*>(smem + SmemLayout::sig_off) + (SPLIT ? 0 : wg * SIG_FLOATS);
  const bool tan_wg = SPLIT && wg == 1;        // every row of this warpgroup is a tangent row
  const uint32_t wg_bar = 1u + (uint32_t)wg;   // named barrier of this warpgroup (0 is __syncthreads)
  auto wg_sync = [&]() { named_sync(wg_bar, 128); };
  if (tan_wg) {   // both exchange buffers start empty
    named_arrive(EX_EMPTY + 0, 256);
    named_arrive(EX_EMPTY + 1, 256);
  }

  float d[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) d[i] = 0.f;
  uint32_t qb = 0;    // weight-ring steps consumed by this warpgroup
  int prev = -1;      // ring slot of the step still in flight (released once its MMAs have completed)

  // one pipeline step: the GR slabs of A at a_addr against the next weight step; returns with at most this step's
  // MMAs in flight
  auto step = [&](uint32_t a_addr, bool first) {
    const uint32_t sb = qb % NB;
    mbar_wait(bar(B_FULL + sb), (qb / NB) & 1u);
    const uint32_t b_addr = b_base + sb * C::B_STEP;
    fence_acc(d);
    wg_fence();
#pragma unroll
    for (int sub = 0; sub < GR; ++sub) {
      if constexpr (F16) {
        // one K = 16 step per slab: two 8-column chunks; chunk stride: A 64 rows * 16 B, B 256 rows * 16 B
        const uint64_t a_hi = make_desc(a_addr + sub * A_SUB, ROWS * 16, 128);
        const uint64_t a_lo = make_desc(a_addr + sub * A_SUB + C::A_HALF, ROWS * 16, 128);
        const uint64_t b_hi = make_desc(b_addr + sub * B_SUB, MLP_W * 16, 128);
        const uint64_t b_lo = make_desc(b_addr + sub * B_SUB + C::B_HALF, MLP_W * 16, 128);
        mma_f16(d, a_lo, b_hi, (first && sub == 0) ? 0u : 1u);   // small terms first
        mma_f16(d, a_hi, b_lo, 1u);
        mma_f16(d, a_hi, b_hi, 1u);
      } else {
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
          // two 4-column chunks per K = 8 step
          const uint64_t a_hi = make_desc(a_addr + sub * A_SUB + ks * 2 * (ROWS * 16), ROWS * 16, 128);
          const uint64_t a_lo = make_desc(a_addr + sub * A_SUB + C::A_HALF + ks * 2 * (ROWS * 16), ROWS * 16, 128);
          const uint64_t b_hi = make_desc(b_addr + sub * B_SUB + ks * 2 * (MLP_W * 16), MLP_W * 16, 128);
          const uint64_t b_lo = make_desc(b_addr + sub * B_SUB + C::B_HALF + ks * 2 * (MLP_W * 16), MLP_W * 16, 128);
          mma_tf32(d, a_lo, b_hi, (first && sub == 0 && ks == 0) ? 0u : 1u);
          mma_tf32(d, a_hi, b_lo, 1u);
          mma_tf32(d, a_hi, b_hi, 1u);
        }
      }
    }
    wg_commit();
    fence_acc(d);
    wg_wait<1>();   // the previous step's MMAs are complete: its weight slot and A slot may be reused
    fence_acc(d);
    if (prev >= 0 && lane == 0) mbar_arrive(bar(B_EMPTY + prev));
    prev = (int)sb;
    ++qb;
  };
  auto finish_layer = [&]() {
    wg_wait<0>();
    fence_acc(d);
    if (lane == 0) mbar_arrive(bar(B_EMPTY + prev));
    prev = -1;
  };

  constexpr float K_EXP = 144.26950408889634f;       // 100 * log2(e)
  constexpr float K_LOG = 0.0069314718055994531f;    // ln(2) / 100
  const int off_feat = (MODE == 2) ? L.off_ft : L.off_fg;   // multiple of 16
  const int Lf = (MODE == 2) ? L.Lft : L.Lfg;
  const int Fdim = (MODE == 2) ? L.Fc : L.Fg;   // code width = n_fb blocks of FEAT columns
  const int n_fb = Fdim / FEAT;
  const float* __restrict__ table = (MODE == 2) ? prm.tab.fc : prm.tab.fg;

  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t pbase = SPLIT ? tile * TILE_PTS : (tile * NWG + wg) * PTS;
    // every warp of the warpgroup has seen the previous tile's last MMAs complete before any of them overwrites the
    // first-layer ring, whose rows the whole warpgroup's MMAs read
    wg_sync();
    // the tile's work for one role: TAN_WG = a SPLIT tangent warpgroup; the value warpgroup's layer 0 is MODE 0's.  The
    // roles are separate instantiations, so neither carries the other's state through the register-bound build
    auto tile_work = [&](auto tan_wg_c) {
      constexpr bool TAN_WG = decltype(tan_wg_c)::value;
      {
        // ===================================== layer 0: build + MMA =====================================
        // (TAN_WG: only the head block; the remaining first-layer steps are released unissued)
        // two threads per row: half h owns features {8g + 4h + i : g < 4, i < 4} and writes columns [8h, 8h+8) of
        // every first-layer slab (see tc_first_layer_map for the column order)
        const int r = t & (ROWS - 1);
        const int h = t >> 6;
        const int64_t p = pbase + (HALF_ROWS ? (r & 31) : r);
        const bool valid = p < prm.P;
        const bool tangent = TAN_WG || (HALF_ROWS && r >= 32);
        uint32_t q = 0;   // first-layer slabs emitted
        auto emit = [&](const float (&v)[8]) {
          const uint32_t gq = q / GR;                  // GR consecutive slabs share a ring step
          const uint32_t slot = gq % NA0;
          char* a_dst = region + slot * (GR * A_SUB) + (q % GR) * A_SUB;
          if constexpr (F16) store_a_half_f16(a_dst, r, h, v);
          else store_a_half(a_dst, r, h, v);
          ++q;
          if (q % GR == 0) {
            fence_proxy_async();
            wg_sync();
            step(a_base + slot * (GR * A_SUB), gq == 0);
          }
        };
        // ---- gather + blend of this half's 16 features of code block fb (registers) ----
        float feat[16];
        float ds = 0.f;
        // where this point's neighbour data lives (geometry modes: optionally indirected, see FieldIn::index)
        const int64_t ps = (valid && MODE != 2) ? field_src(prm.in, p) : p;
        if (valid) ds = prm.in.ds[ps];
        auto gather = [&](int fb) {
#pragma unroll
          for (int i = 0; i < 16; ++i) feat[i] = 0.f;
          if (valid && !tangent) {
#pragma unroll
            for (int k = 0; k < KNN_K; ++k) {
              const int32_t sl = prm.in.slot[k * prm.in.stride + ps];
              const float w = prm.in.w[k * prm.in.stride + ps];
              const float* row = table + (int64_t)sl * Fdim + fb * FEAT + 4 * h;
#pragma unroll
              for (int g4 = 0; g4 < 4; ++g4) {
                const float4 a = __ldg(reinterpret_cast<const float4*>(row + 8 * g4));
                feat[g4 * 4 + 0] = __fadd_rn(feat[g4 * 4 + 0], __fmul_rn(a.x, w));
                feat[g4 * 4 + 1] = __fadd_rn(feat[g4 * 4 + 1], __fmul_rn(a.y, w));
                feat[g4 * 4 + 2] = __fadd_rn(feat[g4 * 4 + 2], __fmul_rn(a.z, w));
                feat[g4 * 4 + 3] = __fadd_rn(feat[g4 * 4 + 3], __fmul_rn(a.w, w));
              }
            }
          }
        };
        gather(0);
        // ---- head block: columns [0, off_feat): PE(ds) [, nabla, PE(view)], zero padded ----
        {
          float head[64];
#pragma unroll
          for (int i = 0; i < 64; ++i) head[i] = 0.f;
          auto st = [&](int col, float v) { head[col] = v; };
          if (valid) {
            if (tangent) {
              store_scalar_pe_tangent(ds, 0, L.Ld, st);
            } else {
              store_scalar_pe(ds, 0, L.Ld, st);
              if (MODE == 2) {
                float dx, dy, dz;
                load_dir(prm.in, p, dx, dy, dz);
                store_vec3_pe(dx, dy, dz, L.off_view, L.Lv, st);
                if (L.use_nabla) {
                  st(L.off_nabla + 0, prm.in.nabla[0 * prm.in.stride + p]);
                  st(L.off_nabla + 1, prm.in.nabla[1 * prm.in.stride + p]);
                  st(L.off_nabla + 2, prm.in.nabla[2 * prm.in.stride + p]);
                }
              }
            }
          }
          for (int s = 0; s < off_feat / SLAB_K; ++s) {
            float v[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = head[s * 16 + 8 * h + i];
            emit(v);
          }
        }
        for (int fb = 0; fb < (TAN_WG ? 0 : n_fb); ++fb) {   // (TAN_WG: the feature and band columns are zero)
          if (fb > 0) gather(fb);
          // ---- raw features: slab s holds groups g = 2s, 2s+1: columns [8h, 8h+8) = feat[2s][0..3], feat[2s+1][0..3] ----
#pragma unroll
          for (int s2 = 0; s2 < 2; ++s2) {
            float v[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = feat[s2 * 8 + i];
            emit(v);
          }
          // ---- bands: slab (b, g): columns [8h, 8h+8) = [sin(2^b f[g][0..3]), cos(2^b f[g][0..3])] ----
          float fr = 1.f;
          for (int b = 0; b < Lf; ++b) {
#pragma unroll
            for (int g4 = 0; g4 < 4; ++g4) {
              float v[8];
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                float sn = 0.f, cs = 0.f;
                if (valid && !tangent) sincosf(feat[g4 * 4 + i] * fr, &sn, &cs);
                v[i] = sn;
                v[4 + i] = cs;
              }
              emit(v);
            }
            fr *= 2.f;
          }
        }
        if constexpr (GR > 1) {   // the first layer is padded with zero slabs (zero weights) to a whole number of steps
          const float zero[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
          // (a tangent warpgroup only completes the step that holds the end of the head block)
          while (TAN_WG ? q % GR != 0 : q < (uint32_t)prm.n_slabs[0]) emit(zero);
        }
        finish_layer();
        if constexpr (TAN_WG) {
          // the remaining first-layer steps would multiply exact zeros: not issued, but every weight slot is still
          // released in ring order, and only after its FULL phase completed (the producer has then seen the slot's
          // previous EMPTY phase complete, so this arrival counts in the phase of this step)
          for (int s = (int)(q / GR); s < prm.n_slabs[0] / GR; ++s) {
            const uint32_t sb = qb % NB;
            mbar_wait(bar(B_FULL + sb), (qb / NB) & 1u);
            if (lane == 0) mbar_arrive(bar(B_EMPTY + sb));
            ++qb;
          }
        }
      }

      // ========================================== layers, epilogues ==========================================
      const int cq = 2 * (lane & 3);              // first of this thread's two adjacent columns in every 8-column group
      const int rr = 16 * warp + (lane >> 2);     // this thread's rows: rr and rr + 8
      // accumulator values per epilogue chunk: column quarters, or eighths for the SPLIT exchange
      constexpr int CH = SPLIT ? 16 : 32;
      static_assert((128 / CH) % 2 == 0, "chunk qq of every layer uses exchange buffer qq % 2");
      for (int l = 0; l < NL; ++l) {
        if (l > 0) {
          const int steps = prm.n_slabs[l] / GR;
          for (int j = 0; j < steps; ++j) step(a_base + j * (GR * A_SUB), j == 0);
          finish_layer();
        }
        const bool last = (l == NL - 1);
        const float* bl = cst + l * MLP_W;
        const float* wo = cst + NL * MLP_W;
        float o[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
#pragma unroll
        for (int qq = 0; qq < 128 / CH; ++qq) {   // MODE 1 exchanges exp(100 z) one chunk at a time
          // column of chunk value i: d[4 n8 + 2 hh + jj] holds column 8 n8 + cq + jj
          auto col = [&](int i) { return 8 * ((CH * qq + i) >> 2) + cq + (i & 1); };
          float v[CH];
#pragma unroll
          for (int i = 0; i < CH; ++i) v[i] = F16 ? d[CH * qq + i] * (1.0f / F16_W_SCALE) : d[CH * qq + i];
          if (MODE == 2) {
#pragma unroll
            for (int i = 0; i < CH; ++i) v[i] = fmaxf(v[i] + bl[col(i)], 0.f);
          } else if (MODE == 0) {
#pragma unroll
            for (int i = 0; i < CH; ++i) {
              const float z = v[i] + bl[col(i)];
              const float y = __log2f(1.0f + fast_exp2(z * K_EXP)) * K_LOG;
              v[i] = z > 0.2f ? z : y;   // 100 z > 20
            }
          } else if constexpr (SPLIT) {
            // warpgroup 0 (value rows) publishes e = exp(100 z) of eighth qq into buffer qq % 2 and keeps
            // softplus = log(1 + e) / 100; warpgroup 1 (tangent rows: same fragment, same point) scales W t by
            // sigma'(z) = e / (1 + e), then frees the buffer for eighth qq + 2
            float* buf = sig + (qq & 1) * SIG_FLOATS;
            if constexpr (!TAN_WG) {
              named_sync(EX_EMPTY + (qq & 1), 256);
#pragma unroll
              for (int i = 0; i < CH; ++i) {
                const float z = v[i] + bl[col(i)];
                const float e = fast_exp2(z * K_EXP);
                buf[i * 128 + t] = e;
                v[i] = z > 0.2f ? z : __log2f(1.0f + e) * K_LOG;
              }
              named_arrive(EX_FULL + (qq & 1), 256);
            } else {
              named_sync(EX_FULL + (qq & 1), 256);
#pragma unroll
              for (int i = 0; i < CH; ++i) {
                const float e = buf[i * 128 + t];
                // 100 z > 20  <=>  e > exp(20)
                v[i] *= e > 485165195.4097903f ? 1.f : __fdividef(e, e + 1.f);
              }
              named_arrive(EX_EMPTY + (qq & 1), 256);
            }
          } else {
            // MODE 1, TF32: value rows (warps 0, 1) publish e = exp(100 z); softplus = log(1 + e) / 100 for the value
            // rows, sigma'(z) * (W t) with sigma' = e / (1 + e) for the tangent rows (warps 2, 3: same fragment, same
            // point)
            if (t < 64) {
#pragma unroll
              for (int i = 0; i < CH; ++i) {
                const float z = v[i] + bl[col(i)];
                const float e = fast_exp2(z * K_EXP);
                sig[i * 64 + t] = e;
                v[i] = z > 0.2f ? z : __log2f(1.0f + e) * K_LOG;
              }
            }
            wg_sync();
            if (t >= 64) {
#pragma unroll
              for (int i = 0; i < CH; ++i) {
                const float e = sig[i * 64 + (t - 64)];
                // 100 z > 20  <=>  e > exp(20)
                v[i] *= e > 485165195.4097903f ? 1.f : __fdividef(e, e + 1.f);
              }
            }
            wg_sync();   // the buffer is rewritten by the next quarter
          }
          if (!last) {
#pragma unroll
            for (int i = 0; i < CH; i += 2) store_a_pair<F16>(region, rr + 8 * ((i >> 1) & 1), col(i), v[i], v[i + 1]);
          } else {
#pragma unroll
            for (int i = 0; i < CH; ++i) {
              const int c = col(i);
              const int hh = (i >> 1) & 1;
              o[hh][0] = fmaf(v[i], wo[c], o[hh][0]);
              if (MODE == 2) {
                o[hh][1] = fmaf(v[i], wo[MLP_W + c], o[hh][1]);
                o[hh][2] = fmaf(v[i], wo[2 * MLP_W + c], o[hh][2]);
              }
            }
          }
        }
        if (!last) {
          fence_proxy_async();
          wg_sync();   // the next layer's A operand is complete
        } else {
          // the four threads of a quad hold the partial dot products of the same two rows
#pragma unroll
          for (int hh = 0; hh < 2; ++hh)
#pragma unroll
            for (int k = 0; k < 3; ++k) {
              o[hh][k] += __shfl_xor_sync(0xffffffffu, o[hh][k], 1);
              o[hh][k] += __shfl_xor_sync(0xffffffffu, o[hh][k], 2);
            }
          if ((lane & 3) == 0) {
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              const int row = rr + 8 * hh;
              const int64_t p = pbase + (HALF_ROWS ? (row & 31) : row);
              if (p >= prm.P) continue;
              if (MODE == 2) {
                prm.out0[0 * prm.in.stride + p] = sigmoid_acc(o[hh][0] + __ldg(prm.b_out + 0));
                prm.out0[1 * prm.in.stride + p] = sigmoid_acc(o[hh][1] + __ldg(prm.b_out + 1));
                prm.out0[2 * prm.in.stride + p] = sigmoid_acc(o[hh][2] + __ldg(prm.b_out + 2));
              } else if (MODE == 0 || (SPLIT ? !TAN_WG : row < 32)) {
                prm.out0[p] = o[hh][0] + __ldg(prm.b_out);
              } else if (prm.out1) {
                const int64_t ps = field_src(prm.in, p);
                prm.out1[0 * prm.in.stride + p] = o[hh][0] * prm.in.grad[0 * prm.in.stride + ps];
                prm.out1[1 * prm.in.stride + p] = o[hh][0] * prm.in.grad[1 * prm.in.stride + ps];
                prm.out1[2 * prm.in.stride + p] = o[hh][0] * prm.in.grad[2 * prm.in.stride + ps];
              }
            }
          }
        }
      }
    };
    if (tan_wg) tile_work(std::true_type{});
    else tile_work(std::false_type{});
  }
  // the tangent warpgroup's last two EMPTY arrivals have no matching wait yet: take them, so that no named barrier is
  // left part-way through a phase when the CTA exits
  if (SPLIT && wg == 0) {
    named_sync(EX_EMPTY + 0, 256);
    named_sync(EX_EMPTY + 1, 256);
  }
}

// ------------------------------------------------------------------------------------------------------------
// packing: W^T [K][256] fp32 (already weight-norm folded, OUR column order) -> per-slab hi/lo tf32 images
// ------------------------------------------------------------------------------------------------------------
__global__ void pack_tc_kernel(const float* __restrict__ wt /*[K_src][256]*/, const int32_t* __restrict__ kmap /*[K]*/,
                               int K, float* __restrict__ dst) {
  // one thread per (k, n)
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= (int64_t)K * MLP_W) return;
  const int n = (int)(t % MLP_W);
  const int k = (int)(t / MLP_W);
  const int ksrc = kmap[k];
  const float x = ksrc >= 0 ? wt[(int64_t)ksrc * MLP_W + n] : 0.f;
  const float hi = tc::tf32_rna(x);
  const float lo = tc::tf32_rna(x - hi);
  const int slab = k / tc::SLAB_K, kk = k % tc::SLAB_K;
  float* base = dst + (int64_t)slab * (tc::B_SLOT32 / 4);
  const int off = (kk / 4) * (MLP_W * 4) + n * 4 + (kk % 4);
  base[off] = hi;
  base[tc::B_HALF32 / 4 + off] = lo;
}

// fp16x3 variant: per slab [hi | lo] x [k/8][256][k%8] halves of 2^8 W (hi = fp16(x), lo = fp16(x - hi))
__global__ void pack_tc16_kernel(const float* __restrict__ wt /*[K_src][256]*/, const int32_t* __restrict__ kmap /*[K]*/,
                                 int K, float* __restrict__ dst) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= (int64_t)K * MLP_W) return;
  const int n = (int)(t % MLP_W);
  const int k = (int)(t / MLP_W);
  const int ksrc = kmap[k];
  const float x = (ksrc >= 0 ? wt[(int64_t)ksrc * MLP_W + n] : 0.f) * tc::F16_W_SCALE;
  const __half hi = __float2half_rn(x);
  const __half lo = __float2half_rn(x - __half2float(hi));
  const int slab = k / tc::SLAB_K, kk = k % tc::SLAB_K;
  __half* base = reinterpret_cast<__half*>(dst + (int64_t)slab * (tc::B_SLOT16 / 4));
  const int off = (kk / 8) * (MLP_W * 8) + n * 8 + (kk % 8);
  base[off] = hi;
  base[tc::B_HALF16 / 2 + off] = lo;
}

// TC first-layer column k -> FFMA first-layer column (both in "our" orders; see FieldLayout).
// Builder half h (0/1) owns features F(g, h, i) = 8 g + 4 h + i (g < 4, i < 4) and columns [8h, 8h+8) of each slab:
//   raw slab s (2):       col 8h + 4u + i  = feature F(2s + u, h, i)            (u < 2)
//   band slab (b, g):     col 8h + i       = sin(2^b F(g, h, i)),  col 8h + 4 + i = cos(2^b F(g, h, i))
static std::vector<int32_t> tc_first_layer_map(const FieldLayout& L, bool color) {
  const int off = color ? L.off_ft : L.off_fg;
  const int Lf = color ? L.Lft : L.Lfg;
  std::vector<int32_t> m;
  for (int k = 0; k < off; ++k) m.push_back(k);                 // head block: identical order
  const int Fdim = color ? L.Fc : L.Fg;
  auto F = [](int g, int h, int i) { return 8 * g + 4 * h + i; };
  for (int fb = 0; fb < Fdim / FEAT; ++fb) {   // one run of (2 raw + 4 Lf band) slabs per 32-column code block
    const int f0 = fb * FEAT;
    for (int s = 0; s < 2; ++s)
      for (int h = 0; h < 2; ++h)
        for (int u = 0; u < 2; ++u)
          for (int i = 0; i < 4; ++i) m.push_back(off + f0 + F(2 * s + u, h, i));
    for (int b = 0; b < Lf; ++b)
      for (int g = 0; g < 4; ++g)
        for (int h = 0; h < 2; ++h) {
          for (int i = 0; i < 4; ++i) m.push_back(off + (1 + 2 * b) * Fdim + f0 + F(g, h, i));  // sin block
          for (int i = 0; i < 4; ++i) m.push_back(off + (2 + 2 * b) * Fdim + f0 + F(g, h, i));  // cos block
        }
  }
  return m;
}

static int pack_one(const MlpFfma& src, const FieldLayout& L, bool color, bool f16, MlpTc* dst, cudaStream_t stream) {
  int64_t total = 0;
  dst->total_slabs = 0;
  const int slot_floats = (f16 ? tc::B_SLOT16 : tc::B_SLOT32) / 4;
  for (int l = 0; l < src.n_layers; ++l) {
    dst->n_slabs[l] = src.K[l] / tc::SLAB_K;
    if (f16) dst->n_slabs[l] = (int)align_up((int64_t)dst->n_slabs[l], (int64_t)tc::GR16);   // whole ring steps (zero slabs)
    dst->slab_off[l] = total;
    total += (int64_t)dst->n_slabs[l] * slot_floats;
    dst->total_slabs += dst->n_slabs[l];
  }
  NMB_CUDA_OK(dst->w.alloc(total));
  NMB_CUDA_OK(cudaMemsetAsync(dst->w.p, 0, (size_t)total * sizeof(float), stream));   // padding slabs stay zero
  for (int l = 0; l < src.n_layers; ++l) {
    std::vector<int32_t> kmap;
    if (l == 0) {
      kmap = tc_first_layer_map(L, color);
      NMB_CHECK((int)kmap.size() == src.K[0], "first-layer column map size mismatch");
    } else {
      kmap.resize(MLP_W);
      for (int i = 0; i < MLP_W; ++i) kmap[i] = i;
    }
    DevBuf<int32_t>& km = dst->kmap[l];   // kept in the field; pageable upload = staged before the call returns
    NMB_CUDA_OK(km.alloc((int64_t)kmap.size()));
    NMB_CUDA_OK(cudaMemcpyAsync(km.p, kmap.data(), kmap.size() * 4, cudaMemcpyHostToDevice, stream));
    const int64_t n = (int64_t)src.K[l] * MLP_W;
    if (f16) {
      pack_tc16_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, stream>>>(src.w.p + src.w_off[l], km.p, src.K[l],
                                                                      dst->w.p + dst->slab_off[l]);
    } else {
      pack_tc_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, stream>>>(src.w.p + src.w_off[l], km.p, src.K[l],
                                                                    dst->w.p + dst->slab_off[l]);
    }
    NMB_LAUNCH_OK();
  }
  return 0;
}

int pack_mlp_tc(const nmb_field_desc*, const FieldLayout& lay, nmb_field* f, cudaStream_t stream) {
  const bool f16 = f->engine == 2;   // geo_t / col_t hold the images of the engine the field was created for
  int rc = pack_one(f->geo_f, lay, false, f16, &f->geo_t, stream);
  if (rc) return rc;
  return pack_one(f->col_f, lay, true, f16, &f->col_t, stream);
}

template <int MODE, bool F16>
static int launch_tc(const nmb_field* f, const MlpFfma& fm, const MlpTc& tm, const FieldIn& in, int64_t P, float* out0,
                     float* out1, cudaStream_t stream) {
  if (P <= 0) return 0;
  tc::Params prm;
  prm.lay = f->lay;
  prm.in = in;
  prm.tab = FieldTables{f->fg.p, in.color_table ? in.color_table : f->fc.p};
  prm.w = tm.w.p;
  prm.bias = fm.b.p;
  prm.w_out = fm.w_out.p;
  prm.b_out = fm.b_out.p;
  for (int i = 0; i < MAX_LAYERS; ++i) {
    prm.slab_off[i] = tm.slab_off[i];
    prm.n_slabs[i] = i < fm.n_layers ? tm.n_slabs[i] : 0;
  }
  prm.n_layers = fm.n_layers;
  prm.P = P;
  prm.out0 = out0;
  prm.out1 = out1;
  using C = tc::Cfg<F16>;
  const size_t smem = tc::SmemLayoutT<F16, MODE == 1>::total;
  static DeviceOnce attr_once;
  NMB_CUDA_OK(attr_once.run([&] {
    return cudaFuncSetAttribute(mlp_tc_kernel<MODE, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  }));
  const int64_t tiles = ceil_div(P, (int64_t)tc::tile_points<MODE, F16>());
  const int64_t grid = tiles < (int64_t)sm_count() ? tiles : (int64_t)sm_count();
  ProfScope prof(MODE == 2 ? PROF_COLOR : (MODE == 1 ? PROF_GEO_JVP : PROF_GEO), P, stream);
  mlp_tc_kernel<MODE, F16><<<(unsigned)grid, C::THREADS, smem, stream>>>(prm);
  NMB_LAUNCH_OK();
  return 0;
}

int launch_geo_tc(const nmb_field* f, const FieldIn& in, int64_t P, float* sdf, float* nabla, cudaStream_t stream) {
  if (f->engine == 2) {
    if (nabla) return launch_tc<1, true>(f, f->geo_f, f->geo_t, in, P, sdf, nabla, stream);
    return launch_tc<0, true>(f, f->geo_f, f->geo_t, in, P, sdf, nullptr, stream);
  }
  if (nabla) return launch_tc<1, false>(f, f->geo_f, f->geo_t, in, P, sdf, nabla, stream);
  return launch_tc<0, false>(f, f->geo_f, f->geo_t, in, P, sdf, nullptr, stream);
}

int launch_color_tc(const nmb_field* f, const FieldIn& in, int64_t P, float* rgb, cudaStream_t stream) {
  if (f->engine == 2) return launch_tc<2, true>(f, f->col_f, f->col_t, in, P, rgb, nullptr, stream);
  return launch_tc<2, false>(f, f->col_f, f->col_t, in, P, rgb, nullptr, stream);
}

}  // namespace nmb
