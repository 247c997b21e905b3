// Exact K-nearest-neighbour walk over the octree of csrc/grid.cu (device code shared by grid.cu and shell.cu).
#pragma once
#include <math_constants.h>

#include "grid.cuh"

namespace nmb {

// ------------------------------------------------------------------------------------------------------------
// traversal
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float sq_dist_rn(float qx, float qy, float qz, float px, float py, float pz) {
  // (dx*dx + dy*dy) + dz*dz with every operation individually rounded: no FMA contraction
  const float dx = __fsub_rn(qx, px), dy = __fsub_rn(qy, py), dz = __fsub_rn(qz, pz);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

__device__ __forceinline__ float box_dist_rn(float qx, float qy, float qz, const float4& lo, const float4& hi) {
  // lower bound of sq_dist_rn over every point inside the box (rounding is monotone)
  const float dx = fmaxf(fmaxf(__fsub_rn(lo.x, qx), __fsub_rn(qx, hi.x)), 0.f);
  const float dy = fmaxf(fmaxf(__fsub_rn(lo.y, qy), __fsub_rn(qy, hi.y)), 0.f);
  const float dz = fmaxf(fmaxf(__fsub_rn(lo.z, qz), __fsub_rn(qz, hi.z)), 0.f);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// Lower bound of sq_dist_rn(q, p) over the points p of a node, from its two bounding volumes:
//  * the tight axis-aligned box (exact-safe: rounding is monotone), and
//  * a "disc": all points satisfy |p - c| <= r and |u . (p - c)| <= t, hence with a = u . (q - c) and
//    b = sqrt(|q - c|^2 - a^2):  dist^2 >= max(|a| - t, 0)^2 + max(b - r, 0)^2.
// A mesh is locally a thin sheet (t << r), so for a query FAR from the surface the disc bound is within ~t of the true
// distance while the box bound is short by up to the box size; the number of nodes that survive pruning drops from
// ~2*pi*D/size per level to a handful.  The disc value is deflated a little so that fp32 rounding can never make it
// exceed a true distance (r and t are inflated at build time as well).
__device__ __forceinline__ float disc_bound(float qx, float qy, float qz, const float4& cr, const float4& ut) {
  const float dx = qx - cr.x, dy = qy - cr.y, dz = qz - cr.z;
  const float a = ut.x * dx + ut.y * dy + ut.z * dz;
  const float dd = dx * dx + dy * dy + dz * dz;
  const float b = sqrtf(fmaxf(dd - a * a, 0.f));
  const float h = fmaxf(fabsf(a) - ut.w, 0.f);
  const float l = fmaxf(b - cr.w, 0.f);
  return (h * h + l * l) * 0.99998f - 1e-12f;
}

__device__ __forceinline__ float node_bound(float qx, float qy, float qz, const float4& lo, const float4& hi,
                                            const float4& cr, const float4& ut) {
  return fmaxf(box_dist_rn(qx, qy, qz, lo, hi), disc_bound(qx, qy, qz, cr, ut));
}

// Candidates are ranked by the total order (squared distance, slot index): the K smallest under it are unique, so
// the result does not depend on the order in which the walk meets the points (cold walk, warm-started walk and
// brute force agree bit for bit even when distances tie exactly).
__device__ __forceinline__ bool cand_less(float da, int32_t ia, float db, int32_t ib) {
  return da < db || (da == db && ia < ib);
}

// Insert (nd, ni) into the ascending list d[0..K-1] (precondition: (nd, ni) ranks before slot K-1); branch-free.
template <int K>
__device__ __forceinline__ void topk_insert(float (&d)[K], int32_t (&ix)[K], float nd, int32_t ni) {
#pragma unroll
  for (int k = K - 1; k > 0; --k) {
    const bool from_above = cand_less(nd, ni, d[k - 1], ix[k - 1]);  // old slot k-1 (still untouched)
    const bool here = cand_less(nd, ni, d[k], ix[k]);                // old slot k
    const float dk = from_above ? d[k - 1] : (here ? nd : d[k]);
    const int32_t ik = from_above ? ix[k - 1] : (here ? ni : ix[k]);
    d[k] = dk;
    ix[k] = ik;
  }
  if (cand_less(nd, ni, d[0], ix[0])) {
    d[0] = nd;
    ix[0] = ni;
  }
}

#define NMB_CSWAP(a, b)                                   \
  {                                                       \
    const bool s_ = cand_less(cd[a], cn[a], cd[b], cn[b]); \
    const float t_ = s_ ? cd[a] : cd[b];                  \
    const int32_t u_ = s_ ? cn[a] : cn[b];                \
    cd[a] = s_ ? cd[b] : cd[a];                           \
    cn[a] = s_ ? cn[b] : cn[a];                           \
    cd[b] = t_;                                           \
    cn[b] = u_;                                           \
  }
// 19-comparator sorting network on (cd[8], cn[8]), DESCENDING (largest first)
#define NMB_SORT8_DESC()                                                      \
  NMB_CSWAP(0, 1) NMB_CSWAP(2, 3) NMB_CSWAP(4, 5) NMB_CSWAP(6, 7)              \
  NMB_CSWAP(0, 2) NMB_CSWAP(1, 3) NMB_CSWAP(4, 6) NMB_CSWAP(5, 7)              \
  NMB_CSWAP(1, 2) NMB_CSWAP(5, 6) NMB_CSWAP(0, 4) NMB_CSWAP(3, 7)              \
  NMB_CSWAP(1, 5) NMB_CSWAP(2, 6)                                              \
  NMB_CSWAP(1, 4) NMB_CSWAP(3, 6)                                              \
  NMB_CSWAP(2, 4) NMB_CSWAP(3, 5)                                              \
  NMB_CSWAP(3, 4)

// Depth-first, nearest-child-first walk.  On return d[]/ix[] hold the K nearest points (ascending squared
// distance; ix = slot in the Morton-sorted point array).
//   WARM = false: d[] / ix[] are initialised here (empty list).
//   WARM = true : the caller pre-loaded d[] / ix[] with K DISTINCT real points and their distances to q, sorted
//                 ascending (e.g. the neighbours of the previous sample on the same ray).  The walk then starts with
//                 a tight pruning bound; a point already in the list is never inserted twice.
template <int K, bool WARM>
__device__ __forceinline__ void knn_walk(const float4* __restrict__ nodes, const float4* __restrict__ pts, float qx,
                                         float qy, float qz, float (&d)[K], int32_t (&ix)[K]) {
  if (!WARM) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      d[k] = CUDART_INF_F;
      ix[k] = 0x7fffffff;
    }
  }
  int32_t sn[STACK_MAX];
  float sd[STACK_MAX];
  int sp = 1;
  sn[0] = 0;
  sd[0] = 0.f;
  // "while-while" traversal: every lane first descends through INTERNAL nodes until it holds a leaf, then all lanes
  // of the warp scan their leaves together - the two code paths are not interleaved lane by lane, which keeps far
  // more lanes active per issued instruction than a single pop-and-branch loop.
  while (true) {
    int32_t leaf_b = 0, leaf_e = 0;
    while (sp > 0) {
      --sp;
      const int32_t n = sn[sp];
      if (sd[sp] > d[K - 1]) continue;   // '>' (not '>='): an equidistant point with a smaller index may still enter
      const float4 a = __ldg(&nodes[NODE_F4 * n]);
      const float4 b = __ldg(&nodes[NODE_F4 * n + 1]);
      const int32_t link = __float_as_int(a.w);
      const int32_t cnt = __float_as_int(b.w);
      if (cnt < 0) {
        leaf_b = link;
        leaf_e = link - cnt;
        break;
      }
      float cd[8];
      int32_t cn[8];
      const float worst = d[K - 1];
      int m = 0, only = 0;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        cd[c] = CUDART_INF_F;
        cn[c] = link + c;
        if (c < cnt) {
          const float4* nc = nodes + NODE_F4 * (link + c);
          // box first (cheap, exact-safe); the disc bound is only evaluated for children the box cannot reject
          float bd = box_dist_rn(qx, qy, qz, __ldg(nc), __ldg(nc + 1));
          if (bd <= worst) {
            bd = fmaxf(bd, disc_bound(qx, qy, qz, __ldg(nc + 2), __ldg(nc + 3)));
            if (bd <= worst) {
              cd[c] = bd;
              ++m;
              only = c;
            }
          }
        }
      }
      if (sp + m > STACK_MAX) {
        // cannot happen for depth <= 10 (at most 7 net pushes per level); never drop a subtree silently: the launch
        // fails with a trap (reported by the next CUDA call) instead of returning inexact neighbours
        __trap();
      }
      if (m == 1) {
        sn[sp] = link + only;
        sd[sp] = cd[only];
        ++sp;
      } else if (m > 1) {
        // only the nearest survivor goes on top of the stack, the others keep child order: any push order is exact
        // (the pop test prunes), only the pruning efficiency depends on it
        float best = cd[0];
        int bi = 0;
#pragma unroll
        for (int c = 1; c < 8; ++c) {
          const bool lt = cd[c] < best;
          best = lt ? cd[c] : best;
          bi = lt ? c : bi;
        }
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          if (cd[c] < CUDART_INF_F && c != bi) {
            sn[sp] = cn[c];
            sd[sp] = cd[c];
            ++sp;
          }
        }
        sn[sp] = link + bi;
        sd[sp] = best;
        ++sp;
      }
    }
    if (leaf_e == leaf_b) break;   // stack exhausted without another leaf
    for (int32_t i = leaf_b; i < leaf_e; ++i) {
      const float4 p = __ldg(&pts[i]);
      const float dd = sq_dist_rn(qx, qy, qz, p.x, p.y, p.z);
      if (cand_less(dd, i, d[K - 1], ix[K - 1])) {
        bool dup = false;
        if (WARM) {
#pragma unroll
          for (int k = 0; k < K; ++k) dup |= (ix[k] == i);
        }
        if (!dup) topk_insert<K>(d, ix, dd, i);
      }
    }
  }
}

// re-rank K known points against a new query: distances recomputed, then sorted ascending (same network, reversed)
template <int K>
__device__ __forceinline__ void warm_rerank(const float4* __restrict__ pts, float qx, float qy, float qz,
                                            float (&d)[K], int32_t (&ix)[K]) {
  static_assert(K == 8, "sorting network is for 8 entries");
  float cd[8];
  int32_t cn[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float4 p = __ldg(&pts[ix[k]]);
    cd[k] = sq_dist_rn(qx, qy, qz, p.x, p.y, p.z);
    cn[k] = ix[k];
  }
  NMB_SORT8_DESC()
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    d[k] = cd[7 - k];
    ix[k] = cn[7 - k];
  }
}
#undef NMB_CSWAP

}  // namespace nmb
