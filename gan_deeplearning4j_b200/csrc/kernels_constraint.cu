// kernels_constraint.cu -- DL4J's weight constraints (LayerConstraint: MaxNormConstraint, MinMaxNormConstraint, UnitNormConstraint,
// NonNegativeConstraint), applied to the fp32 master parameters after the updater, with the bf16 weight operands (straight and packed
// pixel-shuffle copies) rewritten through upd_shadow.  Semantics: include/b200gan.h (b2g_constraint); the job plan: kernels.h (ConJob) and
// engine.cu (net_build_constraints); restatement: oracle/dl4j_oracle.py; exact emulation of this order: tests/ew_ref.py.
//
// Summation order of a group's squared norm, in double over (double)w * (double)w (exact), fixed by the shape and not by the grid:
//   K2 == 1 (the innermost axis reduced): the group's j's are cut into chunks of CON_CHUNK; in a chunk, thread t of 256 sums j = chunk_base + t + 256 q
//     for q ascending, the 256 sums are folded by block_sum (each warp's xor butterfly, then the 8 warp sums in warp order onto 0.0); the
//     group's sum is 0.0 + the chunk sums in chunk order (the one-pass path has one chunk: its block sum).
//   K2 > 1 (the innermost axis kept: strided groups): chunks of CON_SCHUNK j's; in a chunk, warp w sums the rows j = chunk_base + w + 8 i for i ascending (lane l is
//     group k2 = 32 tile + l), the 8 warp sums are added in warp order onto 0.0; the group's sum is 0.0 + the chunk sums in chunk order.
// The multiplier is computed in double from norm = sqrt(sum) and rounded to fp32 once; each element becomes the fp32 product w * m.
//
// A translation unit of its own, like kernels_gradnorm.cu: the updater kernel keeps the code nvcc generates for it without these kernels.
#include <stdint.h>
#include "kernels.h"
#include "common.cuh"

namespace b2g {

static const double CON_EPS = 1e-6;      // BaseConstraint.DEFAULT_EPSILON

// Index arithmetic in 32 bits: a constrained tensor has fewer than 2^31 elements (one layer's parameters).
__device__ __forceinline__ int64_t con_off(const ConJob& jb, int g, int j) {        // element j of group g -> its index in the tensor
  if (jb.K1 == 1 && jb.K2 == 1) return (int64_t)g * jb.R + j;                       // [K0][R]: the group is one contiguous run
  const int k2 = g % jb.K2; g /= jb.K2;
  const int k1 = g % jb.K1, k0 = g / jb.K1, r1 = j % jb.R1, r0 = j / jb.R1;
  return ((((int64_t)k0 * jb.R0 + r0) * jb.K1 + k1) * jb.R1 + r1) * jb.K2 + k2;
}
__device__ __forceinline__ int con_group(const ConJob& jb, int64_t e64) {           // tensor index -> its group
  int e = (int)e64;
  if (jb.K1 == 1 && jb.K2 == 1) return e / jb.R;
  const int k2 = e % jb.K2; e /= jb.K2 * jb.R1;
  const int k1 = e % jb.K1; e /= jb.K1;
  return ((e / jb.R0) * jb.K1 + k1) * jb.K2 + k2;
}
// b2g_constraint_kind 0-2 on the group's sum of squares
__device__ __forceinline__ float con_mult(const ConJob& jb, double s) {
  const double norm = sqrt(s);
  double m;
  if (jb.kind == 0) m = fmin(norm, jb.max_norm) / (norm + CON_EPS);
  else if (jb.kind == 1)      // rounded products and sum, no fused multiply-add: the multiplier is the formula's, operation by operation
    m = __dadd_rn(__dmul_rn(jb.rate, fmin(fmax(norm, jb.min_norm), jb.max_norm)), __dmul_rn(1.0 - jb.rate, norm)) / (norm + CON_EPS);
  else m = norm == 0.0 ? 1.0 : 1.0 / norm;      // UnitNorm: an all-zero group is left as it is
  return (float)m;
}
__device__ __forceinline__ void con_store(const ConJob& jb, float* params, __nv_bfloat16* shadow, int64_t e, float w) {
  params[jb.sg.off + e] = w;
  if (shadow && jb.sg.off_bf >= 0) upd_shadow(jb.sg, shadow, jb.sg.off + e, __float2bfloat16_rn(w));
}
// the job whose blocks [begin, begin + count) hold block b (a round has few jobs)
template <bool SECOND>
__device__ __forceinline__ int con_find(const ConJob* jobs, int j0, int j1, int b) {
  int j = j0;
  while (j + 1 < j1 && (SECOND ? jobs[j + 1].blk2_begin : jobs[j + 1].blk_begin) <= b) ++j;
  return j;
}

__global__ void __launch_bounds__(256) constraint_onepass_kernel(float* __restrict__ params, __nv_bfloat16* __restrict__ shadow, const ConJob* __restrict__ jobs,
                                                                 int j0, int j1) {
  pdl_enter();
  __shared__ double red[8];
  __shared__ float m_s;
  const ConJob jb = jobs[con_find<false>(jobs, j0, j1, blockIdx.x)];      // a copy: a reference spills
  const int b = blockIdx.x - jb.blk_begin;
  if (jb.path == CON_ELEMWISE) {         // NonNegative: w < 0 -> +0; -0.0 and NaN stay (replaceWhere(.., 0, lessThan(0)))
    const int64_t base = (int64_t)b * CON_CHUNK, end = min(base + (int64_t)CON_CHUNK, jb.sg.len);
    for (int64_t e = base + threadIdx.x; e < end; e += blockDim.x)
      if (params[jb.sg.off + e] < 0.f) con_store(jb, params, shadow, e, 0.f);
    return;
  }
  // one group, read once: 16 values per thread
  float v[CON_CHUNK / 256];
  double acc = 0.0;
#pragma unroll
  for (int q = 0; q < CON_CHUNK / 256; ++q) {
    const int j = threadIdx.x + 256 * q;
    v[q] = j < jb.R ? params[jb.sg.off + con_off(jb, b, j)] : 0.f;
    acc += (double)v[q] * (double)v[q];
  }
  const double tot = block_sum(acc, red);
  if (threadIdx.x == 0) m_s = con_mult(jb, tot);
  __syncthreads();
  const float m = m_s;
#pragma unroll
  for (int q = 0; q < CON_CHUNK / 256; ++q) {
    const int j = threadIdx.x + 256 * q;
    if (j < jb.R) con_store(jb, params, shadow, con_off(jb, b, j), v[q] * m);
  }
}

__global__ void __launch_bounds__(256) constraint_norm_kernel(const float* __restrict__ params, const ConJob* __restrict__ jobs, int j0, int j1,
                                                              double* partial, unsigned* ticket, float* __restrict__ mult) {
  pdl_enter();
  __shared__ double red[8][33];
  __shared__ int last;
  const ConJob& jb = jobs[con_find<false>(jobs, j0, j1, blockIdx.x)];
  const int b = blockIdx.x - jb.blk_begin;
  const float* p = params + jb.sg.off;
  if (jb.K2 == 1) {                       // block (group, chunk)
    const int g = b / jb.chunks, c = b % jb.chunks;
    double acc = 0.0;
    for (int j = c * CON_CHUNK + threadIdx.x; j < min(jb.R, (c + 1) * CON_CHUNK); j += 256) { const double w = p[con_off(jb, g, j)]; acc += w * w; }
    const double tot = block_sum(acc, &red[0][0]);
    if (threadIdx.x == 0) partial[jb.part_begin + (int64_t)g * jb.chunks + c] = tot;
  } else {                                // strided groups: block (k0 k1, tile of 32 k2, chunk); lane = k2 in the tile, warp = row phase
    const int tiles = (jb.K2 + 31) / 32, c = b % jb.chunks, tile = (b / jb.chunks) % tiles, gk = b / (jb.chunks * tiles);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, k2 = tile * 32 + lane;
    double acc = 0.0;
    if (k2 < jb.K2)
      for (int j = c * CON_SCHUNK + warp; j < min(jb.R, (c + 1) * CON_SCHUNK); j += 8) { const double w = p[con_off(jb, gk * jb.K2 + k2, j)]; acc += w * w; }
    red[warp][lane] = acc;
    __syncthreads();
    if (warp == 0 && k2 < jb.K2) {
      double s = 0.0;
      for (int w = 0; w < 8; ++w) s += red[w][lane];
      partial[jb.part_begin + (int64_t)(gk * jb.K2 + k2) * jb.chunks + c] = s;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) { __threadfence(); last = atomicAdd(ticket, 1u) == gridDim.x - 1; }
  __syncthreads();
  if (!last) return;
  // the last block: every partial is visible (each writer fenced before taking its ticket); one thread per group adds its chunks in order
  __threadfence();
  for (int k = j0; k < j1; ++k) {
    const ConJob& jk = jobs[k];
    for (int g = threadIdx.x; g < jk.groups; g += blockDim.x) {
      double s = 0.0;
      for (int c = 0; c < jk.chunks; ++c) s += __ldcg(partial + jk.part_begin + (int64_t)g * jk.chunks + c);
      mult[jk.mult_begin + g] = con_mult(jk, s);
    }
  }
  if (threadIdx.x == 0) { *ticket = 0u; __threadfence(); }
}

__global__ void __launch_bounds__(256) constraint_scale_kernel(float* __restrict__ params, __nv_bfloat16* __restrict__ shadow, const ConJob* __restrict__ jobs,
                                                               int j0, int j1, const float* __restrict__ mult) {
  pdl_enter();
  const ConJob& jb = jobs[con_find<true>(jobs, j0, j1, blockIdx.x)];
  const int64_t base = (int64_t)(blockIdx.x - jb.blk2_begin) * CON_CHUNK, end = min(base + (int64_t)CON_CHUNK, jb.sg.len);
  for (int64_t e = base + threadIdx.x; e < end; e += blockDim.x)
    con_store(jb, params, shadow, e, params[jb.sg.off + e] * mult[jb.mult_begin + con_group(jb, e)]);
}

void k_constraint_onepass(float* params, __nv_bfloat16* shadow, const ConJob* jobs, int j0, int j1, int blocks, cudaStream_t s) {
  if (!blocks) return;
  launch_pdl(constraint_onepass_kernel, dim3(blocks), dim3(256), (size_t)0, s, params, shadow, jobs, j0, j1); LAUNCHED();
}
void k_constraint_twopass(float* params, __nv_bfloat16* shadow, const ConJob* jobs, int j0, int j1, int norm_blocks, int scale_blocks, double* partial,
                          unsigned* ticket, float* mult, cudaStream_t s) {
  if (!norm_blocks) return;
  launch_pdl(constraint_norm_kernel, dim3(norm_blocks), dim3(256), (size_t)0, s, (const float*)params, jobs, j0, j1, partial, ticket, mult); LAUNCHED();
  launch_pdl(constraint_scale_kernel, dim3(scale_blocks), dim3(256), (size_t)0, s, params, shadow, jobs, j0, j1, (const float*)mult); LAUNCHED();
}

}  // namespace b2g
