// kernels_ew.cu -- the HBM-bound kernels of the GAN step: layout conversion, BatchNorm statistics /
// apply / backward, activations, max-pool, upsampling, binary cross-entropy, column sums, and the
// one-pass updater (divide-by-minibatch -> clip -> RmsProp/Adam -> +l2*W + l1*sign(W) -> theta -= g).
//
// Semantics follow DL4J 1.0.0-beta3 as restated in oracle/dl4j_oracle.py (SURVEY.md section 8a rows
// a3-a6, a8, a9); the reference call sites are J:123-125,132-134,141-144,159-163,201-202 where
// J = Java/src/main/java/org/deeplearning4j/dl4jGANComputerVision.java of the reference repository.
//
// All of these are bandwidth-bound: threads are mapped so that a warp touches consecutive channels
// (NHWC innermost), reductions are fixed-order two-stage (deterministic), nothing allocates.
#include <stdlib.h>
#include <algorithm>
#include "kernels.h"
#include "common.cuh"

namespace b2g {

uint64_t g_launch_count = 0;
const char* g_ew_last_kernel = "";

// ---------------------------------------------------------------- layout -----------------------------
template <typename T>
__global__ void nchw_f32_to_nhwc_kernel(const float* __restrict__ src, T* __restrict__ dst, int N, int C, int HW) { pdl_enter();
  // one thread per destination element (coalesced writes; reads strided by HW, served by L2)
  size_t total = (size_t)N * C * HW;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int c = i % C; size_t t = i / C; int p = t % HW; size_t n = t / HW;
    stf(dst, i, src[(n * C + c) * HW + p]);
  }
}
template <typename T>
__global__ void nhwc_to_nchw_f32_kernel(const T* __restrict__ src, float* __restrict__ dst, int N, int C, int HW) { pdl_enter();
  size_t total = (size_t)N * C * HW;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int p = i % HW; size_t t = i / HW; int c = t % C; size_t n = t / C;
    dst[i] = ldf(src, (n * HW + p) * C + c);
  }
}
template <typename T>
__global__ void permute_kernel(const T* __restrict__ src, T* __restrict__ dst, int N, int C, int HW, int to_nhwc) { pdl_enter();
  size_t total = (size_t)N * C * HW;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    if (to_nhwc) { int c = i % C; size_t t = i / C; int p = t % HW; size_t n = t / HW; dst[i] = src[(n * C + c) * HW + p]; }
    else         { int p = i % HW; size_t t = i / HW; int c = t % C; size_t n = t / C; dst[i] = src[(n * HW + p) * C + c]; }
  }
}
// activation resolved at compile time for the common cases (the per-element switch costs more than the arithmetic in these kernels)
#define DISPATCH_ACT(act, ACTC, ...)                                                            \
  switch (act) {                                                                                \
    case ACT_IDENTITY: { constexpr int ACTC = ACT_IDENTITY; __VA_ARGS__; } break;               \
    case ACT_RELU: { constexpr int ACTC = ACT_RELU; __VA_ARGS__; } break;                       \
    case ACT_LRELU: { constexpr int ACTC = ACT_LRELU; __VA_ARGS__; } break;                     \
    default: { constexpr int ACTC = -1; __VA_ARGS__; } break;                                   \
  }
int device_sm_count() {
  static int sms[64] = {}; int d = 0; cudaGetDevice(&d); if (d < 0 || d >= 64) d = 0;
  if (!sms[d]) { int v = 0; cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, d); sms[d] = v > 0 ? v : 1; }
  return sms[d];
}
static inline int vec4_blocks(size_t n_vec) { const size_t cap = (size_t)device_sm_count() * 4; size_t b = (n_vec + 1023) / 1024; if (b > cap) b = cap; if (b < 1) b = 1; return (int)b; }
static inline int ew_blocks(size_t n, int per = 256) { const size_t cap = (size_t)device_sm_count() * 16; size_t b = (n + per - 1) / per; if (b > cap) b = cap; if (b < 1) b = 1; return (int)b; }

void k_nchw_f32_to_nhwc(int prec, const float* src, void* dst, int N, int C, int HW, cudaStream_t s) {
  size_t n = (size_t)N * C * HW; if (!n) return;
  DISPATCH_PREC(prec, T, (launch_pdl(nchw_f32_to_nhwc_kernel<T>, dim3(ew_blocks(n)), dim3(256), (size_t)(0), s, src, (T*)dst, N, C, HW))); LAUNCHED();
  g_ew_last_kernel = "nchw_f32_to_nhwc_kernel";
}
void k_nhwc_to_nchw_f32(int prec, const void* src, float* dst, int N, int C, int HW, cudaStream_t s) {
  size_t n = (size_t)N * C * HW; if (!n) return;
  DISPATCH_PREC(prec, T, (launch_pdl(nhwc_to_nchw_f32_kernel<T>, dim3(ew_blocks(n)), dim3(256), (size_t)(0), s, (const T*)src, dst, N, C, HW))); LAUNCHED();
  g_ew_last_kernel = "nhwc_to_nchw_f32_kernel";
}
void k_permute(int prec, const void* src, void* dst, int N, int C, int HW, int to_nhwc, cudaStream_t s) {
  size_t n = (size_t)N * C * HW; if (!n) return;
  DISPATCH_PREC(prec, T, (launch_pdl(permute_kernel<T>, dim3(ew_blocks(n)), dim3(256), (size_t)(0), s, (const T*)src, (T*)dst, N, C, HW, to_nhwc))); LAUNCHED();
  g_ew_last_kernel = "permute_kernel";
}
__global__ void cast_f32_to_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, size_t n) { pdl_enter();
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) dst[i] = __float2bfloat16_rn(src[i]);
}
void k_cast_f32_to_bf16(const float* src, __nv_bfloat16* dst, size_t n, cudaStream_t s) {
  if (!n) return; launch_pdl(cast_f32_to_bf16_kernel, dim3(ew_blocks(n)), dim3(256), (size_t)(0), s, src, dst, n); LAUNCHED();
  g_ew_last_kernel = "cast_f32_to_bf16_kernel";
}
// ---------------------------------------------------------------- sliced column reductions ---------------
// Thread idx -> (slice s = idx / C, channel c = idx % C); it sums rows s, s+S, s+2S, ... so that a warp
// reads consecutive addresses.  partial[(g*S + s)*C + c].  Stage 2: one warp per channel, fixed order.
static const int SLICE_ELEMS = 1 << 20;     // S*C partial sums per group at most
static inline int pick_slices(int rows, int C) {
  int cap = SLICE_ELEMS / (C > 0 ? C : 1); if (cap < 1) cap = 1; if (cap > 2048) cap = 2048;
  int S = rows / 8; if (S < 1) S = 1; if (S > cap) S = cap; return S;
}
size_t k_bn_scratch_floats(int C, int groups) { return (size_t)2 * groups * (SLICE_ELEMS + 2 * (size_t)C) + 64; }
size_t k_colsum_scratch_floats(int C) { return (size_t)(SLICE_ELEMS + C) + 64; }

__device__ __forceinline__ void unpack8(const uint4& u, float (&v)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int j = 0; j < 4; ++j) { float2 f = __bfloat1622float2(h[j]); v[2 * j] = f.x; v[2 * j + 1] = f.y; }
}
__device__ __forceinline__ uint4 pack8(const float (&v)[8]) {
  uint4 u; __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
  for (int j = 0; j < 4; ++j) h[j] = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]);
  return u;
}

// The statistics are accumulated around a per-(group, channel) pivot k = the group's first row: sum (x-k) and sum (x-k)^2.  The one-pass
// variance E[(x-k)^2] - E[x-k]^2 then loses nothing to cancellation when |mean| >> std (a constant channel gives exactly 0), which the
// raw E[x^2] - E[x]^2 in fp32 partial sums does.  The pivots go to pivot[g*C + c] for the final kernel.
template <typename T>
__global__ void bn_stats_partial_kernel(const T* __restrict__ x, int rows, int C, int S, float* __restrict__ psum, float* __restrict__ psq, float* __restrict__ pivot) { pdl_enter();
  int g = blockIdx.y;
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= S * C) return;
  int c = idx % C, sl = idx / C;
  const T* xg = x + (size_t)g * rows * C;
  const float k = ldf(xg, c);
  if (sl == 0) pivot[g * C + c] = k;
  float a = 0.f, b = 0.f;
  for (int r = sl; r < rows; r += S) { float v = ldf(xg, (size_t)r * C + c) - k; a += v; b = fmaf(v, v, b); }
  psum[((size_t)g * S + sl) * C + c] = a; psq[((size_t)g * S + sl) * C + c] = b;
}
// bf16, C % 8 == 0, C <= 2048: a 256-thread block = (C/8 channel-octets) x TY row lanes reduces a contiguous chunk of rows
// with 16-byte loads, folds its TY lanes in shared memory and writes ONE partial row per block: many threads in stage 1,
// few partials for stage 2.
static inline int vec_ty(int C) { int c8 = C / 8; int ty = 256 / c8; return ty < 1 ? 1 : ty; }
static inline bool vec_ok(int prec, int C) { return prec == PREC_BF16 && C % 8 == 0 && C / 8 <= 256 && 256 % (C / 8) == 0; }
static inline int vec_blocks(int rows, int C) { int ty = vec_ty(C); int b = rows / (ty * 4); int cap = SLICE_ELEMS / C; if (cap > 256) cap = 256; if (b > cap) b = cap; if (b < 1) b = 1; return b; }
template <int NV>
__device__ __forceinline__ void block_fold_write(float (&acc)[NV][8], int C, int C8, int c8, int ty, int TY, float* const (&dst)[NV], size_t row_off) {
  __shared__ float sred[NV][2048];
#pragma unroll
  for (int v = 0; v < NV; ++v)
#pragma unroll
    for (int j = 0; j < 8; ++j) sred[v][ty * C + c8 * 8 + j] = acc[v][j];
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
#pragma unroll
    for (int v = 0; v < NV; ++v) { float a = 0.f; for (int k = 0; k < TY; ++k) a += sred[v][k * C + c]; dst[v][row_off + c] = a; }
  }
}
// stage 2: block = 32 adjacent channels x 16 slice lanes (coalesced 128-byte rows of the partial arrays), fixed-order tree in double
__global__ void __launch_bounds__(1024) bn_stats_final_kernel(const float* __restrict__ psum, const float* __restrict__ psq, const float* __restrict__ pivot, int rows, int C, int S, int groups, float eps,
                                      float* __restrict__ mean, float* __restrict__ invstd,
                                      const float* __restrict__ run_mean, const float* __restrict__ run_var, float* g_mean, float* g_var, float decay) { pdl_enter();
  __shared__ double sa[32][33], sb[32][33];      // 32 channels x 32 slice lanes: S <= 256 partial rows in ONE batch of 8 loads per thread
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5, c = blockIdx.x * 32 + tx;
  double acc_gm = 0.0, acc_gv = 0.0;
  for (int g = 0; g < groups; ++g) {
    double a = 0.0, b = 0.0;
    if (c < C) for (int sl0 = ty; sl0 < S; sl0 += 32 * 8) {      // 16 independent loads in flight per thread: one L2 round trip per batch
      float va[8], vb[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) { const int sl = sl0 + 32 * q; va[q] = sl < S ? psum[((size_t)g * S + sl) * C + c] : 0.f; vb[q] = sl < S ? psq[((size_t)g * S + sl) * C + c] : 0.f; }
#pragma unroll
      for (int q = 0; q < 8; ++q) { a += va[q]; b += vb[q]; }
    }
    sa[ty][tx] = a; sb[ty][tx] = b;
    __syncthreads();
    if (ty == 0 && c < C) {
      for (int k = 1; k < 32; ++k) { a += sa[k][tx]; b += sb[k][tx]; }
      const double d = a / rows, mu = (double)pivot[g * C + c] + d; double var = b / rows - d * d; if (var < 0) var = 0;
      mean[g * C + c] = (float)mu; invstd[g * C + c] = (float)(1.0 / sqrt(var + (double)eps));
      if (g_mean) { acc_gm += (1.0 - decay) * ((double)run_mean[c] - mu); acc_gv += (1.0 - decay) * ((double)run_var[c] - var); }
    }
    __syncthreads();
  }
  // BatchNormalization running stats as pseudo-gradients through a NoOp updater; groups (the two D minibatches) averaged
  if (g_mean && ty == 0 && c < C) { g_mean[c] = (float)(acc_gm / groups); g_var[c] = (float)(acc_gv / groups); }
}
void k_bn_stats(int prec, const void* x, int rows, int C, int groups, float* scratch, float* mean, float* invstd, float eps,
                const float* run_mean, const float* run_var, float* g_mean, float* g_var, float decay, cudaStream_t s) {
  const int S = pick_slices(rows, C);
  float* psum = scratch; float* psq = scratch + (size_t)groups * S * C; float* pivot = psq + (size_t)groups * S * C;
  dim3 grid((S * C + 255) / 256, groups);
  DISPATCH_PREC(prec, T, (launch_pdl(bn_stats_partial_kernel<T>, dim3(grid), dim3(256), (size_t)(0), s, (const T*)x, rows, C, S, psum, psq, pivot)));
  LAUNCHED();
  launch_pdl(bn_stats_final_kernel, dim3((C + 31) / 32), dim3(1024), (size_t)(0), s, psum, psq, (const float*)pivot, rows, C, S, groups, eps, mean, invstd, run_mean, run_var, g_mean, g_var, decay); LAUNCHED();
}
__global__ void bn_prep_infer_kernel(const float* __restrict__ rm, const float* __restrict__ rv, int C, int groups, float eps, float* mean, float* invstd) { pdl_enter();
  int i = blockIdx.x * blockDim.x + threadIdx.x; if (i >= C * groups) return;
  int c = i % C; mean[i] = rm[c]; invstd[i] = 1.0f / sqrtf(rv[c] + eps);
}
__global__ void bn_fold_kernel(const float* __restrict__ rm, const float* __restrict__ rv, const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ cb, int C, float eps, float* scale, float* shift) { pdl_enter();
  int c = blockIdx.x * blockDim.x + threadIdx.x; if (c >= C) return;
  const float sc = gamma[c] / sqrtf(rv[c] + eps); scale[c] = sc; shift[c] = beta[c] - rm[c] * sc + (cb ? cb[c] * sc : 0.f);
}
void k_bn_fold(const float* rm, const float* rv, const float* gamma, const float* beta, const float* cb, int C, float eps, float* scale, float* shift, cudaStream_t s) {
  launch_pdl(bn_fold_kernel, dim3((C + 255) / 256), dim3(256), (size_t)0, s, rm, rv, gamma, beta, cb, C, eps, scale, shift); LAUNCHED();
}
void k_bn_prep_infer(const float* run_mean, const float* run_var, int C, int groups, float eps, float* mean, float* invstd, cudaStream_t s) {
  launch_pdl(bn_prep_infer_kernel, dim3((C * groups + 255) / 256), dim3(256), (size_t)(0), s, run_mean, run_var, C, groups, eps, mean, invstd); LAUNCHED();
}

template <typename T>
__global__ void bn_apply_kernel(const T* __restrict__ x, T* __restrict__ y, int rows, int C, int groups, const float* __restrict__ mean,
                                const float* __restrict__ invstd, const float* __restrict__ gamma, const float* __restrict__ beta, int act, float alpha) { pdl_enter();
  size_t per_group = (size_t)rows * C, total = per_group * groups;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int c = i % C; int g = i / per_group;
    float v = (ldf(x, i) - mean[g * C + c]) * invstd[g * C + c];
    stf(y, i, act_fwd(act, fmaf(gamma[c], v, beta[c]), alpha));
  }
}
// bf16, C % 8 == 0 and 256 % (C/8) == 0: 16-byte vectors.  The grid stride (gridDim.x * 256 vectors) is a multiple of C/8, so a thread always
// meets the same 8 channels: their coefficients are loaded once per group instead of 4-6 scalar loads per element.
template <int ACTC>
__global__ void __launch_bounds__(256, 3) bn_apply_bf16x8_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int rows, int C, int groups, const float* __restrict__ mean,
                                       const float* __restrict__ invstd, const float* __restrict__ gamma, const float* __restrict__ beta, int act, float alpha) { pdl_enter();
  const int C8 = C / 8; const size_t per_group = (size_t)rows * C8;
  const size_t t0 = blockIdx.x * (size_t)blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
  const int c0 = (int)(t0 % C8) * 8;
  for (int g = 0; g < groups; ++g) {
    float mu[8], is[8], ga[8], be[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { mu[j] = mean[g * C + c0 + j]; is[j] = invstd[g * C + c0 + j]; ga[j] = gamma[c0 + j]; be[j] = beta[c0 + j]; }
    const uint4* xg = x + g * per_group; uint4* yg = y + g * per_group;
    for (size_t i = t0; i < per_group; i += 4 * stride) {        // four independent 16-byte loads in flight per thread
      uint4 xa[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) if (i + q * stride < per_group) xa[q] = xg[i + q * stride];
#pragma unroll
      for (int q = 0; q < 4; ++q) if (i + q * stride < per_group) {
        float v[8]; unpack8(xa[q], v);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = act_fwd(ACTC < 0 ? act : ACTC, fmaf(ga[j], (v[j] - mu[j]) * is[j], be[j]), alpha);
        yg[i + q * stride] = pack8(v);
      }
    }
  }
}
void k_bn_apply(int prec, const void* x, void* y, int rows, int C, int groups, const float* mean, const float* invstd,
                const float* gamma, const float* beta, int act, float alpha, cudaStream_t s) {
  size_t n = (size_t)rows * C * groups; if (!n) return;
  if (vec_ok(prec, C)) {
    DISPATCH_ACT(act, ACTC, launch_pdl(bn_apply_bf16x8_kernel<ACTC>, dim3(vec4_blocks((size_t)rows * C / 8)), dim3(256), (size_t)(0), s, (const uint4*)x, (uint4*)y, rows, C, groups, mean, invstd, gamma, beta, act, alpha));
  } else {
    DISPATCH_PREC(prec, T, (launch_pdl(bn_apply_kernel<T>, dim3(ew_blocks(n)), dim3(256), (size_t)(0), s, (const T*)x, (T*)y, rows, C, groups, mean, invstd, gamma, beta, act, alpha)));
  }
  LAUNCHED();
}

// backward of a = act(y), y = gamma*xhat + beta
template <typename T>
__global__ void bn_bwd_partial_kernel(const T* __restrict__ x, const T* __restrict__ eo, int rows, int C, int S, const float* __restrict__ mean,
                                      const float* __restrict__ invstd, const float* __restrict__ gamma, const float* __restrict__ beta, int act, float alpha,
                                      float* __restrict__ p1, float* __restrict__ p2) { pdl_enter();
  int g = blockIdx.y;
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= S * C) return;
  int c = idx % C, sl = idx / C;
  const T* xg = x + (size_t)g * rows * C; const T* eg = eo + (size_t)g * rows * C;
  float mu = mean[g * C + c], is = invstd[g * C + c], ga = gamma[c], be = beta[c];
  float a = 0.f, b = 0.f;
  for (int r = sl; r < rows; r += S) {
    float xh = (ldf(xg, (size_t)r * C + c) - mu) * is;
    float dy = ldf(eg, (size_t)r * C + c) * act_grad_from_pre(act, fmaf(ga, xh, be), alpha);
    a += dy; b = fmaf(dy, xh, b);
  }
  p1[((size_t)g * S + sl) * C + c] = a; p2[((size_t)g * S + sl) * C + c] = b;
}
__global__ void __launch_bounds__(1024) bn_bwd_final_kernel(const float* __restrict__ p1, const float* __restrict__ p2, int rows, int C, int S, int groups,
                                    float* __restrict__ c1, float* __restrict__ c2, float* g_gamma, float* g_beta, int want) { pdl_enter();
  __shared__ double sa[32][33], sb[32][33];      // 32 channels x 32 slice lanes: S <= 256 partial rows in ONE batch of 8 loads per thread
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5, c = blockIdx.x * 32 + tx;
  double tg = 0.0, tb = 0.0;
  for (int g = 0; g < groups; ++g) {
    double a = 0.0, b = 0.0;
    if (c < C) for (int sl0 = ty; sl0 < S; sl0 += 32 * 8) {
      float va[8], vb[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) { const int sl = sl0 + 32 * q; va[q] = sl < S ? p1[((size_t)g * S + sl) * C + c] : 0.f; vb[q] = sl < S ? p2[((size_t)g * S + sl) * C + c] : 0.f; }
#pragma unroll
      for (int q = 0; q < 8; ++q) { a += va[q]; b += vb[q]; }
    }
    sa[ty][tx] = a; sb[ty][tx] = b;
    __syncthreads();
    if (ty == 0 && c < C) {
      for (int k = 1; k < 32; ++k) { a += sa[k][tx]; b += sb[k][tx]; }
      c1[g * C + c] = (float)(a / rows); c2[g * C + c] = (float)(b / rows); tb += a; tg += b;
    }
    __syncthreads();
  }
  if (want && ty == 0 && c < C) { g_beta[c] += (float)tb; g_gamma[c] += (float)tg; }
}
template <typename T>
__global__ void bn_bwd_apply_kernel(const T* __restrict__ x, const T* __restrict__ eo, T* __restrict__ ei, int rows, int C, int groups,
                                    const float* __restrict__ mean, const float* __restrict__ invstd, const float* __restrict__ gamma,
                                    const float* __restrict__ beta, int act, float alpha, const float* __restrict__ c1, const float* __restrict__ c2) { pdl_enter();
  size_t per_group = (size_t)rows * C, total = per_group * groups;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int c = i % C; int g = i / per_group; int k = g * C + c;
    float xh = (ldf(x, i) - mean[k]) * invstd[k];
    float dy = ldf(eo, i) * act_grad_from_pre(act, fmaf(gamma[c], xh, beta[c]), alpha);
    stf(ei, i, gamma[c] * invstd[k] * (dy - c1[k] - xh * c2[k]));
  }
}
void k_bn_bwd(int prec, const void* x, const void* eps_out, void* eps_in, int rows, int C, int groups,
              const float* mean, const float* invstd, const float* gamma, const float* beta, int act, float alpha,
              float* scratch, float* g_gamma, float* g_beta, int want, cudaStream_t s) {
  const int S = pick_slices(rows, C);
  float* p1 = scratch; float* p2 = p1 + (size_t)groups * S * C; float* c1 = p2 + (size_t)groups * S * C; float* c2 = c1 + (size_t)groups * C;
  dim3 grid((S * C + 255) / 256, groups);
  DISPATCH_PREC(prec, T, (launch_pdl(bn_bwd_partial_kernel<T>, dim3(grid), dim3(256), (size_t)(0), s, (const T*)x, (const T*)eps_out, rows, C, S, mean, invstd, gamma, beta, act, alpha, p1, p2)));
  LAUNCHED();
  launch_pdl(bn_bwd_final_kernel, dim3((C + 31) / 32), dim3(1024), (size_t)(0), s, p1, p2, rows, C, S, groups, c1, c2, g_gamma, g_beta, want); LAUNCHED();
  if (eps_in) {
    size_t n = (size_t)rows * C * groups;
    DISPATCH_PREC(prec, T, (launch_pdl(bn_bwd_apply_kernel<T>, dim3(ew_blocks(n)), dim3(256), (size_t)(0), s, (const T*)x, (const T*)eps_out, (T*)eps_in, rows, C, groups, mean, invstd, gamma, beta, act, alpha, c1, c2)));
    LAUNCHED();
  }
}


// ---------------------------------------------------------------- BatchNorm on 128-bit accumulators ----------------
// north_star's "BatchNorm fused with its producer": the batch statistics arrive in acc[groups][2][2][C] (common.cuh sacc_add) from the
// tensor-core GEMM epilogues (kernels_tc.cu EPI_STATS / EPI_BNBWD) or from the *_stats_acc kernels below; the apply kernels turn them into
// per-channel coefficients in shared memory (once per block, in double) and stream the tensor once.  bf16, C % 8 == 0, 256 % (C/8) == 0.
bool k_bn_vec_ok(int prec, int C) { return vec_ok(prec, C); }
size_t k_bn_acc_elems(int C, int groups) { return (size_t)groups * 4 * C; }

// The block fold runs in double.  bn_stats_acc_kernel also sums per thread in double: bn_apply_acc_kernel forms E[x^2] - E[x]^2, a difference
// of large numbers when |mean| >> std, so this kernel's sum x^2 is not rounded to fp32 on its way into the 128-bit accumulators (the kernel is
// bandwidth-bound; the double arithmetic is not on its critical path).  The backward per-thread sums stay fp32 (a few rows each); the fold
// over up to 256 row lanes stays in double because with unit coefficients the same kernel accumulates (sum dy', sum dy'*z), whose conversion
// to sum dy'*xhat cancels.  The EPI_STATS / EPI_BNBWD GEMM epilogues, the other producers of these accumulators, reduce in fp32 over each
// 128-row tile.
template <int NV, typename A>
__device__ __forceinline__ void block_fold_acc(A (&acc)[NV][8], int C, int c8, int ty, int TY, unsigned long long* accbase /* statistic v at accbase + v*2*C */) {
  __shared__ double sred[NV][2048];
#pragma unroll
  for (int v = 0; v < NV; ++v)
#pragma unroll
    for (int j = 0; j < 8; ++j) sred[v][ty * C + c8 * 8 + j] = acc[v][j];
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
#pragma unroll
    for (int v = 0; v < NV; ++v) { double a = 0.0; for (int k = 0; k < TY; ++k) a += sred[v][k * C + c]; sacc_add(accbase + (size_t)v * 2 * C, (size_t)C, (size_t)c, a); }
  }
}
__global__ void __launch_bounds__(256) bn_stats_acc_kernel(const uint4* __restrict__ x, int rows, int C, int S, unsigned long long* __restrict__ accp) { pdl_enter();
  const int g = blockIdx.y, C8 = C / 8, TY = 256 / C8, c8 = threadIdx.x % C8, ty = threadIdx.x / C8, sl = blockIdx.x;
  const int chunk = (rows + S - 1) / S, r0 = sl * chunk, r1 = min(rows, r0 + chunk);
  const uint4* xg = x + (size_t)g * rows * C8;
  double acc[2][8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { acc[0][j] = 0.0; acc[1][j] = 0.0; }
#pragma unroll 4
  for (int r = r0 + ty; r < r1; r += TY) { float v[8]; unpack8(xg[(size_t)r * C8 + c8], v);
#pragma unroll
    for (int j = 0; j < 8; ++j) { acc[0][j] += v[j]; acc[1][j] = fma((double)v[j], (double)v[j], acc[1][j]); } }
  block_fold_acc<2>(acc, C, c8, ty, TY, accp + (size_t)g * 4 * C);
}
void k_bn_stats_acc(const void* x, int rows, int C, int groups, unsigned long long* acc, cudaStream_t s) {
  const int S = vec_blocks(rows, C);
  launch_pdl(bn_stats_acc_kernel, dim3(S, groups), dim3(256), (size_t)0, s, (const uint4*)x, rows, C, S, acc); LAUNCHED();
}

// dynamic shared memory: [groups][2][C] floats = (scale, shift).  coef rows: scale, beta, mean, invstd.
// The backward kernels' pre-activation: the smooth activations need z's value, formed as (x - mean) * scale + beta (with |mean| >> std,
// x * scale + shift loses the low bits of z to the rounding of shift); relu / leaky relu only need its sign, taken from the same
// x * scale + shift the forward evaluated (shift recomputed bit for bit), so that act' and the stored output agree at the kink.
__device__ __forceinline__ float bn_pre_act(int act, float x, float sc, float be, float mu) {
  return (act == ACT_RELU || act == ACT_LRELU) ? fmaf(x, sc, fmaf(-mu, sc, be)) : fmaf(x - mu, sc, be);
}
template <int ACTC>
__global__ void __launch_bounds__(256, 3) bn_apply_acc_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int rows, int C, int groups, const unsigned long long* __restrict__ accp,
                                                             const float* __restrict__ gamma, const float* __restrict__ beta, int act, float alpha, float eps, float* __restrict__ coef,
                                                             const float* __restrict__ run_mean, const float* __restrict__ run_var, float* g_mean, float* g_var, float decay, int replicas) { pdl_enter();
  extern __shared__ float s_cf[];
  const double cnt = (double)rows * replicas, inv_cnt = 1.0 / cnt;       // sync_bn: the accumulators hold the sums of every replica (all-reduced 64-bit integers)
  const bool writer = blockIdx.x == 0;
  const int C8 = C / 8; const size_t per_group = (size_t)rows * C8;
  const size_t t0 = blockIdx.x * (size_t)blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
  // the first batch of activation loads does not depend on the statistics: it flies while the coefficients are derived
  uint4 xa[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) if (t0 + q * stride < per_group) xa[q] = x[t0 + q * stride];
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    double agm = 0.0, agv = 0.0;
    for (int g = 0; g < groups; ++g) {
      const unsigned long long* a = accp + (size_t)g * 4 * C;
      const double mu = sacc_read(a, (size_t)C, (size_t)c) * inv_cnt; double var = sacc_read(a + 2 * (size_t)C, (size_t)C, (size_t)c) * inv_cnt - mu * mu; if (var < 0) var = 0;
      const float is = (float)(1.0 / sqrt(var + (double)eps)), sc = gamma[c] * is, sh = fmaf(-(float)mu, sc, beta[c]);
      s_cf[(g * 2 + 0) * C + c] = sc; s_cf[(g * 2 + 1) * C + c] = sh;
      if (writer) {
        coef[(size_t)(g * 4 + 0) * C + c] = sc; coef[(size_t)(g * 4 + 1) * C + c] = beta[c]; coef[(size_t)(g * 4 + 2) * C + c] = (float)mu; coef[(size_t)(g * 4 + 3) * C + c] = is;
        if (g_mean) { agm += (1.0 - decay) * ((double)run_mean[c] - mu); agv += (1.0 - decay) * ((double)run_var[c] - var); }
      }
    }
    // BatchNormalization running stats as pseudo-gradients through a NoOp updater; groups (the two D minibatches) averaged
    if (writer && g_mean) { g_mean[c] = (float)(agm / groups); g_var[c] = (float)(agv / groups); }
  }
  __syncthreads();
  const int c0 = (int)(t0 % C8) * 8;
  bool preloaded = true;
  for (int g = 0; g < groups; ++g) {
    float sc[8], sh[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { sc[j] = s_cf[(g * 2 + 0) * C + c0 + j]; sh[j] = s_cf[(g * 2 + 1) * C + c0 + j]; }
    const uint4* xg = x + g * per_group; uint4* yg = y + g * per_group;
    for (size_t i = t0; i < per_group; i += 4 * stride) {        // four independent 16-byte loads in flight per thread
      if (!preloaded) {
#pragma unroll
        for (int q = 0; q < 4; ++q) if (i + q * stride < per_group) xa[q] = xg[i + q * stride];
      }
      preloaded = false;
#pragma unroll
      for (int q = 0; q < 4; ++q) if (i + q * stride < per_group) {
        float v[8]; unpack8(xa[q], v);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = act_fwd(ACTC < 0 ? act : ACTC, fmaf(v[j], sc[j], sh[j]), alpha);
        yg[i + q * stride] = pack8(v);
      }
    }
  }
}
void k_bn_apply_acc(const void* x, void* y, int rows, int C, int groups, const unsigned long long* acc, const float* gamma, const float* beta, int act, float alpha, float eps,
                    float* coef, const float* run_mean, const float* run_var, float* g_mean, float* g_var, float decay, cudaStream_t s, int replicas) {
  const size_t smem = sizeof(float) * 2 * groups * C;
  DISPATCH_ACT(act, ACTC, launch_pdl(bn_apply_acc_kernel<ACTC>, dim3(vec4_blocks((size_t)rows * C / 8)), dim3(256), smem, s, (const uint4*)x, (uint4*)y, rows, C, groups, acc, gamma, beta, act, alpha, eps,
                                     coef, run_mean, run_var, g_mean, g_var, decay, replicas));
  LAUNCHED();
}

template <int ACTC>
__global__ void __launch_bounds__(256, 3) bn_bwd_stats_acc_kernel(const uint4* __restrict__ x, const uint4* __restrict__ eo, int rows, int C, int S, const float* __restrict__ coef,
                                                                 int act, float alpha, unsigned long long* __restrict__ accp) { pdl_enter();
  const int g = blockIdx.y, C8 = C / 8, TY = 256 / C8, c8 = threadIdx.x % C8, ty = threadIdx.x / C8, sl = blockIdx.x;
  const int chunk = (rows + S - 1) / S, r0 = sl * chunk, r1 = min(rows, r0 + chunk);
  const uint4* xg = x + (size_t)g * rows * C8; const uint4* eg = eo + (size_t)g * rows * C8;
  float sc[8], be[8], mu[8], is[8], acc[2][8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { const int c = c8 * 8 + j; sc[j] = coef[(size_t)(g * 4 + 0) * C + c]; be[j] = coef[(size_t)(g * 4 + 1) * C + c]; mu[j] = coef[(size_t)(g * 4 + 2) * C + c]; is[j] = coef[(size_t)(g * 4 + 3) * C + c]; acc[0][j] = 0.f; acc[1][j] = 0.f; }
#pragma unroll 4
  for (int r = r0 + ty; r < r1; r += TY) {
    float xv[8], ev[8]; unpack8(xg[(size_t)r * C8 + c8], xv); unpack8(eg[(size_t)r * C8 + c8], ev);
#pragma unroll
    for (int j = 0; j < 8; ++j) { const float xh = (xv[j] - mu[j]) * is[j]; const float dy = ev[j] * act_grad_from_pre(ACTC < 0 ? act : ACTC, bn_pre_act(ACTC < 0 ? act : ACTC, xv[j], sc[j], be[j], mu[j]), alpha); acc[0][j] += dy; acc[1][j] = fmaf(dy, xh, acc[1][j]); }
  }
  block_fold_acc<2>(acc, C, c8, ty, TY, accp + (size_t)g * 4 * C);
}
void k_bn_bwd_stats_acc(const void* x, const void* eps_out, int rows, int C, int groups, const float* coef, int act, float alpha, unsigned long long* acc, cudaStream_t s) {
  const int S = vec_blocks(rows, C);
  DISPATCH_ACT(act, ACTC, launch_pdl(bn_bwd_stats_acc_kernel<ACTC>, dim3(S, groups), dim3(256), (size_t)0, s, (const uint4*)x, (const uint4*)eps_out, rows, C, S, coef, act, alpha, acc));
  LAUNCHED();
}

// dynamic shared memory: [groups][2][C] floats = (mean of dy', mean of dy'*xhat)
template <int ACTC, bool PREMUL>
__global__ void __launch_bounds__(256, 2) bn_bwd_apply_acc_kernel(const uint4* __restrict__ x, const uint4* __restrict__ eo, uint4* __restrict__ ei, int rows, int C, int groups,
                                                                 const float* __restrict__ coef, int act, float alpha, const unsigned long long* __restrict__ accp,
                                                                 float* g_gamma, float* g_beta, int want, int replicas) { pdl_enter();
  extern __shared__ float s_k[];
  const double cnt = (double)rows * replicas, inv_cnt = 1.0 / cnt;       // sync_bn: global sums; dgamma / dbeta are left as (global sum) / replicas, the gradient all-reduce restores the sum
  const bool writer = blockIdx.x == 0 && want;
  const int C8 = C / 8; const size_t per_group = (size_t)rows * C8;
  const size_t t0 = blockIdx.x * (size_t)blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
  uint4 xa[4], ea[4];      // first batch of loads: independent of the sums, in flight during the prologue
  if (ei) {
#pragma unroll
    for (int q = 0; q < 4; ++q) if (t0 + q * stride < per_group) { xa[q] = x[t0 + q * stride]; ea[q] = eo[t0 + q * stride]; }
  }
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    double tb = 0.0, tg = 0.0;
    for (int g = 0; g < groups; ++g) {
      const unsigned long long* a = accp + (size_t)g * 4 * C;
      const double s1 = sacc_read(a, (size_t)C, (size_t)c); double s2 = sacc_read(a + 2 * (size_t)C, (size_t)C, (size_t)c);
      if (PREMUL) s2 = (double)coef[(size_t)(g * 4 + 3) * C + c] * (s2 - (double)coef[(size_t)(g * 4 + 2) * C + c] * s1);      // (sum dy'*z) -> sum dy'*xhat
      s_k[(g * 2 + 0) * C + c] = (float)(s1 * inv_cnt); s_k[(g * 2 + 1) * C + c] = (float)(s2 * inv_cnt); tb += s1; tg += s2;
    }
    if (writer) { g_beta[c] += (float)(tb / replicas); g_gamma[c] += (float)(tg / replicas); }
  }
  __syncthreads();
  if (!ei) return;
  const int c0 = (int)(t0 % C8) * 8;
  bool preloaded = true;
  for (int g = 0; g < groups; ++g) {
    float sc[8], be[8], mu[8], is[8], k1[8], k2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { const int c = c0 + j; sc[j] = coef[(size_t)(g * 4 + 0) * C + c]; be[j] = coef[(size_t)(g * 4 + 1) * C + c]; mu[j] = coef[(size_t)(g * 4 + 2) * C + c]; is[j] = coef[(size_t)(g * 4 + 3) * C + c];
      k1[j] = s_k[(g * 2 + 0) * C + c]; k2[j] = s_k[(g * 2 + 1) * C + c]; }
    const uint4* xg = x + g * per_group; const uint4* eg = eo + g * per_group; uint4* ig = ei + g * per_group;
    for (size_t i = t0; i < per_group; i += 4 * stride) {
      if (!preloaded) {
#pragma unroll
        for (int q = 0; q < 4; ++q) if (i + q * stride < per_group) { xa[q] = xg[i + q * stride]; ea[q] = eg[i + q * stride]; }
      }
      preloaded = false;
#pragma unroll
      for (int q = 0; q < 4; ++q) if (i + q * stride < per_group) {
        float xv[8], ev[8], o[8]; unpack8(xa[q], xv); unpack8(ea[q], ev);
#pragma unroll
        for (int j = 0; j < 8; ++j) { const float xh = (xv[j] - mu[j]) * is[j];
          const float dy = PREMUL ? ev[j] : ev[j] * act_grad_from_pre(ACTC < 0 ? act : ACTC, bn_pre_act(ACTC < 0 ? act : ACTC, xv[j], sc[j], be[j], mu[j]), alpha); o[j] = sc[j] * (dy - k1[j] - xh * k2[j]); }
        ig[i + q * stride] = pack8(o);
      }
    }
  }
}
void k_bn_bwd_apply_acc(const void* x, const void* eps_out, void* eps_in, int rows, int C, int groups, const float* coef, int act, float alpha, int premul,
                        const unsigned long long* acc, float* g_gamma, float* g_beta, int want, cudaStream_t s, int replicas) {
  const size_t smem = sizeof(float) * 2 * groups * C;
  const dim3 grid(eps_in ? vec4_blocks((size_t)rows * C / 8) : 1);
  if (premul) { launch_pdl(bn_bwd_apply_acc_kernel<ACT_IDENTITY, true>, grid, dim3(256), smem, s, (const uint4*)x, (const uint4*)eps_out, (uint4*)eps_in, rows, C, groups, coef, act, alpha, acc, g_gamma, g_beta, want, replicas); }
  else { DISPATCH_ACT(act, ACTC, launch_pdl(bn_bwd_apply_acc_kernel<ACTC, false>, grid, dim3(256), smem, s, (const uint4*)x, (const uint4*)eps_out, (uint4*)eps_in, rows, C, groups, coef, act, alpha, acc, g_gamma, g_beta, want, replicas)); }
  LAUNCHED();
}


// ---------------------------------------------------------------- gradient all-reduce over peer memory ----------------
// (kernels.h: P2pArgs).  System-scope release / acquire on the flag words order the peer-memory data accesses; every slice of the vector has
// exactly one reader-writer GPU, so the sum is written in place.  The sum order is rank 0..W-1 on every GPU: all replicas hold identical bits.
// Waits are bounded: a rank that never arrives traps the kernel (an error the host sees) instead of hanging the GPU.
__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) { asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p) { unsigned v; asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ void p2p_wait_all(const unsigned* flags, int world, unsigned e) {
  for (int r = 0; r < world; ++r) {
    unsigned it = 0;
    while ((int)(ld_acquire_sys(flags + r) - e) < 0) { if (++it > (1u << 27)) __trap(); __nanosleep(32); }
  }
}
__global__ void __launch_bounds__(512) p2p_allreduce_kernel(const P2pArgs a) {
  __shared__ unsigned s_e;
  if (threadIdx.x == 0) s_e = *reinterpret_cast<volatile unsigned*>(a.state) + 1;
  __syncthreads();
  const unsigned e = s_e; const int W = a.world;
  unsigned* mine = a.flags[a.rank];
  if (blockIdx.x == 0 && threadIdx.x < W) st_release_sys(a.flags[threadIdx.x] + a.rank, e);       // "my gradients are final" -> every rank (this kernel runs after backward in stream order)
  if (threadIdx.x == 0) p2p_wait_all(mine, W, e);                                                   // every rank's gradients are final
  __syncthreads();
  const size_t nv = a.n / 4, chunk = (nv + W - 1) / W, v0 = min(nv, (size_t)a.rank * chunk), v1 = min(nv, v0 + chunk);
  for (size_t i = v0 + blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < v1; i += (size_t)gridDim.x * blockDim.x) {
    float4 acc = __ldcg(reinterpret_cast<const float4*>(a.grads[0]) + i);
    for (int r = 1; r < W; ++r) { const float4 v = __ldcg(reinterpret_cast<const float4*>(a.grads[r]) + i); acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w; }
    for (int r = 0; r < W; ++r) __stcg(reinterpret_cast<float4*>(a.grads[r]) + i, acc);
  }
  if (a.rank == W - 1 && blockIdx.x == 0 && threadIdx.x < (a.n & 3)) {      // the last n % 4 elements
    const size_t i = nv * 4 + threadIdx.x; float acc = __ldcg(a.grads[0] + i);
    for (int r = 1; r < W; ++r) acc += __ldcg(a.grads[r] + i);
    for (int r = 0; r < W; ++r) __stcg(a.grads[r] + i, acc);
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned t = atomicAdd(a.state + 1, 1u);
    if (t == gridDim.x - 1) {            // last block of this GPU: its slice is complete everywhere
      a.state[1] = 0;
      for (int r = 0; r < W; ++r) st_release_sys(a.flags[r] + 8 + a.rank, e);
      p2p_wait_all(mine + 8, W, e);      // every slice has landed in this GPU's buffer: the updater may read it
      *reinterpret_cast<volatile unsigned*>(a.state) = e;
      __threadfence();
    }
  }
}
void k_p2p_allreduce(const P2pArgs& a, cudaStream_t s) {
  const size_t slice = (a.n / 4 + a.world - 1) / a.world;
  int blocks = (int)((slice + 2047) / 2048); if (blocks > 120) blocks = 120; if (blocks < 1) blocks = 1;      // all blocks resident at once (the barriers spin)
  p2p_allreduce_kernel<<<blocks, 512, 0, s>>>(a); LAUNCHED();      // plain launch: starts after backward has completed, never lets the updater in early
}

// ---------------------------------------------------------------- activations ---------------------------
template <typename T>
__global__ void act_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, size_t n, int act, float alpha) { pdl_enter();
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) stf(y, i, act_fwd(act, ldf(x, i), alpha));
}
template <typename T>
__global__ void act_bwd_out_kernel(const T* __restrict__ a, const T* __restrict__ eo, T* __restrict__ ei, size_t n, int act, float alpha) { pdl_enter();
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    stf(ei, i, ldf(eo, i) * act_grad_from_out(act, ldf(a, i), alpha));
}
void k_act_fwd(int prec, const void* x, void* y, size_t n, int act, float alpha, cudaStream_t s) {
  if (!n) return; DISPATCH_PREC(prec, T, (launch_pdl(act_fwd_kernel<T>, dim3(ew_blocks(n)), dim3(256), (size_t)(0), s, (const T*)x, (T*)y, n, act, alpha))); LAUNCHED();
  g_ew_last_kernel = "act_fwd_kernel";
}
// bf16, 16-byte vectors (n % 8 == 0): the D1 / G-last activation derivative runs over the largest tensors of the step
template <int ACTC>
__global__ void __launch_bounds__(256, 4) act_bwd_out_bf16x8_kernel(const uint4* __restrict__ a, const uint4* __restrict__ eo, uint4* __restrict__ ei, size_t n8, int act, float alpha) { pdl_enter();
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n8; i += 4 * stride) {
    uint4 aa[4], ea[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) if (i + q * stride < n8) { aa[q] = a[i + q * stride]; ea[q] = eo[i + q * stride]; }
#pragma unroll
    for (int q = 0; q < 4; ++q) if (i + q * stride < n8) {
      float av[8], ev[8], o[8]; unpack8(aa[q], av); unpack8(ea[q], ev);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = ev[j] * act_grad_from_out(ACTC < 0 ? act : ACTC, av[j], alpha);
      ei[i + q * stride] = pack8(o);
    }
  }
}
void k_act_bwd_from_output(int prec, const void* a, const void* eo, void* ei, size_t n, int act, float alpha, cudaStream_t s) {
  if (!n) return;
  if (prec == PREC_BF16 && n % 8 == 0 && ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(eo) | reinterpret_cast<uintptr_t>(ei)) & 15) == 0) {
    DISPATCH_ACT(act, ACTC, launch_pdl(act_bwd_out_bf16x8_kernel<ACTC>, dim3(vec4_blocks(n / 8)), dim3(256), (size_t)0, s, (const uint4*)a, (const uint4*)eo, (uint4*)ei, n / 8, act, alpha)); LAUNCHED();
    g_ew_last_kernel = "act_bwd_out_bf16x8_kernel"; return;
  }
  DISPATCH_PREC(prec, T, (launch_pdl(act_bwd_out_kernel<T>, dim3(ew_blocks(n)), dim3(256), (size_t)(0), s, (const T*)a, (const T*)eo, (T*)ei, n, act, alpha))); LAUNCHED();
  g_ew_last_kernel = "act_bwd_out_kernel";
}
void k_sigmoid_out(int prec, const void* z, void* p, size_t n, cudaStream_t s) { k_act_fwd(prec, z, p, n, ACT_SIGMOID, 0.f, s); }

// ---------------------------------------------------------------- max-pool / upsample ---------------------
template <typename T>
__global__ void maxpool_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, uint8_t* __restrict__ arg, int N, int H, int W, int C, int OH, int OW, int KH, int KW, int SH, int SW) { pdl_enter();
  size_t total = (size_t)N * OH * OW * C;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int c = i % C; size_t t = i / C; int ox = t % OW; t /= OW; int oy = t % OH; size_t n = t / OH;
    float best = -INFINITY; int bi = 0;
    for (int r = 0; r < KH; ++r) for (int q = 0; q < KW; ++q) {   // row-major window order; first max wins (DL4J tie rule)
      float v = ldf(x, ((n * H + oy * SH + r) * W + ox * SW + q) * C + c);
      if (v > best) { best = v; bi = r * KW + q; }
    }
    stf(y, i, best); arg[i] = (uint8_t)bi;
  }
}
template <typename T>
__global__ void maxpool_bwd_kernel(const T* __restrict__ eo, const uint8_t* __restrict__ arg, T* __restrict__ ei, int N, int H, int W, int C, int OH, int OW, int KH, int KW, int SH, int SW) { pdl_enter();
  // gather form (deterministic): each input pixel sums the eps of the windows whose arg-max it is
  size_t total = (size_t)N * H * W * C;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int c = i % C; size_t t = i / C; int ix = t % W; t /= W; int iy = t % H; size_t n = t / H;
    float acc = 0.f;
    for (int r = 0; r < KH; ++r) { int ty = iy - r; if (ty < 0 || ty % SH) continue; int oy = ty / SH; if (oy >= OH) continue;
      for (int q = 0; q < KW; ++q) { int tx = ix - q; if (tx < 0 || tx % SW) continue; int ox = tx / SW; if (ox >= OW) continue;
        size_t o = ((n * OH + oy) * OW + ox) * C + c;
        if (arg[o] == r * KW + q) acc += ldf(eo, o);
      } }
    stf(ei, i, acc);
  }
}
void k_maxpool_fwd(int prec, const void* x, void* y, uint8_t* arg, int N, int H, int W, int C, int OH, int OW, int KH, int KW, int SH, int SW, cudaStream_t s) {
  size_t n = (size_t)N * OH * OW * C; if (!n) return;
  DISPATCH_PREC(prec, T, (launch_pdl(maxpool_fwd_kernel<T>, dim3(ew_blocks(n)), dim3(256), (size_t)(0), s, (const T*)x, (T*)y, arg, N, H, W, C, OH, OW, KH, KW, SH, SW))); LAUNCHED();
  g_ew_last_kernel = "maxpool_fwd_kernel";
}
void k_maxpool_bwd(int prec, const void* eo, const uint8_t* arg, void* ei, int N, int H, int W, int C, int OH, int OW, int KH, int KW, int SH, int SW, cudaStream_t s) {
  size_t n = (size_t)N * H * W * C; if (!n) return;
  DISPATCH_PREC(prec, T, (launch_pdl(maxpool_bwd_kernel<T>, dim3(ew_blocks(n)), dim3(256), (size_t)(0), s, (const T*)eo, arg, (T*)ei, N, H, W, C, OH, OW, KH, KW, SH, SW))); LAUNCHED();
  g_ew_last_kernel = "maxpool_bwd_kernel";
}
template <typename T>
__global__ void upsample_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, int N, int H, int W, int C, int f) { pdl_enter();
  size_t total = (size_t)N * H * f * W * f * C;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int c = i % C; size_t t = i / C; int ox = t % (W * f); t /= (W * f); int oy = t % (H * f); size_t n = t / (H * f);
    y[i] = x[((n * H + oy / f) * W + ox / f) * C + c];
  }
}
template <typename T>
__global__ void upsample_bwd_kernel(const T* __restrict__ eo, T* __restrict__ ei, int N, int H, int W, int C, int f) { pdl_enter();
  size_t total = (size_t)N * H * W * C;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int c = i % C; size_t t = i / C; int ix = t % W; t /= W; int iy = t % H; size_t n = t / H;
    float acc = 0.f;
    for (int a = 0; a < f; ++a) for (int b = 0; b < f; ++b) acc += ldf(eo, ((n * H * f + iy * f + a) * (size_t)(W * f) + ix * f + b) * C + c);
    stf(ei, i, acc);
  }
}
void k_upsample_fwd(int prec, const void* x, void* y, int N, int H, int W, int C, int f, cudaStream_t s) {
  size_t n = (size_t)N * H * f * W * f * C; if (!n) return;
  DISPATCH_PREC(prec, T, (launch_pdl(upsample_fwd_kernel<T>, dim3(ew_blocks(n)), dim3(256), (size_t)(0), s, (const T*)x, (T*)y, N, H, W, C, f))); LAUNCHED();
  g_ew_last_kernel = "upsample_fwd_kernel";
}
void k_upsample_bwd(int prec, const void* eo, void* ei, int N, int H, int W, int C, int f, cudaStream_t s) {
  size_t n = (size_t)N * H * W * C; if (!n) return;
  DISPATCH_PREC(prec, T, (launch_pdl(upsample_bwd_kernel<T>, dim3(ew_blocks(n)), dim3(256), (size_t)(0), s, (const T*)eo, (T*)ei, N, H, W, C, f))); LAUNCHED();
  g_ew_last_kernel = "upsample_bwd_kernel";
}

// ---------------------------------------------------------------- XENT ---------------------------------
// LossBinaryXENT + sigmoid on the logit (J:159-163): clip_eps>0 DL4J-exact, 0 = BCE-with-logits.  WM: row i's score and dz scaled by
// loss_wm_scale(wm, i, 0) (the score in double: (double)loss * (double)scale), summed in the unweighted order.
template <typename T, bool WM>
__global__ void xent_kernel(const T* __restrict__ z, const float* __restrict__ y, T* __restrict__ dz, float* __restrict__ loss_sums, int rows, float clip,
                            LossWM wm) { pdl_enter();
  int g = blockIdx.x;
  __shared__ double red[32];
  double acc = 0.0;
  for (int r = threadIdx.x; r < rows; r += blockDim.x) {
    size_t i = (size_t)g * rows + r;
    float zi = ldf(z, i), yi = y[i], loss, grad;
    float sg = 1.0f / (1.0f + expf(-zi));
    if (clip > 0.f) {
      float p = fminf(fmaxf(sg, clip), 1.0f - clip);
      loss = -(yi * logf(p) + (1.0f - yi) * logf(1.0f - p));
      grad = (p - yi) / (p * (1.0f - p)) * sg * (1.0f - sg);
    } else {
      loss = fmaxf(zi, 0.f) + log1pf(expf(-fabsf(zi))) - yi * zi;
      grad = sg - yi;
    }
    if (WM) { const float sc = loss_wm_scale(wm, i, 0); acc += __dmul_rn((double)loss, (double)sc); grad *= sc; }
    else acc += loss;
    stf(dz, i, grad);
  }
  for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = acc;
  __syncthreads();
  if (threadIdx.x == 0) { double t = 0; for (int w = 0; w < (blockDim.x + 31) / 32; ++w) t += red[w]; loss_sums[g] = (float)t; }
}
void k_xent(int prec, const void* z, const float* y, void* dz, float* loss_sums, int rows, int groups, float clip, cudaStream_t s) {
  DISPATCH_PREC(prec, T, (launch_pdl(xent_kernel<T, false>, dim3(groups), dim3(1024), (size_t)(0), s, (const T*)z, y, (T*)dz, loss_sums, rows, clip, LossWM{}))); LAUNCHED();
  g_ew_last_kernel = "xent_kernel";
}
void k_xent_wm(int prec, const void* z, const float* y, void* dz, float* loss_sums, int rows, int groups, float clip, const LossWM& wm, cudaStream_t s) {
  DISPATCH_PREC(prec, T, (launch_pdl(xent_kernel<T, true>, dim3(groups), dim3(1024), (size_t)(0), s, (const T*)z, y, (T*)dz, loss_sums, rows, clip, wm))); LAUNCHED();
  g_ew_last_kernel = "xent_kernel<wm>";
}

// LossMCXENT with softmax (J:357-362), K classes per row: one thread per row, block-level loss sum.  WM (labels given; mask per row, mw = 1):
// m_r = the row's mask (1 without one); with weights sy = sum_k w_k y_k in fp32, class order, and dz_k = m_r * (p_k * sy - w_k y_k)
// (LossMCXENT's weighted gradient), without them dz_k = m_r * (p_k - y_k); the score term is (double)(m_r * w_k y_k) * log(clamp(p_k)).
template <typename T, bool WM>
__global__ void softmax_xent_kernel(const T* __restrict__ z, const float* __restrict__ y, T* __restrict__ dz, T* __restrict__ p_out, float* __restrict__ loss_sum, int rows, int K,
                                    LossWM wm) { pdl_enter();
  __shared__ double red[32];
  double acc = 0.0;
  for (int r = threadIdx.x; r < rows; r += blockDim.x) {
    float m = -INFINITY; for (int k = 0; k < K; ++k) m = fmaxf(m, ldf(z, (size_t)r * K + k));
    float den = 0.f; for (int k = 0; k < K; ++k) den += expf(ldf(z, (size_t)r * K + k) - m);
    float sy = 0.f, mr = 1.f;
    if (WM) {
      if (wm.w) for (int k = 0; k < K; ++k) sy += __fmul_rn(wm.w[k], y[(size_t)r * K + k]);
      if (wm.m) mr = wm.m[r];
    }
    for (int k = 0; k < K; ++k) {
      const float p = expf(ldf(z, (size_t)r * K + k) - m) / den;
      if (p_out) stf(p_out, (size_t)r * K + k, p);
      if (WM) {
        const float yk = y[(size_t)r * K + k], wy = wm.w ? wm.w[k] * yk : yk;
        stf(dz, (size_t)r * K + k, mr * (wm.w ? __fmul_rn(p, sy) - wy : p - yk)); acc -= __dmul_rn((double)(mr * wy), log((double)fminf(fmaxf(p, 1e-10f), 1.0f - 1e-10f)));
      }
      else if (dz) { const float yk = y[(size_t)r * K + k]; stf(dz, (size_t)r * K + k, p - yk); acc -= (double)yk * log((double)fminf(fmaxf(p, 1e-10f), 1.0f - 1e-10f)); }
    }
  }
  for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = acc;
  __syncthreads();
  if (threadIdx.x == 0 && loss_sum) { double t = 0; for (int w = 0; w < (blockDim.x + 31) / 32; ++w) t += red[w]; loss_sum[0] = (float)t; }
}
void k_softmax_xent(int prec, const void* z, const float* y, void* dz, void* p_out, float* loss_sums, int rows, int K, cudaStream_t s) {
  DISPATCH_PREC(prec, T, (launch_pdl(softmax_xent_kernel<T, false>, dim3(1), dim3(1024), (size_t)0, s, (const T*)z, y, (T*)dz, (T*)p_out, loss_sums, rows, K, LossWM{}))); LAUNCHED();
  g_ew_last_kernel = "softmax_xent_kernel";
}
void k_softmax_xent_wm(int prec, const void* z, const float* y, void* dz, float* loss_sums, int rows, int K, const LossWM& wm, cudaStream_t s) {
  DISPATCH_PREC(prec, T, (launch_pdl(softmax_xent_kernel<T, true>, dim3(1), dim3(1024), (size_t)0, s, (const T*)z, y, (T*)dz, (T*)nullptr, loss_sums, rows, K, wm))); LAUNCHED();
  g_ew_last_kernel = "softmax_xent_kernel<wm>";
}

// ---------------------------------------------------------------- regression / margin losses ----------------
// LossMSE, LossL1, LossL2, LossMAE, LossHinge, LossSquaredHinge and LossWasserstein as ILossFunction.computeGradient(labels, preOutput,
// activationFn): a = act(z) in fp32, dz = dL/da * act'(a) with the derivative taken from a; formulas at b2g_loss (include/b200gan.h).
// Group g's rows * n_out elements are split into k_loss_blocks() slices fixed by the shape, one block each (at most LOSS_MAX_GRID blocks in
// all: one wave, so the kernel lets its successor in at once).  A block sums its elements' scores in double (its block_sum order is fixed) and
// writes the sum to partial[]; the last block to finish folds each group's partials, one warp per group, each lane a strided subset in slice
// order and then the warp's xor butterfly: the loss sums do not depend on the order the blocks ran in.
constexpr int LOSS_THREADS = 256, LOSS_ELEMS_PER_BLOCK = 1024, LOSS_MAX_GRID = 1024;
int k_loss_blocks(size_t n_per_group, int groups) {
  const size_t b = (n_per_group + LOSS_ELEMS_PER_BLOCK - 1) / LOSS_ELEMS_PER_BLOCK;
  return (int)std::min<size_t>(std::max<size_t>(b, 1), std::max(1, LOSS_MAX_GRID / groups));
}
// WM: element i's score and dz scaled by sc = loss_wm_scale(wm, i / n_out, i % n_out): the score l * (double)sc, dz = (dL/da * act'(a)) * sc.
template <typename T, bool WM>
__global__ void __launch_bounds__(LOSS_THREADS) loss_kernel(const T* __restrict__ z, const float* __restrict__ y, T* __restrict__ dz, float* __restrict__ loss_sums,
                                                           size_t n_per_group, int n_out, int bpg, int loss, int act, float alpha, double* partial, unsigned* ticket,
                                                           LossWM wm) {
  pdl_enter();
  __shared__ double red[LOSS_THREADS / 32];
  __shared__ int last;
  const int g = blockIdx.x / bpg, b = blockIdx.x % bpg;
  const float nf = (float)n_out;
  double acc = 0.0;
  for (size_t j = (size_t)b * LOSS_THREADS + threadIdx.x; j < n_per_group; j += (size_t)bpg * LOSS_THREADS) {
    const size_t i = (size_t)g * n_per_group + j;
    const float a = act_fwd(act, ldf(z, i), alpha), yi = y[i];
    const double e = (double)a - (double)yi, m = 1.0 - (double)yi * (double)a;    // error a - y; hinge margin 1 - y a
    double l; float ga;                                                              // this element's score (before / nOut) and dL/da
    switch (loss) {
      case LOSS_MSE: l = e * e; ga = 2.0f * (a - yi) / nf; break;
      case LOSS_L2: l = e * e; ga = 2.0f * (a - yi); break;
      case LOSS_L1: l = fabs(e); ga = (float)((a > yi) - (a < yi)); break;
      case LOSS_MAE: l = fabs(e); ga = (float)((a > yi) - (a < yi)) / nf; break;
      case LOSS_HINGE: l = fmax(m, 0.0); ga = m > 0.0 ? -yi : 0.f; break;
      case LOSS_SQUARED_HINGE: l = m > 0.0 ? m * m : 0.0; ga = m > 0.0 ? -2.0f * yi * (float)m : 0.f; break;
      default: l = (double)yi * (double)a; ga = yi / nf; break;                   // LOSS_WASSERSTEIN
    }
    if (WM) { const float sc = loss_wm_scale(wm, i / n_out, (int)(i % n_out)); acc += __dmul_rn(l, (double)sc); stf(dz, i, ga * act_grad_from_out(act, a, alpha) * sc); }
    else { acc += l; stf(dz, i, ga * act_grad_from_out(act, a, alpha)); }
  }
  const double tot = block_sum(acc, red);
  if (threadIdx.x == 0) {
    partial[blockIdx.x] = tot;
    __threadfence();
    last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();      // every partial is visible: each writer fenced before taking its ticket
  const bool per_out = loss == LOSS_MSE || loss == LOSS_MAE || loss == LOSS_WASSERSTEIN;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int gg = warp; gg < (int)(gridDim.x / bpg); gg += LOSS_THREADS / 32) {
    double s = 0.0;
    for (int k = lane; k < bpg; k += 32) s += __ldcg(partial + (size_t)gg * bpg + k);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) loss_sums[gg] = (float)(per_out ? s / n_out : s);
  }
  if (threadIdx.x == 0) { *ticket = 0u; __threadfence(); }
}
void k_loss(int prec, int loss, int act, float alpha, const void* z, const float* y, void* dz, float* loss_sums, int rows_per_group, int n_out, int groups,
            double* partial, unsigned* ticket, cudaStream_t s) {
  const size_t n = (size_t)rows_per_group * n_out; const int bpg = k_loss_blocks(n, groups);
  DISPATCH_PREC(prec, T, (launch_pdl(loss_kernel<T, false>, dim3(groups * bpg), dim3(LOSS_THREADS), (size_t)0, s, (const T*)z, y, (T*)dz, loss_sums, n, n_out, bpg,
                                     loss, act, alpha, partial, ticket, LossWM{}))); LAUNCHED();
  g_ew_last_kernel = "loss_kernel";
}
void k_loss_wm(int prec, int loss, int act, float alpha, const void* z, const float* y, void* dz, float* loss_sums, int rows_per_group, int n_out, int groups,
               double* partial, unsigned* ticket, const LossWM& wm, cudaStream_t s) {
  const size_t n = (size_t)rows_per_group * n_out; const int bpg = k_loss_blocks(n, groups);
  DISPATCH_PREC(prec, T, (launch_pdl(loss_kernel<T, true>, dim3(groups * bpg), dim3(LOSS_THREADS), (size_t)0, s, (const T*)z, y, (T*)dz, loss_sums, n, n_out, bpg,
                                     loss, act, alpha, partial, ticket, wm))); LAUNCHED();
  g_ew_last_kernel = "loss_kernel<wm>";
}

// ---------------------------------------------------------------- column sum / misc reductions -----------
template <typename T>
__global__ void colsum_partial_kernel(const T* __restrict__ x, int rows, int C, int S, float* __restrict__ p) { pdl_enter();
  int idx = blockIdx.x * blockDim.x + threadIdx.x; if (idx >= S * C) return;
  int c = idx % C, sl = idx / C; float a = 0.f;
  for (int r = sl; r < rows; r += S) a += ldf(x, (size_t)r * C + c);
  p[(size_t)sl * C + c] = a;
}
__global__ void __launch_bounds__(256) colsum_partial_bf16x8_kernel(const uint4* __restrict__ x, int rows, int C, int S, float* __restrict__ p) { pdl_enter();
  const int C8 = C / 8, TY = 256 / C8, c8 = threadIdx.x % C8, ty = threadIdx.x / C8, sl = blockIdx.x;
  const int chunk = (rows + S - 1) / S, r0 = sl * chunk, r1 = min(rows, r0 + chunk);
  float acc[1][8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[0][j] = 0.f;
  for (int r = r0 + ty; r < r1; r += TY) { float v[8]; unpack8(x[(size_t)r * C8 + c8], v);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[0][j] += v[j]; }
  float* const dst[1] = {p};
  block_fold_write<1>(acc, C, C8, c8, ty, TY, dst, (size_t)sl * C);
}
__global__ void __launch_bounds__(512) colsum_final_kernel(const float* __restrict__ p, int C, int S, float* out, int accumulate) { pdl_enter();
  __shared__ double sa[16][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5, c = blockIdx.x * 32 + tx;
  double a = 0.0;
  if (c < C) for (int sl0 = ty; sl0 < S; sl0 += 16 * 8) {
    float va[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) { const int sl = sl0 + 16 * q; va[q] = sl < S ? p[(size_t)sl * C + c] : 0.f; }
#pragma unroll
    for (int q = 0; q < 8; ++q) a += va[q];
  }
  sa[ty][tx] = a;
  __syncthreads();
  if (ty == 0 && c < C) { for (int k = 1; k < 16; ++k) a += sa[k][tx]; out[c] = (accumulate ? out[c] : 0.f) + (float)a; }
}
// bf16, C <= 4 (the G-last bias gradient: 3 channels x every pixel of the batch), rows % 8 == 0: a thread walks groups of 8 pixels = C 16-byte
// vectors (element k of a group belongs to channel k % C), block-folds its C sums and writes one partial row; <= 256 partial rows
template <int C>
__global__ void __launch_bounds__(256) colsum_small_c_kernel(const uint4* __restrict__ x, size_t groups8, float* __restrict__ p) { pdl_enter();
  float acc[C];
#pragma unroll
  for (int c = 0; c < C; ++c) acc[c] = 0.f;
  for (size_t gidx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; gidx < groups8; gidx += (size_t)gridDim.x * blockDim.x) {
    uint4 u[C];
#pragma unroll
    for (int q = 0; q < C; ++q) u[q] = x[gidx * C + q];
#pragma unroll
    for (int q = 0; q < C; ++q) { float v[8]; unpack8(u[q], v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[(q * 8 + j) % C] += v[j]; }
  }
  __shared__ float red[8][C];
#pragma unroll
  for (int c = 0; c < C; ++c) { float a = acc[c]; for (int m = 16; m; m >>= 1) a += __shfl_xor_sync(0xffffffffu, a, m); if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][c] = a; }
  __syncthreads();
  if (threadIdx.x < C) { float a = 0.f; for (int w = 0; w < 8; ++w) a += red[w][threadIdx.x]; p[(size_t)blockIdx.x * C + threadIdx.x] = a; }
}
void k_colsum(int prec, const void* x, int rows, int C, float* scratch, float* out, int accumulate, cudaStream_t s) {
  if (prec == PREC_BF16 && C >= 1 && C <= 4 && rows % 8 == 0 && rows >= 4096 && (reinterpret_cast<uintptr_t>(x) & 15) == 0) {
    const size_t groups8 = (size_t)rows / 8; int S = (int)std::min<size_t>(256, (groups8 + 255) / 256);
    switch (C) {
      case 1: launch_pdl(colsum_small_c_kernel<1>, dim3(S), dim3(256), (size_t)0, s, (const uint4*)x, groups8, scratch); g_ew_last_kernel = "colsum_small_c_kernel<1>"; break;
      case 2: launch_pdl(colsum_small_c_kernel<2>, dim3(S), dim3(256), (size_t)0, s, (const uint4*)x, groups8, scratch); g_ew_last_kernel = "colsum_small_c_kernel<2>"; break;
      case 3: launch_pdl(colsum_small_c_kernel<3>, dim3(S), dim3(256), (size_t)0, s, (const uint4*)x, groups8, scratch); g_ew_last_kernel = "colsum_small_c_kernel<3>"; break;
      default: launch_pdl(colsum_small_c_kernel<4>, dim3(S), dim3(256), (size_t)0, s, (const uint4*)x, groups8, scratch); g_ew_last_kernel = "colsum_small_c_kernel<4>"; break;
    }
    LAUNCHED();
    launch_pdl(colsum_final_kernel, dim3(1), dim3(512), (size_t)(0), s, scratch, C, S, out, accumulate); LAUNCHED();
    return;
  }
  // the 16-byte loads of the bf16x8 kernel need a 16-byte aligned x; any other x takes the element-wise kernel
  const bool vec = vec_ok(prec, C) && (reinterpret_cast<uintptr_t>(x) & 15) == 0;
  int S = vec ? vec_blocks(rows, C) : pick_slices(rows, C);
  if (vec) { launch_pdl(colsum_partial_bf16x8_kernel, dim3(S), dim3(256), (size_t)(0), s, (const uint4*)x, rows, C, S, scratch); g_ew_last_kernel = "colsum_partial_bf16x8_kernel"; }
  else { DISPATCH_PREC(prec, T, (launch_pdl(colsum_partial_kernel<T>, dim3((S * C + 255) / 256), dim3(256), (size_t)(0), s, (const T*)x, rows, C, S, scratch))); g_ew_last_kernel = "colsum_partial_kernel"; }
  LAUNCHED();
  launch_pdl(colsum_final_kernel, dim3((C + 31) / 32), dim3(512), (size_t)(0), s, scratch, C, S, out, accumulate); LAUNCHED();
}
// The regularization score terms, in an order fixed by the segment table: each thread walks every segment with a non-zero coefficient in
// turn and adds coef * its own double sum over the segment; then a warp butterfly and the warps in order.  ABS: |x| (l1), else x^2 (l2).
template <bool ABS>
__device__ __forceinline__ void segments_norm(const float* __restrict__ p, const int64_t* off, const int64_t* len, const float* coef, int nseg, double* out) {
  __shared__ double red[32];
  double acc = 0.0;
  for (int sgi = 0; sgi < nseg; ++sgi) {
    if (coef[sgi] == 0.f) continue;
    const float* q = p + off[sgi]; double a = 0.0;
    for (int64_t i = threadIdx.x; i < len[sgi]; i += blockDim.x) a += ABS ? fabs((double)q[i]) : (double)q[i] * q[i];
    acc += coef[sgi] * a;
  }
  for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = acc;
  __syncthreads();
  if (threadIdx.x == 0) { double t = 0; for (int w = 0; w < (blockDim.x + 31) / 32; ++w) t += red[w]; *out = t; }
}
__global__ void sumsq_segments_kernel(const float* __restrict__ p, const int64_t* off, const int64_t* len, const float* coef, int nseg, double* out) { pdl_enter();
  segments_norm<false>(p, off, len, coef, nseg, out);
}
__global__ void sumabs_segments_kernel(const float* __restrict__ p, const int64_t* off, const int64_t* len, const float* coef, int nseg, double* out) { pdl_enter();
  segments_norm<true>(p, off, len, coef, nseg, out);
}
void k_sumsq_segments(const float* p, const int64_t* so, const int64_t* sl, const float* sc, int nseg, double* out, cudaStream_t s) {
  launch_pdl(sumsq_segments_kernel, dim3(1), dim3(1024), (size_t)(0), s, p, so, sl, sc, nseg, out); LAUNCHED();
  g_ew_last_kernel = "sumsq_segments_kernel";
}
void k_sumabs_segments(const float* p, const int64_t* so, const int64_t* sl, const float* sc, int nseg, double* out, cudaStream_t s) {
  launch_pdl(sumabs_segments_kernel, dim3(1), dim3(1024), (size_t)(0), s, p, so, sl, sc, nseg, out); LAUNCHED();
  g_ew_last_kernel = "sumabs_segments_kernel";
}
__global__ void reduce_splits_kernel(const float* __restrict__ src, float* __restrict__ dst, size_t n, int splits, size_t stride, int accumulate) { pdl_enter();
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float a = accumulate ? dst[i] : 0.f;
    for (int k = 0; k < splits; ++k) a += src[(size_t)k * stride + i];
    dst[i] = a;
  }
}
// many splits, few outputs (the 3-channel edge weight gradients: ~300 partials of 3072 values): one warp per output element, lanes
// stride over the splits, fixed-order shuffle tree
__global__ void reduce_splits_wide_kernel(const float* __restrict__ src, float* __restrict__ dst, size_t n, int splits, size_t stride, int accumulate) { pdl_enter();
  const size_t o = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5; const int lane = threadIdx.x & 31;
  if (o >= n) return;
  float a = 0.f;
  for (int k = lane; k < splits; k += 32) a += src[(size_t)k * stride + o];
  for (int m = 16; m; m >>= 1) a += __shfl_xor_sync(0xffffffffu, a, m);
  if (lane == 0) dst[o] = (accumulate ? dst[o] : 0.f) + a;
}
void k_reduce_splits(const float* src, float* dst, size_t n, int splits, size_t stride, int accumulate, cudaStream_t s) {
  if (n && splits >= 64 && n <= (1u << 16)) {
    launch_pdl(reduce_splits_wide_kernel, dim3((unsigned)((n * 32 + 255) / 256)), dim3(256), (size_t)0, s, src, dst, n, splits, stride, accumulate); LAUNCHED();
    g_ew_last_kernel = "reduce_splits_wide_kernel"; return;
  }
  if (!n) return; launch_pdl(reduce_splits_kernel, dim3(ew_blocks(n)), dim3(256), (size_t)(0), s, src, dst, n, splits, stride, accumulate); LAUNCHED();
  g_ew_last_kernel = "reduce_splits_kernel";
}

// every split-K partial sum of a backward pass in ONE launch: block -> (job, chunk); few splits: a thread owns 4 consecutive outputs and walks
// the splits with float4 loads; many splits, few outputs (the 3-channel edge layers: ~300 partials of 3072 values): one warp per output
void reduce_list_push(ReduceList* rl, const float* src, float* dst, int64_t n, int splits, int64_t stride) {
  if (!rl || rl->count >= ReduceList::MAX_JOBS || n <= 0) return;
  ReduceJob& j = rl->jobs[rl->count++]; j.src = src; j.dst = dst; j.n = n; j.splits = splits; j.stride = stride;
  const bool wide = splits >= 64 && n <= (1 << 16);
  j.blocks = wide ? -(int)((n + 7) / 8) : (int)((n + 1023) / 1024);      // negative: warp-per-output mode
}
__global__ void __launch_bounds__(256) reduce_multi_kernel(const ReduceList rl) { pdl_enter();
  int b = blockIdx.x, ji = 0;
  while (ji < rl.count) { const int nb = abs(rl.jobs[ji].blocks); if (b < nb) break; b -= nb; ++ji; }
  if (ji >= rl.count) return;
  const ReduceJob& jb = rl.jobs[ji];
  if (jb.blocks < 0) {
    const int64_t o = (int64_t)b * 8 + (threadIdx.x >> 5); const int lane = threadIdx.x & 31;
    if (o >= jb.n) return;
    float a = 0.f;
    for (int k = lane; k < jb.splits; k += 32) a += jb.src[(int64_t)k * jb.stride + o];
    for (int m = 16; m; m >>= 1) a += __shfl_xor_sync(0xffffffffu, a, m);
    if (lane == 0) jb.dst[o] = a;
    return;
  }
  const int64_t i = ((int64_t)b * 256 + threadIdx.x) * 4;
  if (i >= jb.n) return;
  if (i + 4 <= jb.n && (jb.stride & 3) == 0 && ((reinterpret_cast<uintptr_t>(jb.src) | reinterpret_cast<uintptr_t>(jb.dst)) & 15) == 0) {
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
    for (int k = 0; k < jb.splits; ++k) { const float4 v = *reinterpret_cast<const float4*>(jb.src + (int64_t)k * jb.stride + i); a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w; }
    *reinterpret_cast<float4*>(jb.dst + i) = a;
  } else {
    for (int64_t e = i; e < jb.n && e < i + 4; ++e) { float a = 0.f; for (int k = 0; k < jb.splits; ++k) a += jb.src[(int64_t)k * jb.stride + e]; jb.dst[e] = a; }
  }
}
void k_reduce_multi(const ReduceList& rl, cudaStream_t s) {
  int blocks = 0; for (int i = 0; i < rl.count; ++i) blocks += abs(rl.jobs[i].blocks);
  if (!blocks) return;
  launch_pdl(reduce_multi_kernel, dim3(blocks), dim3(256), (size_t)0, s, rl); LAUNCHED();
  g_ew_last_kernel = "reduce_multi_kernel";
}

// ---------------------------------------------------------------- updater -------------------------------
// One pass over params: 28 B/param for Adam (read p,g,m,v; write p,m,v), 20 B/param RmsProp, +2 B bf16 shadow.  EXT kinds: Nesterovs and
// AdaGrad 20 B, AdaMax, Nadam and AdaDelta 28 B, AMSGrad 36 B (include/b200gan.h, b2g_updater, states each formula).
// SCALED: the L2 gradient normalization multiplier of the segment (kernels_gradnorm.cu) follows the minibatch division
// EXT: the kinds 4-9 besides 0-3 (a net that has one still has NoOp BatchNorm mean/var segments); s2 is AMSGrad's v-hat.  alpha_t: Adam's and
// AMSGrad's lr * sqrt(1 - b2^t) / (1 - b1^t), AdaMax's and Nadam's lr / (1 - b1^t), per block.
template <bool SCALED, bool EXT = false>
__device__ __forceinline__ float upd_elem(const UpdSeg& sg, float g, float p, float& s0, float& s1, float gscale, float alpha_t, float gmult,
                                          float* s2 = nullptr) {
  g *= gscale;
  if (SCALED) g *= gmult;
  if (sg.clip > 0.f) g = fminf(fmaxf(g, -sg.clip), sg.clip);
  float u;
  if (sg.kind == 0) u = sg.lr * g;
  else if (sg.kind == 1) { s0 = sg.b1 * s0 + (1.0f - sg.b1) * g * g; u = sg.lr * g / (sqrtf(s0) + sg.eps); }
  else if (sg.kind == 2) { s0 = sg.b1 * s0 + (1.0f - sg.b1) * g; s1 = sg.b2 * s1 + (1.0f - sg.b2) * g * g; u = alpha_t * s0 / (sqrtf(s1) + sg.eps); }
  else if (!EXT || sg.kind == 3) u = g;
  else if (sg.kind == 4) { const float vp = s0; s0 = sg.b1 * s0 - sg.lr * g; u = sg.b1 * vp - (1.0f + sg.b1) * s0; }             // Nesterovs
  else if (sg.kind == 5) { s0 = s0 + g * g; u = sg.lr * g / (sqrtf(s0) + sg.eps); }                                               // AdaGrad
  else if (sg.kind == 6) { s0 = sg.b1 * s0 + (1.0f - sg.b1) * g; s1 = fmaxf(sg.b2 * s1, fabsf(g)) + 1e-32f; u = alpha_t * s0 / s1; }  // AdaMax
  else if (sg.kind == 7) { s0 = sg.b1 * s0 + (1.0f - sg.b1) * g; s1 = sg.b2 * s1 + (1.0f - sg.b2) * g * g;                        // Nadam
                           u = alpha_t * (sg.b1 * s0 + (1.0f - sg.b1) * g) / (sqrtf(s1) + sg.eps); }
  else if (sg.kind == 8) { s0 = sg.b1 * s0 + (1.0f - sg.b1) * g; s1 = sg.b2 * s1 + (1.0f - sg.b2) * g * g; *s2 = fmaxf(*s2, s1);   // AMSGrad
                           u = alpha_t * s0 / (sqrtf(*s2) + sg.eps); }
  else { s0 = sg.b1 * s0 + (1.0f - sg.b1) * g * g; u = sqrtf(s1 + sg.eps) / sqrtf(s0 + sg.eps) * g;                              // AdaDelta
         s1 = sg.b1 * s1 + (1.0f - sg.b1) * u * u; }
  if (sg.l2 != 0.f) u = fmaf(sg.l2, p, u);
  if (sg.l1 != 0.f) u = fmaf(sg.l1, (float)((p > 0.f) - (p < 0.f)), u);     // + l1 * sign(p), exact: sign(+-0) = 0
  return p - u;
}
// SCHED: the segment's lr comes from its schedule (thread 0 evaluates it once per block, at *step before the increment or at *epoch)
// EXT: kinds 4-9 (upd_elem); st2 (AMSGrad's v-hat, allocated only for nets with an AMSGrad segment) is read by EXT instantiations only
template <bool SCALED, bool SCHED, bool EXT>
__global__ void __launch_bounds__(256) updater_kernel(float* __restrict__ params, const float* __restrict__ grads, float* __restrict__ st0, float* __restrict__ st1,
                                                      const UpdSeg* __restrict__ segs, const int32_t* __restrict__ chunk_seg, const int64_t* __restrict__ chunk_off,
                                                      float inv_mb, float inv_world, int* __restrict__ step, unsigned* __restrict__ ticket, __nv_bfloat16* __restrict__ shadow,
                                                      const float* __restrict__ gn_mult, const UpdSched* __restrict__ sched, const int64_t* __restrict__ epoch,
                                                      float* __restrict__ st2) { pdl_enter();
  UpdSeg sg = segs[chunk_seg[blockIdx.x]];
  const float gmult = SCALED ? gn_mult[chunk_seg[blockIdx.x]] : 1.0f;
  const int64_t base = chunk_off[blockIdx.x];
  const int64_t end = min(base + (int64_t)UPD_CHUNK, sg.off + sg.len);
  const int t = *step + 1;
  if (SCHED) {
    __shared__ float lr_s;
    if (threadIdx.x == 0) lr_s = sched_lr(sched[chunk_seg[blockIdx.x]], sg.lr, t - 1, (long long)*epoch);
    __syncthreads();
    sg.lr = lr_s;
  }
  float alpha_t = 0.f;
  if (!EXT) {
    if (sg.kind == 2) alpha_t = sg.lr * sqrtf(1.0f - powf(sg.b2, (float)t)) / (1.0f - powf(sg.b1, (float)t));
  } else {
    if (sg.kind == 2 || sg.kind == 8) alpha_t = sg.lr * sqrtf(1.0f - powf(sg.b2, (float)t)) / (1.0f - powf(sg.b1, (float)t));
    else if (sg.kind == 6 || sg.kind == 7) alpha_t = sg.lr / (1.0f - powf(sg.b1, (float)t));
  }
  const float gscale = sg.div_mb ? inv_mb : inv_world;     // BN running-stat pseudo-gradients: no /mb, mean over ranks
  // state slots each kind reads and writes: s0 every kind but Sgd / NoOp, s1 Adam / AdaMax / Nadam / AMSGrad / AdaDelta, s2 AMSGrad
  const bool has0 = EXT ? (sg.kind != 0 && sg.kind != 3) : (sg.kind == 1 || sg.kind == 2);
  const bool has1 = EXT ? (sg.kind == 2 || (sg.kind >= 6 && sg.kind <= 9)) : sg.kind == 2;
  const bool has2 = EXT && sg.kind == 8, sh = shadow && sg.off_bf >= 0;
  if (((base | end) & 3) == 0 && (!sh || ((sg.off_bf + (base - sg.off)) & 3) == 0)) {
    // 16-byte path: a full 4096-element chunk is four float4 per thread and array, all 16 loads issued before the first use (20 with v-hat)
    float4 gv[4], pv[4], s0[4], s1[4], s2[EXT ? 4 : 1];
#pragma unroll
    for (int q = 0; q < 4; ++q) { const int64_t i = base + 4 * (threadIdx.x + q * (int64_t)blockDim.x); const bool ok = i < end; const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
      gv[q] = ok ? *reinterpret_cast<const float4*>(grads + i) : z; pv[q] = ok ? *reinterpret_cast<const float4*>(params + i) : z;
      s0[q] = (ok && has0) ? *reinterpret_cast<const float4*>(st0 + i) : z; s1[q] = (ok && has1) ? *reinterpret_cast<const float4*>(st1 + i) : z;
      if (EXT) s2[EXT ? q : 0] = (ok && has2) ? *reinterpret_cast<const float4*>(st2 + i) : z; }
#pragma unroll
    for (int q = 0; q < 4; ++q) { const int64_t i = base + 4 * (threadIdx.x + q * (int64_t)blockDim.x); if (i >= end) continue;
      float4 p4;
      if (!EXT) {
        p4.x = upd_elem<SCALED>(sg, gv[q].x, pv[q].x, s0[q].x, s1[q].x, gscale, alpha_t, gmult); p4.y = upd_elem<SCALED>(sg, gv[q].y, pv[q].y, s0[q].y, s1[q].y, gscale, alpha_t, gmult);
        p4.z = upd_elem<SCALED>(sg, gv[q].z, pv[q].z, s0[q].z, s1[q].z, gscale, alpha_t, gmult); p4.w = upd_elem<SCALED>(sg, gv[q].w, pv[q].w, s0[q].w, s1[q].w, gscale, alpha_t, gmult);
      } else {
        float4& h = s2[EXT ? q : 0];
        p4.x = upd_elem<SCALED, true>(sg, gv[q].x, pv[q].x, s0[q].x, s1[q].x, gscale, alpha_t, gmult, &h.x);
        p4.y = upd_elem<SCALED, true>(sg, gv[q].y, pv[q].y, s0[q].y, s1[q].y, gscale, alpha_t, gmult, &h.y);
        p4.z = upd_elem<SCALED, true>(sg, gv[q].z, pv[q].z, s0[q].z, s1[q].z, gscale, alpha_t, gmult, &h.z);
        p4.w = upd_elem<SCALED, true>(sg, gv[q].w, pv[q].w, s0[q].w, s1[q].w, gscale, alpha_t, gmult, &h.w);
      }
      *reinterpret_cast<float4*>(params + i) = p4;
      if (has0) *reinterpret_cast<float4*>(st0 + i) = s0[q];
      if (has1) *reinterpret_cast<float4*>(st1 + i) = s1[q];
      if (EXT && has2) *reinterpret_cast<float4*>(st2 + i) = s2[EXT ? q : 0];
      if (sh) {
        const __nv_bfloat162 lo = __floats2bfloat162_rn(p4.x, p4.y), hi = __floats2bfloat162_rn(p4.z, p4.w);
        if (sg.off_ps < 0) *reinterpret_cast<uint2*>(shadow + sg.off_bf + (i - sg.off)) = make_uint2(*reinterpret_cast<const uint32_t*>(&lo), *reinterpret_cast<const uint32_t*>(&hi));
        else { upd_shadow(sg, shadow, i, lo.x); upd_shadow(sg, shadow, i + 1, lo.y); upd_shadow(sg, shadow, i + 2, hi.x); upd_shadow(sg, shadow, i + 3, hi.y); }
      }
    }
  } else {
    for (int64_t i0 = base + threadIdx.x; i0 < end; i0 += 4 * blockDim.x) {
      float gv[4], pv[4], s0[4], s1[4], s2[EXT ? 4 : 1];
#pragma unroll
      for (int q = 0; q < 4; ++q) { const int64_t i = i0 + q * (int64_t)blockDim.x; const bool ok = i < end;
        gv[q] = ok ? grads[i] : 0.f; pv[q] = ok ? params[i] : 0.f; s0[q] = (ok && has0) ? st0[i] : 0.f; s1[q] = (ok && has1) ? st1[i] : 0.f;
        if (EXT) s2[EXT ? q : 0] = (ok && has2) ? st2[i] : 0.f; }
#pragma unroll
      for (int q = 0; q < 4; ++q) { const int64_t i = i0 + q * (int64_t)blockDim.x; if (i >= end) continue;
        const float p = EXT ? upd_elem<SCALED, true>(sg, gv[q], pv[q], s0[q], s1[q], gscale, alpha_t, gmult, &s2[EXT ? q : 0])
                            : upd_elem<SCALED>(sg, gv[q], pv[q], s0[q], s1[q], gscale, alpha_t, gmult);
        params[i] = p; if (has0) st0[i] = s0[q]; if (has1) st1[i] = s1[q]; if (EXT && has2) st2[i] = s2[EXT ? q : 0];
        if (sh) upd_shadow(sg, shadow, i, __float2bfloat16_rn(p));
      }
    }
  }
  // iteration counter (Adam's t): every block has read *step above; the last one to get here bumps it for the next launch
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned done = atomicAdd(ticket, 1u);
    if (done == gridDim.x - 1) { *step = t; *ticket = 0u; __threadfence(); }
  }
}
void k_updater(float* params, const float* grads, float* st0, float* st1, float* st2, const UpdSeg* segs, const int32_t* chunk_seg, const int64_t* chunk_off,
               int nchunks, float inv_mb, float inv_world, int* step_dev, unsigned* ticket, __nv_bfloat16* shadow, const float* gn_mult,
               const UpdSched* sched, const int64_t* epoch_dev, bool ext, cudaStream_t s) {
  if (!nchunks) return;
  auto kern = ext ? (gn_mult ? (sched ? updater_kernel<true, true, true> : updater_kernel<true, false, true>)
                             : (sched ? updater_kernel<false, true, true> : updater_kernel<false, false, true>))
                  : (gn_mult ? (sched ? updater_kernel<true, true, false> : updater_kernel<true, false, false>)
                             : (sched ? updater_kernel<false, true, false> : updater_kernel<false, false, false>));
  launch_pdl(kern, dim3(nchunks), dim3(256), (size_t)(0), s, params, grads, st0, st1, segs, chunk_seg, chunk_off, inv_mb, inv_world, step_dev, ticket, shadow, gn_mult,
             sched, epoch_dev, st2);
  LAUNCHED();
}
__global__ void sched_lr_kernel(const UpdSeg* segs, const UpdSched* sched, int seg, const int* step, const int64_t* epoch, float* out) {
  if (threadIdx.x == 0 && blockIdx.x == 0) *out = sched_lr(sched[seg], segs[seg].lr, *step, (long long)*epoch);
}
void k_sched_lr(const UpdSeg* segs, const UpdSched* sched, int seg, const int* step_dev, const int64_t* epoch_dev, float* out, cudaStream_t s) {
  sched_lr_kernel<<<1, 32, 0, s>>>(segs, sched, seg, step_dev, epoch_dev, out); LAUNCHED();
}
__global__ void fill_f32_kernel(float* p, float v, size_t n) { pdl_enter();
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}
__global__ void scale_f32_kernel(float* p, float v, size_t n) { pdl_enter();
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] *= v;
}
void k_scale_f32(float* p, float v, size_t n, cudaStream_t s) { if (!n) return; launch_pdl(scale_f32_kernel, dim3(ew_blocks(n)), dim3(256), (size_t)(0), s, p, v, n); LAUNCHED(); }
void k_fill_f32(float* p, float v, size_t n, cudaStream_t s) { if (!n) return; launch_pdl(fill_f32_kernel, dim3(ew_blocks(n)), dim3(256), (size_t)(0), s, p, v, n); LAUNCHED(); }

}  // namespace b2g
