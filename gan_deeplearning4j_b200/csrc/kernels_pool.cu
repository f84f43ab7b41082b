// kernels_pool.cu -- average, sum and p-norm pooling: SubsamplingLayer AVG / SUM / PNORM with padding (pool2d_*) and GlobalPoolingLayer
// MAX / AVG / SUM / PNORM (global_pool_*).  Formulas, rounding and summation order: include/b200gan.h (b2g_pooling); oracle restatement:
// tests/pooling_ref.py.
//
// NHWC; one thread per (pixel, 16-byte channel vector) when C is a multiple of the vector width and every tensor is 16-byte aligned, else one
// thread per element (the same code at a vector width of 1).  Each kind is its own instantiation, chosen once on the host.  Every result is a
// pure function of the inputs and the shape: no atomics on data, fixed summation orders.  The max-pool and upsample kernels stay in kernels_ew.cu.
#include <stdint.h>
#include <limits.h>
#include <algorithm>
#include "kernels.h"
#include "common.cuh"

namespace b2g {

static inline int ew_blocks(size_t n) { const size_t cap = (size_t)device_sm_count() * 16; size_t b = (n + 255) / 256; if (b > cap) b = cap; if (b < 1) b = 1; return (int)b; }

// VW elements: a 16-byte vector (VW = 16 / sizeof(T)) or one element
template <int VW> __device__ __forceinline__ void ldv(const float* p, float (&v)[VW]) {
  if constexpr (VW == 1) v[0] = *p;
  else { const float4 f = *reinterpret_cast<const float4*>(p); v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w; }
}
template <int VW> __device__ __forceinline__ void ldv(const __nv_bfloat16* p, float (&v)[VW]) {
  if constexpr (VW == 1) v[0] = __bfloat162float(*p);
  else {
    const uint4 u = *reinterpret_cast<const uint4*>(p); const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
    for (int j = 0; j < 4; ++j) { const float2 f = __bfloat1622float2(h[j]); v[2 * j] = f.x; v[2 * j + 1] = f.y; }
  }
}
template <int VW> __device__ __forceinline__ void stv(float* p, const float (&v)[VW]) {
  if constexpr (VW == 1) *p = v[0];
  else *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
template <int VW> __device__ __forceinline__ void stv(__nv_bfloat16* p, const float (&v)[VW]) {
  if constexpr (VW == 1) *p = __float2bfloat16_rn(v[0]);
  else {
    uint4 u; __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
    for (int j = 0; j < 4; ++j) h[j] = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]);
    *reinterpret_cast<uint4*>(p) = u;
  }
}

// p-norm pieces for a whole p >= 1 (p = 1 and 2 exactly, else powf)
constexpr float PNORM_FLOOR = 1e-8f;
__device__ __forceinline__ float pn_pow(float a, int p) { return p == 1 ? a : p == 2 ? a * a : powf(a, (float)p); }                // a^p, a = |x|
__device__ __forceinline__ float pn_root(float s, int p) { return p == 1 ? s : p == 2 ? sqrtf(s) : powf(s, 1.0f / (float)p); }     // s^(1/p)
__device__ __forceinline__ float pn_num(float x, int p) {                                                                          // sign(x)|x|^(p-1)
  return p == 1 ? (float)((x > 0.f) - (x < 0.f)) : p == 2 ? x : copysignf(powf(fabsf(x), (float)(p - 1)), x);
}
__device__ __forceinline__ float pn_den(float y, int p) { return fmaxf(p == 1 ? 1.0f : p == 2 ? y : powf(y, (float)(p - 1)), PNORM_FLOOR); }   // max(y^(p-1), 1e-8)

// ------------------------------------------------------------------ SubsamplingLayer AVG / SUM / PNORM -----------------------------------
// One thread per (output pixel, channel vector): the window's in-range elements summed in fp32 in row-major window order (padding adds
// nothing), then AVG: sum / (KH*KW), PNORM: sum^(1/p) of |x|^p; rounded once to T.
template <typename T, int K, bool VEC>
__global__ void __launch_bounds__(256) pool2d_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, int N, int H, int W, int C, int OH, int OW, int KH, int KW,
                                                        int SH, int SW, int PH, int PW, int pn) { pdl_enter();
  constexpr int VW = VEC ? 16 / sizeof(T) : 1;
  const int CV = C / VW;
  const size_t total = (size_t)N * OH * OW * CV;
  const float area = (float)(KH * KW);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int cv = (int)(i % CV); size_t t = i / CV; const int ox = (int)(t % OW); t /= OW; const int oy = (int)(t % OH); const size_t n = t / OH;
    float acc[VW];
#pragma unroll
    for (int j = 0; j < VW; ++j) acc[j] = 0.f;
    const int y0 = oy * SH - PH, x0 = ox * SW - PW;
#pragma unroll 1
    for (int r = 0; r < KH; ++r) {
      const int iy = y0 + r; if (iy < 0 || iy >= H) continue;
#pragma unroll 1
      for (int q = 0; q < KW; ++q) {
        const int ix = x0 + q; if (ix < 0 || ix >= W) continue;
        float v[VW]; ldv<VW>(x + ((n * H + iy) * W + ix) * C + (size_t)cv * VW, v);
#pragma unroll
        for (int j = 0; j < VW; ++j) acc[j] += K == POOL_PNORM ? pn_pow(fabsf(v[j]), pn) : v[j];
      }
    }
#pragma unroll
    for (int j = 0; j < VW; ++j) {
      if constexpr (K == POOL_AVG) acc[j] = acc[j] / area;
      else if constexpr (K == POOL_PNORM) acc[j] = pn_root(acc[j], pn);
    }
    stv<VW>(y + i * VW, acc);
  }
}
// Gather form (as maxpool_bwd_kernel): each input element sums, over the windows that cover it (filter row r, then column q, ascending), eps
// (AVG, SUM) or eps / max(y^(p-1), 1e-8) (PNORM); then AVG: / (KH*KW), PNORM: * sign(x)|x|^(p-1).  y = the forward's output.
template <typename T, int K, bool VEC>
__global__ void __launch_bounds__(256) pool2d_bwd_kernel(const T* __restrict__ eo, const T* __restrict__ x, const T* __restrict__ y, T* __restrict__ ei, int N, int H,
                                                        int W, int C, int OH, int OW, int KH, int KW, int SH, int SW, int PH, int PW, int pn) { pdl_enter();
  constexpr int VW = VEC ? 16 / sizeof(T) : 1;
  const int CV = C / VW;
  const size_t total = (size_t)N * H * W * CV;
  const float area = (float)(KH * KW);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int cv = (int)(i % CV); size_t t = i / CV; const int ix = (int)(t % W); t /= W; const int iy = (int)(t % H); const size_t n = t / H;
    float acc[VW];
#pragma unroll
    for (int j = 0; j < VW; ++j) acc[j] = 0.f;
    for (int r = 0; r < KH; ++r) {
      const int ty = iy + PH - r; if (ty < 0 || ty % SH) continue; const int oy = ty / SH; if (oy >= OH) continue;
      for (int q = 0; q < KW; ++q) {
        const int tx = ix + PW - q; if (tx < 0 || tx % SW) continue; const int ox = tx / SW; if (ox >= OW) continue;
        const size_t o = ((n * OH + oy) * OW + ox) * C + (size_t)cv * VW;
        float e[VW]; ldv<VW>(eo + o, e);
        if constexpr (K == POOL_PNORM) {
          float yv[VW]; ldv<VW>(y + o, yv);
#pragma unroll
          for (int j = 0; j < VW; ++j) acc[j] += e[j] / pn_den(yv[j], pn);
        } else {
#pragma unroll
          for (int j = 0; j < VW; ++j) acc[j] += e[j];
        }
      }
    }
    if constexpr (K == POOL_AVG) {
#pragma unroll
      for (int j = 0; j < VW; ++j) acc[j] = acc[j] / area;
    } else if constexpr (K == POOL_PNORM) {
      float xv[VW]; ldv<VW>(x + i * VW, xv);
#pragma unroll
      for (int j = 0; j < VW; ++j) acc[j] *= pn_num(xv[j], pn);
    }
    stv<VW>(ei + i * VW, acc);
  }
}

// ------------------------------------------------------------------ GlobalPoolingLayer ---------------------------------------------------
// A block reduces `cw` channel vectors of one example over a pixel range [p0, p1): thread (tv, tp) = (threadIdx % cw, threadIdx / cw) takes
// channel vector chunk*cw + tv and pixels p0 + tp, p0 + tp + rows, ... (a warp reads whole lines of a pixel row), accumulating in fp32 in that
// order; thread tp = 0 then folds lanes 1 .. rows-1 in lane order.  MAX keeps (value, pixel) and takes a greater value, or an equal value at a
// smaller pixel, so the first maximum in row-major pixel order wins whatever the fold order.  With splits = 1 that thread finalises (AVG: / HW,
// PNORM: ^(1/p)) and stores; otherwise it stores its fp32 partial, and the last block to finish (ticket) folds every (n, c)'s partials in split
// order and finalises.  cw, rows and splits are fixed by the shape (gp_plan), so the result is the same bits on every run.
constexpr int GP_THREADS = 256, GP_TARGET_BLOCKS = 264, GP_MIN_PIXELS_PER_LANE = 4, GP_MAX_SPLITS = 64;
struct GpPlan { int cw, rows, chunks, splits; };
static GpPlan gp_plan(int N, int HW, int CV) {
  GpPlan p;
  p.cw = std::min(CV, 32); p.rows = GP_THREADS / p.cw; p.chunks = (CV + p.cw - 1) / p.cw;
  const long long blocks = (long long)N * p.chunks;
  long long s = blocks >= GP_TARGET_BLOCKS ? 1 : (GP_TARGET_BLOCKS + blocks - 1) / blocks;
  s = std::min<long long>(s, std::max(1, HW / (p.rows * GP_MIN_PIXELS_PER_LANE)));
  p.splits = (int)std::max<long long>(1, std::min<long long>(s, GP_MAX_SPLITS));
  return p;
}
template <int K> __device__ __forceinline__ void gp_combine(float& a, int& ai, float v, int vi) {
  if constexpr (K == POOL_MAX) { if (v > a || (v == a && vi < ai)) { a = v; ai = vi; } }
  else a += v;
}
template <int K> __device__ __forceinline__ float gp_final(float a, int HW, int pn) {
  if constexpr (K == POOL_AVG) return a / (float)HW;
  else if constexpr (K == POOL_PNORM) return pn_root(a, pn);
  else return a;
}

template <typename T, int K, bool VEC>
__global__ void __launch_bounds__(GP_THREADS) global_pool_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, int32_t* __restrict__ idx, int N, int HW, int C, int pn,
                                                                    int cw, int rows, int chunks, int splits, float* __restrict__ part, int32_t* __restrict__ part_idx,
                                                                    unsigned* ticket) { pdl_enter();
  constexpr int VW = VEC ? 16 / sizeof(T) : 1;
  __shared__ float sv[GP_THREADS * VW];
  __shared__ int si[K == POOL_MAX ? GP_THREADS * VW : 1];
  __shared__ int last;
  const int CV = C / VW;
  const int s = blockIdx.x % splits, ch = (blockIdx.x / splits) % chunks, n = blockIdx.x / (splits * chunks);
  const int tv = threadIdx.x % cw, tp = threadIdx.x / cw, cv = ch * cw + tv;
  const bool live = tp < rows && cv < CV;
  const int p0 = (int)((long long)HW * s / splits), p1 = (int)((long long)HW * (s + 1) / splits);
  float acc[VW]; int bi[VW];
#pragma unroll
  for (int j = 0; j < VW; ++j) { acc[j] = K == POOL_MAX ? -INFINITY : 0.f; bi[j] = INT_MAX; }
  if (live)
    for (int p = p0 + tp; p < p1; p += rows) {
      float v[VW]; ldv<VW>(x + ((size_t)n * HW + p) * C + (size_t)cv * VW, v);
#pragma unroll
      for (int j = 0; j < VW; ++j) {
        if constexpr (K == POOL_MAX) { if (v[j] > acc[j]) { acc[j] = v[j]; bi[j] = p; } }
        else acc[j] += K == POOL_PNORM ? pn_pow(fabsf(v[j]), pn) : v[j];
      }
    }
  if (tp < rows) {
#pragma unroll
    for (int j = 0; j < VW; ++j) { sv[threadIdx.x * VW + j] = acc[j]; if constexpr (K == POOL_MAX) si[threadIdx.x * VW + j] = bi[j]; }
  }
  __syncthreads();
  const bool writer = tp == 0 && cv < CV;
  if (writer) {
    for (int r = 1; r < rows; ++r) {
      const int o = (r * cw + tv) * VW;
#pragma unroll
      for (int j = 0; j < VW; ++j) gp_combine<K>(acc[j], bi[j], sv[o + j], K == POOL_MAX ? si[o + j] : 0);
    }
    const size_t c0 = (size_t)cv * VW;
    if (splits == 1) {
      float r[VW];
#pragma unroll
      for (int j = 0; j < VW; ++j) r[j] = gp_final<K>(acc[j], HW, pn);
      stv<VW>(y + (size_t)n * C + c0, r);
      if constexpr (K == POOL_MAX) {
#pragma unroll
        for (int j = 0; j < VW; ++j) idx[(size_t)n * C + c0 + j] = bi[j];
      }
    } else {
      const size_t o = ((size_t)n * splits + s) * C + c0;
#pragma unroll
      for (int j = 0; j < VW; ++j) { part[o + j] = acc[j]; if constexpr (K == POOL_MAX) part_idx[o + j] = bi[j]; }
      __threadfence();
    }
  }
  if (splits == 1) return;
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();      // every partial is visible: each writer fenced before the block took its ticket
  for (int e = threadIdx.x; e < N * C; e += blockDim.x) {      // N * C < 2^31: the engine's activation buffers are smaller
    const size_t nn = (size_t)(e / C), c = (size_t)(e % C);
    float a = __ldcg(part + nn * splits * C + c); int ai = K == POOL_MAX ? __ldcg(part_idx + nn * splits * C + c) : 0;
    for (int k = 1; k < splits; ++k) {
      const size_t o = (nn * splits + k) * C + c;
      gp_combine<K>(a, ai, __ldcg(part + o), K == POOL_MAX ? __ldcg(part_idx + o) : 0);
    }
    stf(y, e, gp_final<K>(a, HW, pn));
    if constexpr (K == POOL_MAX) idx[e] = ai;
  }
  if (threadIdx.x == 0) { *ticket = 0u; __threadfence(); }
}
// Element-wise over the input: AVG eps / HW, SUM eps, MAX eps at the recorded pixel and 0 elsewhere, PNORM eps / max(y^(p-1), 1e-8) *
// sign(x)|x|^(p-1).
template <typename T, int K, bool VEC>
__global__ void __launch_bounds__(256) global_pool_bwd_kernel(const T* __restrict__ eo, const T* __restrict__ x, const T* __restrict__ y, const int32_t* __restrict__ idx,
                                                             T* __restrict__ ei, int N, int HW, int C, int pn) { pdl_enter();
  constexpr int VW = VEC ? 16 / sizeof(T) : 1;
  const int CV = C / VW;
  const size_t total = (size_t)N * HW * CV;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int cv = (int)(i % CV); const size_t t = i / CV; const int p = (int)(t % HW); const size_t n = t / HW;
    const size_t o = n * C + (size_t)cv * VW;
    float e[VW]; ldv<VW>(eo + o, e);
    if constexpr (K == POOL_AVG) {
#pragma unroll
      for (int j = 0; j < VW; ++j) e[j] = e[j] / (float)HW;
    } else if constexpr (K == POOL_MAX) {
#pragma unroll
      for (int j = 0; j < VW; ++j) e[j] = idx[o + j] == p ? e[j] : 0.f;
    } else if constexpr (K == POOL_PNORM) {
      float xv[VW], yv[VW]; ldv<VW>(x + i * VW, xv); ldv<VW>(y + o, yv);
#pragma unroll
      for (int j = 0; j < VW; ++j) e[j] = e[j] / pn_den(yv[j], pn) * pn_num(xv[j], pn);
    }
    stv<VW>(ei + i * VW, e);
  }
}

// ------------------------------------------------------------------ host wrappers -------------------------------------------------------
static const char* const NAMES[4][4] = {      // [pool2d fwd, pool2d bwd, global fwd, global bwd][b2g_pooling]
  {"pool2d_fwd_kernel<max>", "pool2d_fwd_kernel<avg>", "pool2d_fwd_kernel<sum>", "pool2d_fwd_kernel<pnorm>"},
  {"pool2d_bwd_kernel<max>", "pool2d_bwd_kernel<avg>", "pool2d_bwd_kernel<sum>", "pool2d_bwd_kernel<pnorm>"},
  {"global_pool_fwd_kernel<max>", "global_pool_fwd_kernel<avg>", "global_pool_fwd_kernel<sum>", "global_pool_fwd_kernel<pnorm>"},
  {"global_pool_bwd_kernel<max>", "global_pool_bwd_kernel<avg>", "global_pool_bwd_kernel<sum>", "global_pool_bwd_kernel<pnorm>"}};
int g_pool_last_splits = 1;

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
static bool vec_ok(int prec, int C, std::initializer_list<const void*> ptrs) {
  if (C % (int)(16 / prec_size(prec))) return false;
  for (const void* p : ptrs) if (p && !aligned16(p)) return false;
  return true;
}

template <int K>
static void pool2d_launch(bool bwd, int prec, int pn, const void* eo, const void* x, const void* y, void* out, int N, int H, int W, int C, int OH, int OW,
                          int KH, int KW, int SH, int SW, int PH, int PW, cudaStream_t s) {
  const size_t V = 16 / prec_size(prec);
  const bool vec = bwd ? vec_ok(prec, C, {eo, x, y, out}) : vec_ok(prec, C, {x, out});
  const size_t n = (bwd ? (size_t)N * H * W * C : (size_t)N * OH * OW * C) / (vec ? V : 1);
  const dim3 grid(ew_blocks(n));
#define B2G_POOL2D(VEC)                                                                                                                          \
  do {                                                                                                                                           \
    if (bwd) DISPATCH_PREC(prec, T, (launch_pdl(pool2d_bwd_kernel<T, K, VEC>, grid, dim3(256), (size_t)0, s, (const T*)eo, (const T*)x, (const T*)y, (T*)out, \
                                                N, H, W, C, OH, OW, KH, KW, SH, SW, PH, PW, pn)));                                                \
    else DISPATCH_PREC(prec, T, (launch_pdl(pool2d_fwd_kernel<T, K, VEC>, grid, dim3(256), (size_t)0, s, (const T*)x, (T*)out, N, H, W, C, OH, OW, KH, KW, \
                                            SH, SW, PH, PW, pn)));                                                                               \
  } while (0)
  if (vec) B2G_POOL2D(true); else B2G_POOL2D(false);
#undef B2G_POOL2D
  LAUNCHED();
}
static void pool2d_dispatch(bool bwd, int prec, int kind, int pn, const void* eo, const void* x, const void* y, void* out, int N, int H, int W, int C, int OH,
                            int OW, int KH, int KW, int SH, int SW, int PH, int PW, cudaStream_t s) {
  if ((size_t)N * H * W * C == 0 || (size_t)N * OH * OW * C == 0) return;
  switch (kind) {
    case POOL_AVG: pool2d_launch<POOL_AVG>(bwd, prec, pn, eo, x, y, out, N, H, W, C, OH, OW, KH, KW, SH, SW, PH, PW, s); break;
    case POOL_SUM: pool2d_launch<POOL_SUM>(bwd, prec, pn, eo, x, y, out, N, H, W, C, OH, OW, KH, KW, SH, SW, PH, PW, s); break;
    case POOL_PNORM: pool2d_launch<POOL_PNORM>(bwd, prec, pn, eo, x, y, out, N, H, W, C, OH, OW, KH, KW, SH, SW, PH, PW, s); break;
    default: return;          // MAX is B2G_LAYER_MAXPOOL's kernels
  }
  g_ew_last_kernel = NAMES[bwd ? 1 : 0][kind];
}
void k_pool2d_fwd(int prec, int kind, int pn, const void* x, void* y, int N, int H, int W, int C, int OH, int OW, int KH, int KW, int SH, int SW, int PH, int PW,
                  cudaStream_t s) {
  pool2d_dispatch(false, prec, kind, pn, nullptr, x, nullptr, y, N, H, W, C, OH, OW, KH, KW, SH, SW, PH, PW, s);
}
void k_pool2d_bwd(int prec, int kind, int pn, const void* eps_out, const void* x, const void* y, void* eps_in, int N, int H, int W, int C, int OH, int OW, int KH,
                  int KW, int SH, int SW, int PH, int PW, cudaStream_t s) {
  pool2d_dispatch(true, prec, kind, pn, eps_out, x, y, eps_in, N, H, W, C, OH, OW, KH, KW, SH, SW, PH, PW, s);
}

int k_global_pool_splits(int prec, int N, int HW, int C, int vec) { return gp_plan(N, HW, vec ? C / (int)(16 / prec_size(prec)) : C).splits; }
size_t k_global_pool_partial_elems(int prec, int max_rows, int HW, int C) {
  size_t m = 0;
  for (int n = 1; n <= max_rows; ++n)
    for (int vec = 0; vec < 2; ++vec) {
      if (vec && C % (int)(16 / prec_size(prec))) continue;
      const int sp = k_global_pool_splits(prec, n, HW, C, vec);
      if (sp > 1) m = std::max(m, (size_t)n * sp * C);
    }
  return m;
}

template <int K>
static void global_fwd_launch(int prec, int pn, const void* x, void* y, int32_t* idx, int N, int HW, int C, float* part, int32_t* part_idx, unsigned* ticket,
                              cudaStream_t s) {
  const int V = (int)(16 / prec_size(prec));
  const bool vec = vec_ok(prec, C, {x, y});
  const GpPlan p = gp_plan(N, HW, vec ? C / V : C);
  const dim3 grid((unsigned)((long long)N * p.chunks * p.splits)), block(p.cw * p.rows);
  if (vec) DISPATCH_PREC(prec, T, (launch_pdl(global_pool_fwd_kernel<T, K, true>, grid, block, (size_t)0, s, (const T*)x, (T*)y, idx, N, HW, C, pn, p.cw, p.rows,
                                              p.chunks, p.splits, part, part_idx, ticket)));
  else DISPATCH_PREC(prec, T, (launch_pdl(global_pool_fwd_kernel<T, K, false>, grid, block, (size_t)0, s, (const T*)x, (T*)y, idx, N, HW, C, pn, p.cw, p.rows,
                                          p.chunks, p.splits, part, part_idx, ticket)));
  LAUNCHED();
  g_pool_last_splits = p.splits;
}
void k_global_pool_fwd(int prec, int kind, int pn, const void* x, void* y, int32_t* idx, int N, int HW, int C, float* part, int32_t* part_idx, unsigned* ticket,
                       cudaStream_t s) {
  if ((size_t)N * HW * C == 0) return;
  switch (kind) {
    case POOL_MAX: global_fwd_launch<POOL_MAX>(prec, pn, x, y, idx, N, HW, C, part, part_idx, ticket, s); break;
    case POOL_AVG: global_fwd_launch<POOL_AVG>(prec, pn, x, y, idx, N, HW, C, part, part_idx, ticket, s); break;
    case POOL_SUM: global_fwd_launch<POOL_SUM>(prec, pn, x, y, idx, N, HW, C, part, part_idx, ticket, s); break;
    case POOL_PNORM: global_fwd_launch<POOL_PNORM>(prec, pn, x, y, idx, N, HW, C, part, part_idx, ticket, s); break;
    default: return;
  }
  g_ew_last_kernel = NAMES[2][kind];
}

template <int K>
static void global_bwd_launch(int prec, int pn, const void* eo, const void* x, const void* y, const int32_t* idx, void* ei, int N, int HW, int C, cudaStream_t s) {
  const size_t V = 16 / prec_size(prec);
  const bool vec = vec_ok(prec, C, {eo, x, y, ei});
  const dim3 grid(ew_blocks((size_t)N * HW * C / (vec ? V : 1)));
  if (vec) DISPATCH_PREC(prec, T, (launch_pdl(global_pool_bwd_kernel<T, K, true>, grid, dim3(256), (size_t)0, s, (const T*)eo, (const T*)x, (const T*)y, idx, (T*)ei,
                                              N, HW, C, pn)));
  else DISPATCH_PREC(prec, T, (launch_pdl(global_pool_bwd_kernel<T, K, false>, grid, dim3(256), (size_t)0, s, (const T*)eo, (const T*)x, (const T*)y, idx, (T*)ei,
                                          N, HW, C, pn)));
  LAUNCHED();
}
void k_global_pool_bwd(int prec, int kind, int pn, const void* eps_out, const void* x, const void* y, const int32_t* idx, void* eps_in, int N, int HW, int C,
                       cudaStream_t s) {
  if ((size_t)N * HW * C == 0) return;
  switch (kind) {
    case POOL_MAX: global_bwd_launch<POOL_MAX>(prec, pn, eps_out, x, y, idx, eps_in, N, HW, C, s); break;
    case POOL_AVG: global_bwd_launch<POOL_AVG>(prec, pn, eps_out, x, y, idx, eps_in, N, HW, C, s); break;
    case POOL_SUM: global_bwd_launch<POOL_SUM>(prec, pn, eps_out, x, y, idx, eps_in, N, HW, C, s); break;
    case POOL_PNORM: global_bwd_launch<POOL_PNORM>(prec, pn, eps_out, x, y, idx, eps_in, N, HW, C, s); break;
    default: return;
  }
  g_ew_last_kernel = NAMES[3][kind];
}

}  // namespace b2g
