// common.cuh -- device helpers shared by the kernels of libb200gan.so
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <math.h>
#include <stdlib.h>
#include <stdint.h>
#include "kernels.h"

namespace b2g {

#define LAUNCHED() do { ++::b2g::g_launch_count; } while (0)

// Programmatic dependent launch (launch_pdl sets the attribute on every launch): a kernel launched with the attribute may be SCHEDULED while its predecessor in the stream is
// still running (as soon as every predecessor CTA has exited or called pdl_trigger()), so the ~2 us launch latency and the successor's
// prologue overlap the predecessor's tail; pdl_wait() -- the first thing every kernel of this library does before touching global memory --
// blocks until the predecessor has completed and flushed.  An early trigger in a multi-wave kernel lets waiting successor CTAs hold SM
// slots that the predecessor's later waves need, so only single-wave kernels trigger early, all others
// trigger implicitly when their CTAs exit.  Both instructions are no-ops for a launch without the attribute.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
// elementwise / reduction kernels: their grids are one wave (<= 8 blocks of 256 threads per SM), so they let the successor in at once
__device__ __forceinline__ void pdl_enter() { pdl_trigger(); pdl_wait(); }
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg{}; cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute at[1]; at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// 128-bit fixed-point accumulation of fp32 / fp64 partial sums with two 64-bit integer atomics: hi counts units of 2^-10, lo the remainder in units
// of 2^-60.  Integer addition commutes, so a sum of per-CTA partials is bit-identical whatever order the CTAs arrive in (fp32 / fp64 atomics
// are not), it is exact to 2^-61 per addend, and it cannot overflow below |total| ~ 9e15.  hi_lo[idx] / hi_lo[stride + idx].
__device__ __forceinline__ void sacc_add(unsigned long long* hi_lo, size_t stride, size_t idx, double d) {
  const long long hi = __double2ll_rn(d * 1024.0);
  const double r = d - (double)hi * (1.0 / 1024.0);
  const long long lo = __double2ll_rn(r * 1152921504606846976.0);
  atomicAdd(hi_lo + idx, (unsigned long long)hi);
  atomicAdd(hi_lo + stride + idx, (unsigned long long)lo);
}
__device__ __forceinline__ double sacc_read(const unsigned long long* hi_lo, size_t stride, size_t idx) {
  return (double)(long long)hi_lo[idx] * (1.0 / 1024.0) + (double)(long long)hi_lo[stride + idx] * (1.0 / 1152921504606846976.0);
}

// Sum over the block in a fixed order: each thread's running sum, a xor butterfly inside the warp, the warp sums added in warp order by
// thread 0.  Only thread 0's result is used.
__device__ __forceinline__ double block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  if (threadIdx.x == 0) for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
  return t;
}

// The factor of element (label row r, column j) of a weighted / masked loss (LossWM): w_j * m_rj in fp32, 1 for what is absent
__device__ __forceinline__ float loss_wm_scale(const LossWM& q, size_t r, int j) {
  float s = q.w ? q.w[j] : 1.0f;
  if (q.m) s *= q.m[r * q.mw + (q.mw > 1 ? j : 0)];
  return s;
}

// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11; the Random123 constants): a counter-based generator,
// so a mask element's random word is a pure function of (counter, key) and needs no state beyond the counter the caller forms.
struct Philox4 { uint32_t x[4]; };
__device__ __forceinline__ Philox4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
    const uint32_t lo0 = 0xD2511F53u * c0, hi0 = __umulhi(0xD2511F53u, c0);
    const uint32_t lo1 = 0xCD9E8D57u * c2, hi1 = __umulhi(0xCD9E8D57u, c2);
    c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
  }
  return Philox4{{c0, c1, c2, c3}};
}
__device__ __forceinline__ uint32_t pick4(const Philox4& r, unsigned j) { return j == 0 ? r.x[0] : j == 1 ? r.x[1] : j == 2 ? r.x[2] : r.x[3]; }

// Box-Muller of one Philox word pair (DropoutLayer kinds, weight noise, weight initialization) (include/b200gan.h
// b2g_dropout_kind): u and v are exact, so the draw depends only on logf / sqrtf / sincospif
__device__ __forceinline__ void box_muller(uint32_t xe, uint32_t xo, float& ze, float& zo) {
  const float u = ((float)(xe >> 9) + 0.5f) * 0x1p-23f, v = (float)(xo >> 8) * 0x1p-24f;
  const float r = sqrtf(-2.0f * logf(u));
  float sn, cs; sincospif(2.0f * v, &sn, &cs);
  ze = r * cs; zo = r * sn;
}
__device__ __forceinline__ void normals4(const Philox4& r, float (&z)[4]) { box_muller(r.x[0], r.x[1], z[0], z[1]); box_muller(r.x[2], r.x[3], z[2], z[3]); }

#define DISPATCH_PREC(prec, T, ...)                                   \
  do {                                                                \
    if ((prec) == ::b2g::PREC_F32) { using T = float; __VA_ARGS__; }  \
    else { using T = __nv_bfloat16; __VA_ARGS__; }                    \
  } while (0)

__device__ __forceinline__ float ldf(const float* p, size_t i) { return p[i]; }
__device__ __forceinline__ float ldf(const __nv_bfloat16* p, size_t i) { return __bfloat162float(p[i]); }
__device__ __forceinline__ void stf(float* p, size_t i, float v) { p[i] = v; }
__device__ __forceinline__ void stf(__nv_bfloat16* p, size_t i, float v) { p[i] = __float2bfloat16_rn(v); }

// One 16-byte chunk of V elements of T, widened to fp32 (the element-wise streams of kernels_graph.cu and kernels_prelu.cu)
template <typename T> struct GVec;
template <> struct GVec<float> {
  static constexpr int V = 4;
  static __device__ __forceinline__ void load(const float* p, float* v) { const float4 q = *reinterpret_cast<const float4*>(p); v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w; }
  static __device__ __forceinline__ void store(float* p, const float* v) { *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]); }
};
template <> struct GVec<__nv_bfloat16> {
  static constexpr int V = 8;
  static __device__ __forceinline__ void load(const __nv_bfloat16* p, float* v) {
    const uint4 q = *reinterpret_cast<const uint4*>(p); const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&q);
#pragma unroll
    for (int k = 0; k < 4; ++k) { const float2 f = __bfloat1622float2(h[k]); v[2 * k] = f.x; v[2 * k + 1] = f.y; }
  }
  static __device__ __forceinline__ void store(__nv_bfloat16* p, const float* v) {
    uint4 q; __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&q);
#pragma unroll
    for (int k = 0; k < 4; ++k) h[k] = __floats2bfloat162_rn(v[2 * k], v[2 * k + 1]);
    *reinterpret_cast<uint4*>(p) = q;
  }
};
// Load / store V elements starting at e: the 16-byte path when VEC and the chunk is whole, else element by element (clipped to n)
template <typename T, bool VEC>
__device__ __forceinline__ void ld_chunk(const T* p, size_t e, size_t n, float* v) {
  constexpr int V = GVec<T>::V;
  if (VEC && e + V <= n) { GVec<T>::load(p + e, v); return; }
#pragma unroll
  for (int k = 0; k < V; ++k) v[k] = e + k < n ? ldf(p, e + k) : 0.f;
}
template <typename T, bool VEC>
__device__ __forceinline__ void st_chunk(T* p, size_t e, size_t n, const float* v) {
  constexpr int V = GVec<T>::V;
  if (VEC && e + V <= n) { GVec<T>::store(p + e, v); return; }
#pragma unroll
  for (int k = 0; k < V; ++k) if (e + k < n) stf(p, e + k, v[k]);
}

// org.nd4j.linalg.activations.impl.Activation{Identity,TanH,Sigmoid,ReLU,LReLU}
__device__ __forceinline__ float act_fwd(int act, float z, float alpha) {
  switch (act) {
    case ACT_TANH: return tanhf(z);
    case ACT_SIGMOID: return 1.0f / (1.0f + expf(-z));
    case ACT_RELU: return fmaxf(z, 0.f);
    case ACT_LRELU: return z > 0.f ? z : alpha * z;
    default: return z;
  }
}
// f'(z) from the pre-activation z
__device__ __forceinline__ float act_grad_from_pre(int act, float z, float alpha) {
  switch (act) {
    case ACT_TANH: { float t = tanhf(z); return 1.0f - t * t; }
    case ACT_SIGMOID: { float s = 1.0f / (1.0f + expf(-z)); return s * (1.0f - s); }
    case ACT_RELU: return z > 0.f ? 1.0f : 0.f;
    case ACT_LRELU: return z > 0.f ? 1.0f : alpha;
    default: return 1.0f;
  }
}
// f'(z) from the activation output a = f(z)  (lrelu needs alpha > 0 so that sign(a) = sign(z))
__device__ __forceinline__ float act_grad_from_out(int act, float a, float alpha) {
  switch (act) {
    case ACT_TANH: return 1.0f - a * a;
    case ACT_SIGMOID: return a * (1.0f - a);
    case ACT_RELU: return a > 0.f ? 1.0f : 0.f;
    case ACT_LRELU: return a > 0.f ? 1.0f : alpha;
    default: return 1.0f;
  }
}

}  // namespace b2g
