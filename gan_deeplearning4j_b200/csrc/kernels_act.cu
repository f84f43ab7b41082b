// kernels_act.cu -- the activations of b2g_activation codes 5-16 (ELU, SELU, Softplus, Softsign, HardTanh, HardSigmoid, ReLU6, Swish, Cube,
// RationalTanh, RectifiedTanh, ThresholdedReLU): a = f(z) and eps *= f'(z), both from the stored pre-activation z.  Formulas: include/b200gan.h
// (b2g_activation); oracle restatement: tests/activation_ref.py.
//
// A translation unit of its own, and the math is not in common.cuh's act_fwd switch: that switch is inlined into the GEMM epilogues, the
// BatchNorm kernels and the loss kernel, and new cases there would change the code nvcc generates for every one of them (DESIGN.md 3.1).  Each
// kind is its own instantiation, chosen once on the host; no kernel switches per element.
#include <stdint.h>
#include "kernels.h"
#include "common.cuh"

namespace b2g {

static inline int ew_blocks(size_t n) { const size_t cap = (size_t)device_sm_count() * 16; size_t b = (n + 255) / 256; if (b > cap) b = cap; if (b < 1) b = 1; return (int)b; }

// 16-byte vectors: 4 fp32 or 8 bf16 elements
__device__ __forceinline__ void ld16(const float* p, float (&v)[4]) { const float4 f = *reinterpret_cast<const float4*>(p); v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w; }
__device__ __forceinline__ void ld16(const __nv_bfloat16* p, float (&v)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p); const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int j = 0; j < 4; ++j) { const float2 f = __bfloat1622float2(h[j]); v[2 * j] = f.x; v[2 * j + 1] = f.y; }
}
__device__ __forceinline__ void st16(float* p, const float (&v)[4]) { *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]); }
__device__ __forceinline__ void st16(__nv_bfloat16* p, const float (&v)[8]) {
  uint4 u; __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
  for (int j = 0; j < 4; ++j) h[j] = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]);
  *reinterpret_cast<uint4*>(p) = u;
}

constexpr float SELU_L = 1.0507009873554805f, SELU_A = 1.6732632423543772f;
constexpr float RT_A = 1.7159f, RT_C = 1.41645f;
__device__ __forceinline__ float sigm(float z) { return 1.0f / (1.0f + expf(-z)); }

// f(z); alpha = ELU's alpha / ThresholdedReLU's theta (ignored by the other kinds)
template <int K> __device__ __forceinline__ float ext_f(float z, float alpha) {
  if constexpr (K == ACT_ELU) return z >= 0.f ? z : alpha * expm1f(z);
  else if constexpr (K == ACT_SELU) return z > 0.f ? SELU_L * z : (SELU_L * SELU_A) * expm1f(z);
  else if constexpr (K == ACT_SOFTPLUS) return fmaxf(z, 0.f) + log1pf(expf(-fabsf(z)));
  else if constexpr (K == ACT_SOFTSIGN) return z / (1.0f + fabsf(z));
  else if constexpr (K == ACT_HARDTANH) return fminf(1.0f, fmaxf(-1.0f, z));
  else if constexpr (K == ACT_HARDSIGMOID) return fminf(1.0f, fmaxf(0.f, 0.2f * z + 0.5f));
  else if constexpr (K == ACT_RELU6) return fminf(fmaxf(z, 0.f), 6.0f);
  else if constexpr (K == ACT_SWISH) return z * sigm(z);
  else if constexpr (K == ACT_CUBE) return z * z * z;
  else if constexpr (K == ACT_RATIONALTANH) {
    const float y = z * (2.0f / 3.0f), ay = fabsf(y), y2 = y * y, A = 1.0f + ay + y2 + RT_C * y2 * y2;
    return copysignf(RT_A * (1.0f - 1.0f / A), y);
  }
  else if constexpr (K == ACT_RECTIFIEDTANH) return fmaxf(0.f, tanhf(z));
  else { static_assert(K == ACT_THRESHOLDEDRELU, "kind"); return z > alpha ? z : 0.f; }
}
// f'(z)
template <int K> __device__ __forceinline__ float ext_df(float z, float alpha) {
  if constexpr (K == ACT_ELU) return z >= 0.f ? 1.0f : alpha * expf(z);
  else if constexpr (K == ACT_SELU) return z > 0.f ? SELU_L : (SELU_L * SELU_A) * expf(z);
  else if constexpr (K == ACT_SOFTPLUS) return sigm(z);
  else if constexpr (K == ACT_SOFTSIGN) { const float d = 1.0f + fabsf(z); return 1.0f / (d * d); }
  else if constexpr (K == ACT_HARDTANH) return (z >= -1.0f && z <= 1.0f) ? 1.0f : 0.f;
  else if constexpr (K == ACT_HARDSIGMOID) return (z >= -2.5f && z <= 2.5f) ? 0.2f : 0.f;
  else if constexpr (K == ACT_RELU6) return (z > 0.f && z < 6.0f) ? 1.0f : 0.f;
  else if constexpr (K == ACT_SWISH) { const float s = sigm(z); return s * (1.0f + z * (1.0f - s)); }
  else if constexpr (K == ACT_CUBE) return 3.0f * z * z;
  else if constexpr (K == ACT_RATIONALTANH) {
    const float y = z * (2.0f / 3.0f), ay = fabsf(y), y2 = y * y, A = 1.0f + ay + y2 + RT_C * y2 * y2;
    return (RT_A * (2.0f / 3.0f)) * (1.0f + ay * (2.0f + 4.0f * RT_C * y2)) / (A * A);    // sgn(y) * (2y + 4c y^3) = |y| (2 + 4c y^2)
  }
  else if constexpr (K == ACT_RECTIFIEDTANH) { if (!(z > 0.f)) return 0.f; const float t = tanhf(z); return 1.0f - t * t; }
  else { static_assert(K == ACT_THRESHOLDEDRELU, "kind"); return z > alpha ? 1.0f : 0.f; }
}

// vec = 1: every pointer 16-byte aligned, so the first n / V * V elements run as vectors; the rest (or everything when vec = 0) one element per thread
template <typename T, int K>
__global__ void __launch_bounds__(256) act_ext_fwd_kernel(const T* __restrict__ z, T* __restrict__ a, size_t n, float alpha, int vec) { pdl_enter();
  constexpr int V = 16 / sizeof(T);
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
  const size_t nv = vec ? n / V : 0;
  for (size_t i = tid; i < nv; i += stride) {
    float v[V]; ld16(z + i * V, v);
#pragma unroll
    for (int j = 0; j < V; ++j) v[j] = ext_f<K>(v[j], alpha);
    st16(a + i * V, v);
  }
  for (size_t e = nv * V + tid; e < n; e += stride) stf(a, e, ext_f<K>(ldf(z, e), alpha));
}
// eps = eps * f'(z), in place (the backward pass's epsilon buffer)
template <typename T, int K>
__global__ void __launch_bounds__(256) act_ext_bwd_kernel(const T* __restrict__ z, T* eps, size_t n, float alpha, int vec) { pdl_enter();
  constexpr int V = 16 / sizeof(T);
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
  const size_t nv = vec ? n / V : 0;
  for (size_t i = tid; i < nv; i += stride) {
    float v[V], e[V]; ld16(z + i * V, v); ld16(eps + i * V, e);
#pragma unroll
    for (int j = 0; j < V; ++j) e[j] *= ext_df<K>(v[j], alpha);
    st16(eps + i * V, e);
  }
  for (size_t e = nv * V + tid; e < n; e += stride) stf(eps, e, ldf(eps, e) * ext_df<K>(ldf(z, e), alpha));
}

static const char* const FWD_NAMES[] = {"act_ext_fwd_kernel<elu>", "act_ext_fwd_kernel<selu>", "act_ext_fwd_kernel<softplus>", "act_ext_fwd_kernel<softsign>",
  "act_ext_fwd_kernel<hardtanh>", "act_ext_fwd_kernel<hardsigmoid>", "act_ext_fwd_kernel<relu6>", "act_ext_fwd_kernel<swish>", "act_ext_fwd_kernel<cube>",
  "act_ext_fwd_kernel<rationaltanh>", "act_ext_fwd_kernel<rectifiedtanh>", "act_ext_fwd_kernel<thresholdedrelu>"};
static const char* const BWD_NAMES[] = {"act_ext_bwd_kernel<elu>", "act_ext_bwd_kernel<selu>", "act_ext_bwd_kernel<softplus>", "act_ext_bwd_kernel<softsign>",
  "act_ext_bwd_kernel<hardtanh>", "act_ext_bwd_kernel<hardsigmoid>", "act_ext_bwd_kernel<relu6>", "act_ext_bwd_kernel<swish>", "act_ext_bwd_kernel<cube>",
  "act_ext_bwd_kernel<rationaltanh>", "act_ext_bwd_kernel<rectifiedtanh>", "act_ext_bwd_kernel<thresholdedrelu>"};

bool act_ext_kind(int act) { return act >= ACT_EXT_FIRST && act <= ACT_EXT_LAST; }

template <int K>
static void launch_ext(bool bwd, int prec, const void* z, void* out, size_t n, float alpha, cudaStream_t s) {
  const int vec = ((reinterpret_cast<uintptr_t>(z) | reinterpret_cast<uintptr_t>(out)) & 15) == 0 ? 1 : 0;
  const size_t V = prec == PREC_F32 ? 4 : 8;
  const dim3 grid(ew_blocks(vec ? (n + V - 1) / V : n));
  if (bwd) DISPATCH_PREC(prec, T, (launch_pdl(act_ext_bwd_kernel<T, K>, grid, dim3(256), (size_t)0, s, (const T*)z, (T*)out, n, alpha, vec)));
  else DISPATCH_PREC(prec, T, (launch_pdl(act_ext_fwd_kernel<T, K>, grid, dim3(256), (size_t)0, s, (const T*)z, (T*)out, n, alpha, vec)));
  LAUNCHED();
}
static void dispatch_ext(bool bwd, int prec, int act, const void* z, void* out, size_t n, float alpha, cudaStream_t s) {
  if (!n || !act_ext_kind(act)) return;
  switch (act) {
    case ACT_ELU: launch_ext<ACT_ELU>(bwd, prec, z, out, n, alpha, s); break;
    case ACT_SELU: launch_ext<ACT_SELU>(bwd, prec, z, out, n, alpha, s); break;
    case ACT_SOFTPLUS: launch_ext<ACT_SOFTPLUS>(bwd, prec, z, out, n, alpha, s); break;
    case ACT_SOFTSIGN: launch_ext<ACT_SOFTSIGN>(bwd, prec, z, out, n, alpha, s); break;
    case ACT_HARDTANH: launch_ext<ACT_HARDTANH>(bwd, prec, z, out, n, alpha, s); break;
    case ACT_HARDSIGMOID: launch_ext<ACT_HARDSIGMOID>(bwd, prec, z, out, n, alpha, s); break;
    case ACT_RELU6: launch_ext<ACT_RELU6>(bwd, prec, z, out, n, alpha, s); break;
    case ACT_SWISH: launch_ext<ACT_SWISH>(bwd, prec, z, out, n, alpha, s); break;
    case ACT_CUBE: launch_ext<ACT_CUBE>(bwd, prec, z, out, n, alpha, s); break;
    case ACT_RATIONALTANH: launch_ext<ACT_RATIONALTANH>(bwd, prec, z, out, n, alpha, s); break;
    case ACT_RECTIFIEDTANH: launch_ext<ACT_RECTIFIEDTANH>(bwd, prec, z, out, n, alpha, s); break;
    default: launch_ext<ACT_THRESHOLDEDRELU>(bwd, prec, z, out, n, alpha, s); break;
  }
  g_ew_last_kernel = (bwd ? BWD_NAMES : FWD_NAMES)[act - ACT_EXT_FIRST];
}
void k_act_ext_fwd(int prec, int act, float alpha, const void* z, void* a, size_t n, cudaStream_t s) { dispatch_ext(false, prec, act, z, a, n, alpha, s); }
void k_act_ext_bwd(int prec, int act, float alpha, const void* z, void* eps, size_t n, cudaStream_t s) { dispatch_ext(true, prec, act, z, eps, n, alpha, s); }

}  // namespace b2g
