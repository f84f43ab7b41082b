// kernels_dropout.cu -- DropoutLayer (DL4J 1.0.0-beta3 inverted dropout): the masked forward with its on-device Philox4x32-10 mask and
// pass counter, and the backward that applies the stored mask.  Mask definition: include/b200gan.h (B2G_LAYER_DROPOUT); oracle restatement:
// tests/dropout_ref.py dropout_mask.
//
// A translation unit of its own: compiled inside kernels_ew.cu these kernels changed the code nvcc generated for the updater kernel there
// (register allocation and scheduling of the unchanged source), and the C2 step, which has no DropoutLayer, ran about 1% slower on an H100.
#include <stdint.h>
#include "kernels.h"
#include "common.cuh"

namespace b2g {

static inline int ew_blocks(size_t n) { const size_t cap = (size_t)device_sm_count() * 16; size_t b = (n + 255) / 256; if (b > cap) b = cap; if (b < 1) b = 1; return (int)b; }

// One 16-byte vector per thread and iteration (4 fp32 / 8 bf16 elements = 1 / 2 Philox calls).  The forward's vector loop covers whole
// 32-element mask words only: a warp owns 32 consecutive vectors, i.e. V consecutive words, and assembles them with shuffles, so every
// mask word has one writer.  The rest (count not a multiple of 32*V, or misaligned pointers) runs one element per lane, one word per warp
// (ballot).  Both loops are warp-uniform.
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
__device__ __forceinline__ void ld16(const float* p, float (&v)[4]) { const float4 f = *reinterpret_cast<const float4*>(p); v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w; }
__device__ __forceinline__ void ld16(const __nv_bfloat16* p, float (&v)[8]) { unpack8(*reinterpret_cast<const uint4*>(p), v); }
__device__ __forceinline__ void st16(float* p, const float (&v)[4]) { *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]); }
__device__ __forceinline__ void st16(__nv_bfloat16* p, const float (&v)[8]) { *reinterpret_cast<uint4*>(p) = pack8(v); }
__device__ __forceinline__ uint32_t pick4(const Philox4& r, unsigned j) { return j == 0 ? r.x[0] : j == 1 ? r.x[1] : j == 2 ? r.x[2] : r.x[3]; }

template <typename T>
__global__ void __launch_bounds__(256) dropout_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, uint32_t* __restrict__ mask, size_t n, int vec,
                                                          const DropoutArgs a, unsigned long long* pass, unsigned* ticket, int bump) { pdl_enter();
  constexpr int V = 16 / sizeof(T);
  const unsigned long long P = *(volatile unsigned long long*)pass;       // read on the device: a captured graph draws new masks on every replay
  const uint32_t c1 = (uint32_t)P, c2 = (uint32_t)(P >> 32), k0 = (uint32_t)a.seed, k1 = (uint32_t)(a.seed >> 32);
  const int lane = threadIdx.x & 31;
  const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  const size_t n_main = vec ? n / (32 * V) * (32 * V) : 0;
  for (size_t base = warp * 32 * V; base < n_main; base += nwarps * 32 * V) {
    const size_t e0 = base + (size_t)lane * V;
    float v[V]; ld16(x + e0, v);
    uint32_t bits = 0;
#pragma unroll
    for (int h = 0; h < V / 4; ++h) {
      const Philox4 r = philox4x32_10((uint32_t)(e0 >> 2) + h, c1, c2, a.tag, k0, k1);
#pragma unroll
      for (int j = 0; j < 4; ++j) { const bool keep = a.keep_all || r.x[j] < a.threshold; bits |= (uint32_t)keep << (4 * h + j); v[4 * h + j] = keep ? v[4 * h + j] * a.scale : 0.f; }
    }
    st16(y + e0, v);
    uint32_t w = bits << ((lane * V) & 31);
#pragma unroll
    for (int o = 1; o < 32 / V; o <<= 1) w |= __shfl_xor_sync(0xffffffffu, w, o);
    if ((lane & (32 / V - 1)) == 0) mask[e0 >> 5] = w;
  }
  for (size_t base = n_main + warp * 32; base < n; base += nwarps * 32) {
    const size_t e = base + lane;
    bool keep = false;
    if (e < n) {
      const Philox4 r = philox4x32_10((uint32_t)(e >> 2), c1, c2, a.tag, k0, k1);
      keep = a.keep_all || pick4(r, (unsigned)(e & 3)) < a.threshold;
      stf(y, e, keep ? ldf(x, e) * a.scale : 0.f);
    }
    const uint32_t w = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) mask[base >> 5] = w;
  }
  // pass counter: every block has read P above; the last one to get here advances it for the next train-mode pass
  if (bump) {
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      const unsigned done = atomicAdd(ticket, 1u);
      if (done == gridDim.x - 1) { *pass = P + 1; *ticket = 0u; __threadfence(); }
    }
  }
}
template <typename T>
__global__ void __launch_bounds__(256) dropout_bwd_kernel(const T* eo, T* ei, const uint32_t* __restrict__ mask, size_t n, float scale, int vec) { pdl_enter();
  constexpr int V = 16 / sizeof(T);
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
  const size_t nv = vec ? n / V : 0;
  for (size_t i = tid; i < nv; i += stride) {
    const size_t e0 = i * V;
    const uint32_t bits = mask[e0 >> 5] >> (e0 & 31);
    float v[V]; ld16(eo + e0, v);
#pragma unroll
    for (int j = 0; j < V; ++j) v[j] = ((bits >> j) & 1u) ? v[j] * scale : 0.f;
    st16(ei + e0, v);
  }
  for (size_t e = nv * V + tid; e < n; e += stride) stf(ei, e, ((mask[e >> 5] >> (e & 31)) & 1u) ? ldf(eo, e) * scale : 0.f);
}
static inline bool aligned16(const void* a, const void* b) { return ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b)) & 15) == 0; }
void k_dropout_fwd(int prec, const void* x, void* y, uint32_t* mask, size_t n, const DropoutArgs& a, unsigned long long* pass, unsigned* ticket, int bump_pass, cudaStream_t s) {
  if (!n) return;
  const int vec = aligned16(x, y) ? 1 : 0;
  DISPATCH_PREC(prec, T, (launch_pdl(dropout_fwd_kernel<T>, dim3(ew_blocks((n + 16 / sizeof(T) - 1) / (16 / sizeof(T)))), dim3(256), (size_t)0, s,
                                     (const T*)x, (T*)y, mask, n, vec, a, pass, ticket, bump_pass))); LAUNCHED();
}
void k_dropout_bwd(int prec, const void* eo, void* ei, const uint32_t* mask, size_t n, float scale, cudaStream_t s) {
  if (!n) return;
  const int vec = aligned16(eo, ei) ? 1 : 0;
  DISPATCH_PREC(prec, T, (launch_pdl(dropout_bwd_kernel<T>, dim3(ew_blocks((n + 16 / sizeof(T) - 1) / (16 / sizeof(T)))), dim3(256), (size_t)0, s,
                                     (const T*)eo, (T*)ei, mask, n, scale, vec))); LAUNCHED();
}

}  // namespace b2g
