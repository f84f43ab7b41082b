// kernels_dropout.cu -- DropoutLayer (DL4J 1.0.0-beta3 inverted dropout): the masked forward with its on-device Philox4x32-10 mask and
// pass counter, and the backward that applies the stored mask.  Mask definition: include/b200gan.h (B2G_LAYER_DROPOUT); oracle restatement:
// tests/dropout_ref.py dropout_mask.  Below them, the other IDropout kinds of a DropoutLayer (GaussianDropout, GaussianNoise, AlphaDropout,
// SpatialDropout; include/b200gan.h b2g_dropout_kind) from the same Philox stream and pass counter.
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

// ---- GaussianDropout, GaussianNoise, AlphaDropout, SpatialDropout, and scheduled Dropout (b2g_dropout_kind) ---------------------------------
// The vector loops take one 16-byte vector per thread and iteration: one Philox call per 4 elements and one Box-Muller per 2.  The tails run
// one element per thread.  The per-element masks are written the way dropout_fwd_kernel writes them (a warp assembles whole words).

__device__ __forceinline__ float normal1(const Philox4& r, unsigned j) {
  float ze, zo; box_muller(pick4(r, j & 2u), pick4(r, (j & 2u) + 1u), ze, zo);
  return (j & 1u) ? zo : ze;
}
// GaussianNoise: y = x + sigma z;  GaussianDropout: y = x * m, m = 1 + sigma z (also its backward, with x = dy)
template <int K> __device__ __forceinline__ float gauss_apply(float x, float z, float sigma) {
  if (K == DROP_GAUSSIAN_NOISE) return fmaf(sigma, z, x);
  return x * fmaf(sigma, z, 1.0f);
}
// the pass counter bump of dropout_fwd_kernel: the last block to finish advances *pass
__device__ __forceinline__ void bump_pass_counter(unsigned long long* pass, unsigned* ticket, unsigned long long P) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned done = atomicAdd(ticket, 1u);
    if (done == gridDim.x - 1) { *pass = P + 1; *ticket = 0u; __threadfence(); }
  }
}
// A scheduled layer's constants (NoiseSched): the forward evaluates the schedule, clamps the value and records it; the backward reads the record
template <int K> __device__ __forceinline__ void scheduled_args(NoiseArgs& a, const NoiseSched& q, NoiseRec* rec, int bwd) {
  if (!q.sched) return;
  const float v = bwd ? rec->v : noise_clamp(K, sched_lr(*q.sched, a.value, *q.step, (long long)*q.epoch));
  noise_derive(K, v, a);
  if (!bwd && blockIdx.x == 0 && threadIdx.x == 0) rec->v = v;
}

// Forward of GaussianNoise / GaussianDropout and GaussianDropout's backward (bwd = 1: P and the value from *rec, no bump)
template <typename T, int K>
__global__ void __launch_bounds__(256) gauss_kernel(const T* x, T* y, size_t n, int vec, NoiseArgs a, const NoiseSched q, unsigned long long* pass,
                                                    NoiseRec* rec, unsigned* ticket, int bump, int bwd) { pdl_enter();
  constexpr int V = 16 / sizeof(T);
  const unsigned long long P = bwd ? rec->P : *(volatile unsigned long long*)pass;
  scheduled_args<K>(a, q, rec, bwd);
  const uint32_t c1 = (uint32_t)P, c2 = (uint32_t)(P >> 32), k0 = (uint32_t)a.seed, k1 = (uint32_t)(a.seed >> 32);
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
  if (!bwd && tid == 0) rec->P = P;
  const size_t nv = vec ? n / V : 0;
  for (size_t i = tid; i < nv; i += stride) {
    const size_t e0 = i * V;
    float v[V]; ld16(x + e0, v);
#pragma unroll
    for (int h = 0; h < V / 4; ++h) {
      float z[4]; normals4(philox4x32_10((uint32_t)(e0 >> 2) + h, c1, c2, a.tag, k0, k1), z);
#pragma unroll
      for (int j = 0; j < 4; ++j) v[4 * h + j] = gauss_apply<K>(v[4 * h + j], z[j], a.scale);
    }
    st16(y + e0, v);
  }
  for (size_t e = nv * V + tid; e < n; e += stride)
    stf(y, e, gauss_apply<K>(ldf(x, e), normal1(philox4x32_10((uint32_t)(e >> 2), c1, c2, a.tag, k0, k1), (unsigned)(e & 3)), a.scale));
  if (bump) bump_pass_counter(pass, ticket, P);
}

// Per-element Bernoulli forward: Dropout's y = keep ? x * (1/p) : 0 (scheduled Dropout) or AlphaDropout's y = fmaf(a, keep ? x : a', b), the
// keep bits into mask as dropout_fwd_kernel writes them
template <int K> __device__ __forceinline__ float bern_apply(float x, bool keep, const NoiseArgs& a) {
  if (K == DROP_ALPHA) return fmaf(a.scale, keep ? x : a.fill, a.shift);
  return keep ? x * a.scale : 0.f;
}
template <typename T, int K>
__global__ void __launch_bounds__(256) bern_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, uint32_t* __restrict__ mask, size_t n, int vec,
                                                       NoiseArgs a, const NoiseSched q, NoiseRec* rec, unsigned long long* pass, unsigned* ticket, int bump) { pdl_enter();
  constexpr int V = 16 / sizeof(T);
  const unsigned long long P = *(volatile unsigned long long*)pass;
  scheduled_args<K>(a, q, rec, 0);
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
      for (int j = 0; j < 4; ++j) {
        const bool keep = a.keep_all || r.x[j] < a.threshold;
        bits |= (uint32_t)keep << (4 * h + j); v[4 * h + j] = bern_apply<K>(v[4 * h + j], keep, a);
      }
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
      stf(y, e, bern_apply<K>(ldf(x, e), keep, a));
    }
    const uint32_t w = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) mask[base >> 5] = w;
  }
  if (bump) bump_pass_counter(pass, ticket, P);
}

// SpatialDropout: one keep bit per (row, channel), j = row * C + c.  The forward writes the R*C-bit mask (one word per thread and iteration,
// 8 Philox calls) and applies the keep bits to the elements, drawing them again per element (one Philox call per 4 consecutive j).
// (row, pixel, channel) of a vector's first element is divided out once and then stepped.
struct SpatialPos {
  size_t row; int pix, c;
  __device__ __forceinline__ SpatialPos(size_t e, int hw, int C) { const size_t per = (size_t)hw * C, q = e % per; row = e / per; pix = (int)(q / C); c = (int)(q % C); }
  __device__ __forceinline__ size_t j(int C) const { return row * C + c; }
  __device__ __forceinline__ void next(int hw, int C) { if (++c == C) { c = 0; if (++pix == hw) { pix = 0; ++row; } } }
};
template <typename T>
__global__ void __launch_bounds__(256) spatial_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, uint32_t* __restrict__ mask, size_t n, int vec,
                                                          NoiseArgs a, const NoiseSched q, NoiseRec* rec, unsigned long long* pass, unsigned* ticket, int bump) { pdl_enter();
  constexpr int V = 16 / sizeof(T);
  const unsigned long long P = *(volatile unsigned long long*)pass;
  scheduled_args<DROP_SPATIAL>(a, q, rec, 0);
  const uint32_t c1 = (uint32_t)P, c2 = (uint32_t)(P >> 32), k0 = (uint32_t)a.seed, k1 = (uint32_t)(a.seed >> 32);
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
  const size_t nj = n / ((size_t)a.hw * a.C) * a.C, nwords = (nj + 31) / 32;
  for (size_t wd = tid; wd < nwords; wd += stride) {
    uint32_t w = 0;
#pragma unroll
    for (int h = 0; h < 8; ++h) {
      const size_t g = wd * 8 + h;
      if (4 * g >= nj) break;
      const Philox4 r = philox4x32_10((uint32_t)g, c1, c2, a.tag, k0, k1);
#pragma unroll
      for (int j = 0; j < 4; ++j) w |= (uint32_t)(a.keep_all || r.x[j] < a.threshold) << (4 * h + j);
    }
    if (nj - wd * 32 < 32) w &= (1u << (nj - wd * 32)) - 1u;
    mask[wd] = w;
  }
  const size_t nv = vec ? n / V : 0;
  for (size_t i = tid; i < nv; i += stride) {
    const size_t e0 = i * V;
    float v[V]; ld16(x + e0, v);
    SpatialPos sp(e0, a.hw, a.C);
    size_t g = ~(size_t)0; Philox4 r{};
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const size_t j = sp.j(a.C);
      if ((j >> 2) != g) { g = j >> 2; r = philox4x32_10((uint32_t)g, c1, c2, a.tag, k0, k1); }
      const bool keep = a.keep_all || pick4(r, (unsigned)(j & 3)) < a.threshold;
      v[k] = keep ? v[k] * a.scale : 0.f;
      sp.next(a.hw, a.C);
    }
    st16(y + e0, v);
  }
  for (size_t e = nv * V + tid; e < n; e += stride) {
    const size_t j = SpatialPos(e, a.hw, a.C).j(a.C);
    const bool keep = a.keep_all || pick4(philox4x32_10((uint32_t)(j >> 2), c1, c2, a.tag, k0, k1), (unsigned)(j & 3)) < a.threshold;
    stf(y, e, keep ? ldf(x, e) * a.scale : 0.f);
  }
  if (bump) bump_pass_counter(pass, ticket, P);
}
// Backward of the mask kinds: dx = dy * scale where the forward kept, 0 elsewhere (scale: 1/p, AlphaDropout's a); mask bit j = e, or
// j = row * C + c for SpatialDropout
template <typename T, int K>
__global__ void __launch_bounds__(256) mask_bwd_kernel(const T* eo, T* ei, const uint32_t* __restrict__ mask, size_t n, int vec, NoiseArgs a,
                                                       const NoiseSched q, NoiseRec* rec) { pdl_enter();
  constexpr int V = 16 / sizeof(T);
  scheduled_args<K>(a, q, rec, 1);
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
  const size_t nv = vec ? n / V : 0;
  for (size_t i = tid; i < nv; i += stride) {
    const size_t e0 = i * V;
    float v[V]; ld16(eo + e0, v);
    if (K == DROP_SPATIAL) {
      SpatialPos sp(e0, a.hw, a.C);
#pragma unroll
      for (int k = 0; k < V; ++k) { const size_t j = sp.j(a.C); v[k] = ((mask[j >> 5] >> (j & 31)) & 1u) ? v[k] * a.scale : 0.f; sp.next(a.hw, a.C); }
    } else {
      const uint32_t bits = mask[e0 >> 5] >> (e0 & 31);
#pragma unroll
      for (int k = 0; k < V; ++k) v[k] = ((bits >> k) & 1u) ? v[k] * a.scale : 0.f;
    }
    st16(ei + e0, v);
  }
  for (size_t e = nv * V + tid; e < n; e += stride) {
    const size_t j = K == DROP_SPATIAL ? SpatialPos(e, a.hw, a.C).j(a.C) : e;
    stf(ei, e, ((mask[j >> 5] >> (j & 31)) & 1u) ? ldf(eo, e) * a.scale : 0.f);
  }
}
__global__ void noise_value_kernel(int kind, float value, const NoiseSched q, float* out) {
  if (threadIdx.x || blockIdx.x) return;
  float v = value;
  if (q.sched) {
    v = sched_lr(*q.sched, value, *q.step, (long long)*q.epoch);
    v = kind == DROP_GAUSSIAN_DROPOUT ? noise_clamp(DROP_GAUSSIAN_DROPOUT, v) : kind == DROP_GAUSSIAN_NOISE ? noise_clamp(DROP_GAUSSIAN_NOISE, v) : noise_clamp(DROP_ALPHA, v);
  }
  *out = v;
}

void k_noise_fwd(int prec, int kind, const void* x, void* y, uint32_t* mask, NoiseRec* rec, size_t n, const NoiseArgs& a, const NoiseSched& q,
                 unsigned long long* pass, unsigned* ticket, int bump_pass, cudaStream_t s) {
  if (!n) return;
  const int vec = aligned16(x, y) ? 1 : 0;
  DISPATCH_PREC(prec, T, {
    const dim3 grid(ew_blocks((n + 16 / sizeof(T) - 1) / (16 / sizeof(T))));
    switch (kind) {
      case DROP_GAUSSIAN_DROPOUT: launch_pdl(gauss_kernel<T, DROP_GAUSSIAN_DROPOUT>, grid, dim3(256), (size_t)0, s, (const T*)x, (T*)y, n, vec, a, q, pass, rec, ticket, bump_pass, 0); break;
      case DROP_GAUSSIAN_NOISE: launch_pdl(gauss_kernel<T, DROP_GAUSSIAN_NOISE>, grid, dim3(256), (size_t)0, s, (const T*)x, (T*)y, n, vec, a, q, pass, rec, ticket, bump_pass, 0); break;
      case DROP_ALPHA: launch_pdl(bern_fwd_kernel<T, DROP_ALPHA>, grid, dim3(256), (size_t)0, s, (const T*)x, (T*)y, mask, n, vec, a, q, rec, pass, ticket, bump_pass); break;
      case DROP_BERNOULLI: launch_pdl(bern_fwd_kernel<T, DROP_BERNOULLI>, grid, dim3(256), (size_t)0, s, (const T*)x, (T*)y, mask, n, vec, a, q, rec, pass, ticket, bump_pass); break;
      default: launch_pdl(spatial_fwd_kernel<T>, grid, dim3(256), (size_t)0, s, (const T*)x, (T*)y, mask, n, vec, a, q, rec, pass, ticket, bump_pass); break;
    }
  }); LAUNCHED();
}
void k_noise_bwd(int prec, int kind, const void* eo, void* ei, const uint32_t* mask, const NoiseRec* rec, size_t n, const NoiseArgs& a, const NoiseSched& q,
                 cudaStream_t s) {
  if (!n || kind == DROP_GAUSSIAN_NOISE) return;
  const int vec = aligned16(eo, ei) ? 1 : 0;
  NoiseRec* r = const_cast<NoiseRec*>(rec);
  DISPATCH_PREC(prec, T, {
    const dim3 grid(ew_blocks((n + 16 / sizeof(T) - 1) / (16 / sizeof(T))));
    switch (kind) {
      case DROP_GAUSSIAN_DROPOUT: launch_pdl(gauss_kernel<T, DROP_GAUSSIAN_DROPOUT>, grid, dim3(256), (size_t)0, s, (const T*)eo, (T*)ei, n, vec, a, q,
                                             (unsigned long long*)nullptr, r, (unsigned*)nullptr, 0, 1); break;
      case DROP_ALPHA: launch_pdl(mask_bwd_kernel<T, DROP_ALPHA>, grid, dim3(256), (size_t)0, s, (const T*)eo, (T*)ei, mask, n, vec, a, q, r); break;
      case DROP_BERNOULLI: launch_pdl(mask_bwd_kernel<T, DROP_BERNOULLI>, grid, dim3(256), (size_t)0, s, (const T*)eo, (T*)ei, mask, n, vec, a, q, r); break;
      default: launch_pdl(mask_bwd_kernel<T, DROP_SPATIAL>, grid, dim3(256), (size_t)0, s, (const T*)eo, (T*)ei, mask, n, vec, a, q, r); break;
    }
  }); LAUNCHED();
}
void k_noise_value(int kind, float value, const NoiseSched& q, float* out, cudaStream_t s) {
  noise_value_kernel<<<1, 32, 0, s>>>(kind, value, q, out); LAUNCHED();
}

// ---- weight noise (DropConnect, WeightNoise; b2g_weight_noise) ------------------------------------------------------------------------
// One launch per train-mode pass over the job table: each block finds its job (the largest blk_begin <= blockIdx.x), each thread draws 4
// consecutive elements with one Philox call (j0 is a multiple of 4, so they share a counter).  Loads are 16-byte where the tensor starts on a
// 16-byte boundary (a conv W follows its nOut biases, so it may not), scalar otherwise.
__global__ void __launch_bounds__(256) weight_noise_kernel(const WnJob* __restrict__ jobs, int njobs, uint64_t seed, int rank, const int* step,
                                                           const int64_t* epoch, unsigned long long* pass, unsigned* ticket, int bump) { pdl_enter();
  const unsigned long long P = *(volatile unsigned long long*)pass;
  int lo = 0, hi = njobs - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (jobs[mid].blk_begin <= (int)blockIdx.x) lo = mid; else hi = mid - 1; }
  const WnJob& jb = jobs[lo];
  __shared__ uint32_t s_threshold; __shared__ int s_keep_all;
  if (jb.kind == WN_DROPCONNECT && threadIdx.x == 0) {        // Dropout's keep rule at p, or at the schedule's clamped value
    NoiseArgs a{};
    noise_derive(DROP_BERNOULLI, jb.sched ? noise_clamp(DROP_BERNOULLI, sched_lr(*jb.sched, jb.p, *step, (long long)*epoch)) : jb.p, a);
    s_threshold = a.threshold; s_keep_all = a.keep_all;
  }
  __syncthreads();
  const int64_t i0 = (int64_t)(blockIdx.x - jb.blk_begin) * WN_CHUNK + 4 * (int64_t)threadIdx.x, n = jb.n;
  if (i0 < n) {
    const Philox4 r = philox4x32_10((uint32_t)((jb.j0 + i0) >> 2), (uint32_t)P, (uint32_t)(P >> 32), (uint32_t)jb.layer | ((uint32_t)rank << 16),
                                    (uint32_t)seed, (uint32_t)(seed >> 32));
    const bool full = i0 + 4 <= n;
    float w[4];
    if (full && (reinterpret_cast<uintptr_t>(jb.src) & 15) == 0) ld16(jb.src + i0, w);
    else {
#pragma unroll
      for (int k = 0; k < 4; ++k) w[k] = i0 + k < n ? jb.src[i0 + k] : 0.f;
    }
    if (jb.kind == WN_DROPCONNECT) {
      const uint32_t thr = s_threshold; const int all = s_keep_all;
#pragma unroll
      for (int k = 0; k < 4; ++k) w[k] = (all || r.x[k] < thr) ? w[k] : 0.f;
    } else {
      float nz[4];
      if (jb.dist == WN_NORMAL) {
        normals4(r, nz);
#pragma unroll
        for (int k = 0; k < 4; ++k) nz[k] = fmaf(jb.b, nz[k], jb.a);
      } else {
        const float span = jb.b - jb.a;
#pragma unroll
        for (int k = 0; k < 4; ++k) nz[k] = fmaf(span, (float)(r.x[k] >> 8) * 0x1p-24f, jb.a);
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) w[k] = jb.additive ? w[k] + nz[k] : w[k] * nz[k];
    }
    if (jb.dst_f32) {
      if (full) st16(jb.dst_f32 + i0, w);
      else for (int k = 0; k < 4 && i0 + k < n; ++k) jb.dst_f32[i0 + k] = w[k];
    } else {
      for (int k = 0; k < 4 && i0 + k < n; ++k) upd_shadow(jb.sg, jb.dst_bf16, i0 + k, __float2bfloat16_rn(w[k]));
    }
  }
  if (bump) bump_pass_counter(pass, ticket, P);
}
void k_weight_noise(const WnJob* jobs, int njobs, int nblocks, uint64_t seed, int rank, const int* step, const int64_t* epoch, unsigned long long* pass,
                    unsigned* ticket, int bump_pass, cudaStream_t s) {
  if (!njobs || !nblocks) return;
  launch_pdl(weight_noise_kernel, dim3(nblocks), dim3(256), (size_t)0, s, jobs, njobs, seed, rank, step, epoch, pass, ticket, bump_pass); LAUNCHED();
}

}  // namespace b2g
