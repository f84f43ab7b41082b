// kernels_graph.cu -- the skip-connection vertices of a spine-plus-skip ComputationGraph (B2G_LAYER_ELEMENTWISE / B2G_LAYER_MERGE; semantics
// at b2g_elementwise_op in include/b200gan.h): ElementWiseVertex forward and backward, MergeVertex's NHWC channel concat and its split, and
// the add of a skip source's fp32 gradient accumulator into the spine epsilon.
//
// All of them are memory-bound streams.  Thread t of a one-wave grid takes the 16-byte chunks j = t, t + threads, ... (V = 16 / sizeof(T)
// elements each).  VEC: 16-byte loads and stores of the chunks (every operand aligned, and for the concat every channel slice a whole number
// of chunks); the scalar instantiation visits the same elements element by element.  Every element's arithmetic is the same fp32 expression on
// both paths, so the bits do not depend on the path.
#include <algorithm>

#include "common.cuh"

namespace b2g {

namespace {

constexpr int GR_THREADS = 256;

// V fp32 values of the accumulator (V = 4 or 8: one or two float4)
template <int V> __device__ __forceinline__ void acc_load(const float* p, float* v) {
#pragma unroll
  for (int k = 0; k < V; k += 4) { const float4 q = *reinterpret_cast<const float4*>(p + k); v[k] = q.x; v[k + 1] = q.y; v[k + 2] = q.z; v[k + 3] = q.w; }
}
template <int V> __device__ __forceinline__ void acc_store(float* p, const float* v) {
#pragma unroll
  for (int k = 0; k < V; k += 4) *reinterpret_cast<float4*>(p + k) = make_float4(v[k], v[k + 1], v[k + 2], v[k + 3]);
}

template <int V, bool VEC>
__device__ __forceinline__ void ld_acc(const float* p, size_t e, size_t n, float* v) {
  if (VEC && e + V <= n) { acc_load<V>(p + e, v); return; }
#pragma unroll
  for (int k = 0; k < V; ++k) v[k] = e + k < n ? p[e + k] : 0.f;
}
template <int V, bool VEC>
__device__ __forceinline__ void st_acc(float* p, size_t e, size_t n, const float* v) {
  if (VEC && e + V <= n) { acc_store<V>(p + e, v); return; }
#pragma unroll
  for (int k = 0; k < V; ++k) if (e + k < n) p[e + k] = v[k];
}

// ElementWiseVertex.Op on the inputs (a, b) in the vertex's input order, in fp32
template <int OP> __device__ __forceinline__ float ew_fwd(float a, float b) {
  if (OP == VERTEX_ADD) return a + b;
  if (OP == VERTEX_SUBTRACT) return a - b;
  if (OP == VERTEX_PRODUCT) return a * b;
  if (OP == VERTEX_AVERAGE) return (a + b) * 0.5f;
  return a >= b ? a : b;                       // MAX: a tie takes the first input
}
// dL/da, dL/db from eps
template <int OP> __device__ __forceinline__ void ew_bwd(float e, float a, float b, float* da, float* db) {
  if (OP == VERTEX_ADD) { *da = e; *db = e; }
  else if (OP == VERTEX_SUBTRACT) { *da = e; *db = -e; }
  else if (OP == VERTEX_PRODUCT) { *da = __fmul_rn(e, b); *db = __fmul_rn(e, a); }   // rounded before an accumulate adds it: no FMA contraction
  else if (OP == VERTEX_AVERAGE) { *da = e * 0.5f; *db = e * 0.5f; }
  else { const bool first = a >= b; *da = first ? e : 0.f; *db = first ? 0.f : e; }
}

template <typename T, int OP, bool VEC>
__global__ void __launch_bounds__(GR_THREADS) vertex_ew_fwd_kernel(const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ y, size_t n) {
  pdl_enter();
  constexpr int V = GVec<T>::V;
  const size_t chunks = (n + V - 1) / V;
  for (size_t j = (size_t)blockIdx.x * GR_THREADS + threadIdx.x; j < chunks; j += (size_t)gridDim.x * GR_THREADS) {
    float va[V], vb[V], vy[V];
    ld_chunk<T, VEC>(a, j * V, n, va); ld_chunk<T, VEC>(b, j * V, n, vb);
#pragma unroll
    for (int k = 0; k < V; ++k) vy[k] = ew_fwd<OP>(va[k], vb[k]);
    st_chunk<T, VEC>(y, j * V, n, vy);
  }
}

// spine = the spine input's forward values, skip = the skip input's; order 0: (a, b) = (spine, skip), 1: (skip, spine).  eps (the epsilon w.r.t.
// the vertex output) becomes the spine's share in place -- not rewritten where that share is eps itself (ADD, and SUBTRACT in order 0); the
// skip's share is written (accumulate = 0) or added (1) into the fp32 accumulator acc.
template <typename T, int OP, bool VEC>
__global__ void __launch_bounds__(GR_THREADS) vertex_ew_bwd_kernel(T* __restrict__ eps, const T* __restrict__ spine, const T* __restrict__ skip,
                                                                   float* __restrict__ acc, size_t n, int order, int accumulate) {
  pdl_enter();
  constexpr int V = GVec<T>::V;
  const bool write_spine = !(OP == VERTEX_ADD || (OP == VERTEX_SUBTRACT && order == 0));
  const bool need_x = OP == VERTEX_PRODUCT || OP == VERTEX_MAX;
  const size_t chunks = (n + V - 1) / V;
  for (size_t j = (size_t)blockIdx.x * GR_THREADS + threadIdx.x; j < chunks; j += (size_t)gridDim.x * GR_THREADS) {
    const size_t e0 = j * V;
    float ve[V], vs[V], vk[V], va[V];
    ld_chunk<T, VEC>(eps, e0, n, ve);
    if (need_x) { ld_chunk<T, VEC>(spine, e0, n, vs); ld_chunk<T, VEC>(skip, e0, n, vk); }
    if (accumulate) ld_acc<V, VEC>(acc, e0, n, va);
#pragma unroll
    for (int k = 0; k < V; ++k) {
      float da, db;
      if (order == 0) ew_bwd<OP>(ve[k], need_x ? vs[k] : 0.f, need_x ? vk[k] : 0.f, &da, &db);
      else ew_bwd<OP>(ve[k], need_x ? vk[k] : 0.f, need_x ? vs[k] : 0.f, &da, &db);
      const float sp = order == 0 ? da : db, sk = order == 0 ? db : da;
      ve[k] = sp; va[k] = accumulate ? va[k] + sk : sk;
    }
    if (write_spine) st_chunk<T, VEC>(eps, e0, n, ve);
    st_acc<V, VEC>(acc, e0, n, va);
  }
}

// MergeVertex: y [P][Ca + Cb] = concat(a [P][Ca], b [P][Cb]) along the channels (a, b in the vertex's input order).  VEC: Ca and Cb are whole
// chunks, so every output chunk comes from one input.
template <typename T, bool VEC>
__global__ void __launch_bounds__(GR_THREADS) merge_fwd_kernel(const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ y, size_t P, int Ca, int Cb) {
  pdl_enter();
  constexpr int V = GVec<T>::V;
  const int Ct = Ca + Cb; const size_t n = P * Ct, chunks = (n + V - 1) / V;
  for (size_t j = (size_t)blockIdx.x * GR_THREADS + threadIdx.x; j < chunks; j += (size_t)gridDim.x * GR_THREADS) {
    const size_t e0 = j * V;
    if (VEC) {
      const size_t p = e0 / Ct; const int c = (int)(e0 - p * Ct);
      float v[V];
      if (c < Ca) GVec<T>::load(a + p * Ca + c, v); else GVec<T>::load(b + p * Cb + (c - Ca), v);
      GVec<T>::store(y + e0, v);
    } else {
      for (size_t e = e0; e < e0 + V && e < n; ++e) {
        const size_t p = e / Ct; const int c = (int)(e - p * Ct);
        y[e] = c < Ca ? a[p * Ca + c] : b[p * Cb + (c - Ca)];
      }
    }
  }
}

// MergeVertex backward: eps [P][Ca + Cb] -> the spine's channel slice into dst [P][Cs] (T, a copy) and the skip's into acc [P][Ck] (fp32,
// written or added).  spine_first: the spine is the first input (order 0).
template <typename T, bool VEC>
__global__ void __launch_bounds__(GR_THREADS) merge_bwd_kernel(const T* __restrict__ eps, T* __restrict__ dst, float* __restrict__ acc, size_t P, int Ca, int Cb,
                                                               int spine_first, int accumulate) {
  pdl_enter();
  constexpr int V = GVec<T>::V;
  const int Ct = Ca + Cb; const size_t n = P * Ct, chunks = (n + V - 1) / V;
  const int Cs = spine_first ? Ca : Cb, Ck = spine_first ? Cb : Ca;
  for (size_t j = (size_t)blockIdx.x * GR_THREADS + threadIdx.x; j < chunks; j += (size_t)gridDim.x * GR_THREADS) {
    const size_t e0 = j * V;
    if (VEC) {
      const size_t p = e0 / Ct; const int c = (int)(e0 - p * Ct);
      const bool first = c < Ca; const int cc = first ? c : c - Ca;
      if (first == (spine_first != 0)) *reinterpret_cast<uint4*>(dst + p * Cs + cc) = *reinterpret_cast<const uint4*>(eps + e0);
      else {
        float v[V], w[V]; GVec<T>::load(eps + e0, v);
        float* q = acc + p * Ck + cc;
        if (accumulate) { acc_load<V>(q, w);
#pragma unroll
          for (int k = 0; k < V; ++k) v[k] = w[k] + v[k]; }
        acc_store<V>(q, v);
      }
    } else {
      for (size_t e = e0; e < e0 + V && e < n; ++e) {
        const size_t p = e / Ct; const int c = (int)(e - p * Ct);
        const bool first = c < Ca; const int cc = first ? c : c - Ca;
        if (first == (spine_first != 0)) dst[p * Cs + cc] = eps[e];
        else { float* q = acc + p * Ck + cc; const float v = ldf(eps, e); *q = accumulate ? *q + v : v; }
      }
    }
  }
}

// eps = eps + acc (fp32, rounded once to T) at a skip source
template <typename T, bool VEC>
__global__ void __launch_bounds__(GR_THREADS) skip_add_kernel(T* __restrict__ eps, const float* __restrict__ acc, size_t n) {
  pdl_enter();
  constexpr int V = GVec<T>::V;
  const size_t chunks = (n + V - 1) / V;
  for (size_t j = (size_t)blockIdx.x * GR_THREADS + threadIdx.x; j < chunks; j += (size_t)gridDim.x * GR_THREADS) {
    float ve[V], va[V];
    ld_chunk<T, VEC>(eps, j * V, n, ve); ld_acc<V, VEC>(acc, j * V, n, va);
#pragma unroll
    for (int k = 0; k < V; ++k) ve[k] = ve[k] + va[k];
    st_chunk<T, VEC>(eps, j * V, n, ve);
  }
}

inline bool al16(const void* p) { return (uintptr_t)p % 16 == 0; }
// one wave of 256-thread blocks (pdl_enter lets the successor in at once)
inline dim3 grid_for(size_t chunks) {
  const size_t b = (chunks + GR_THREADS - 1) / GR_THREADS, cap = (size_t)device_sm_count() * 8;
  return dim3((unsigned)std::max<size_t>(1, std::min(b, cap)));
}

#define DISPATCH_VERTEX_OP(op, OPC, ...)                                  \
  switch (op) {                                                           \
    case VERTEX_ADD: { constexpr int OPC = VERTEX_ADD; __VA_ARGS__; } break;           \
    case VERTEX_SUBTRACT: { constexpr int OPC = VERTEX_SUBTRACT; __VA_ARGS__; } break; \
    case VERTEX_PRODUCT: { constexpr int OPC = VERTEX_PRODUCT; __VA_ARGS__; } break;   \
    case VERTEX_AVERAGE: { constexpr int OPC = VERTEX_AVERAGE; __VA_ARGS__; } break;   \
    default: { constexpr int OPC = VERTEX_MAX; __VA_ARGS__; } break;                   \
  }

}  // namespace

void k_vertex_ew_fwd(int prec, int op, const void* a, const void* b, void* y, size_t n, cudaStream_t s) {
  const bool vec = al16(a) && al16(b) && al16(y);
  const size_t V = prec == PREC_F32 ? 4 : 8; const dim3 grid = grid_for((n + V - 1) / V);
  DISPATCH_PREC(prec, T, DISPATCH_VERTEX_OP(op, OPC, {
    if (vec) launch_pdl(vertex_ew_fwd_kernel<T, OPC, true>, grid, dim3(GR_THREADS), (size_t)0, s, (const T*)a, (const T*)b, (T*)y, n);
    else launch_pdl(vertex_ew_fwd_kernel<T, OPC, false>, grid, dim3(GR_THREADS), (size_t)0, s, (const T*)a, (const T*)b, (T*)y, n);
  }));
  LAUNCHED();
  g_ew_last_kernel = vec ? "vertex_ew_fwd_kernel<vec>" : "vertex_ew_fwd_kernel<scalar>";
}

void k_vertex_ew_bwd(int prec, int op, int order, void* eps, const void* spine, const void* skip, float* acc, int accumulate, size_t n, cudaStream_t s) {
  const bool vec = al16(eps) && al16(spine) && al16(skip) && al16(acc);
  const size_t V = prec == PREC_F32 ? 4 : 8; const dim3 grid = grid_for((n + V - 1) / V);
  DISPATCH_PREC(prec, T, DISPATCH_VERTEX_OP(op, OPC, {
    if (vec) launch_pdl(vertex_ew_bwd_kernel<T, OPC, true>, grid, dim3(GR_THREADS), (size_t)0, s, (T*)eps, (const T*)spine, (const T*)skip, acc, n, order, accumulate);
    else launch_pdl(vertex_ew_bwd_kernel<T, OPC, false>, grid, dim3(GR_THREADS), (size_t)0, s, (T*)eps, (const T*)spine, (const T*)skip, acc, n, order, accumulate);
  }));
  LAUNCHED();
  g_ew_last_kernel = vec ? "vertex_ew_bwd_kernel<vec>" : "vertex_ew_bwd_kernel<scalar>";
}

void k_merge_fwd(int prec, const void* a, const void* b, void* y, size_t P, int Ca, int Cb, cudaStream_t s) {
  const int V = prec == PREC_F32 ? 4 : 8;
  const bool vec = al16(a) && al16(b) && al16(y) && Ca % V == 0 && Cb % V == 0;
  const dim3 grid = grid_for((P * (Ca + Cb) + V - 1) / V);
  DISPATCH_PREC(prec, T, {
    if (vec) launch_pdl(merge_fwd_kernel<T, true>, grid, dim3(GR_THREADS), (size_t)0, s, (const T*)a, (const T*)b, (T*)y, P, Ca, Cb);
    else launch_pdl(merge_fwd_kernel<T, false>, grid, dim3(GR_THREADS), (size_t)0, s, (const T*)a, (const T*)b, (T*)y, P, Ca, Cb);
  });
  LAUNCHED();
  g_ew_last_kernel = vec ? "merge_fwd_kernel<vec>" : "merge_fwd_kernel<scalar>";
}

void k_merge_bwd(int prec, const void* eps, void* dst, float* acc, size_t P, int Ca, int Cb, int spine_first, int accumulate, cudaStream_t s) {
  const int V = prec == PREC_F32 ? 4 : 8;
  const bool vec = al16(eps) && al16(dst) && al16(acc) && Ca % V == 0 && Cb % V == 0;
  const dim3 grid = grid_for((P * (Ca + Cb) + V - 1) / V);
  DISPATCH_PREC(prec, T, {
    if (vec) launch_pdl(merge_bwd_kernel<T, true>, grid, dim3(GR_THREADS), (size_t)0, s, (const T*)eps, (T*)dst, acc, P, Ca, Cb, spine_first, accumulate);
    else launch_pdl(merge_bwd_kernel<T, false>, grid, dim3(GR_THREADS), (size_t)0, s, (const T*)eps, (T*)dst, acc, P, Ca, Cb, spine_first, accumulate);
  });
  LAUNCHED();
  g_ew_last_kernel = vec ? "merge_bwd_kernel<vec>" : "merge_bwd_kernel<scalar>";
}

void k_skip_add(int prec, void* eps, const float* acc, size_t n, cudaStream_t s) {
  const bool vec = al16(eps) && al16(acc);
  const size_t V = prec == PREC_F32 ? 4 : 8; const dim3 grid = grid_for((n + V - 1) / V);
  DISPATCH_PREC(prec, T, {
    if (vec) launch_pdl(skip_add_kernel<T, true>, grid, dim3(GR_THREADS), (size_t)0, s, (T*)eps, acc, n);
    else launch_pdl(skip_add_kernel<T, false>, grid, dim3(GR_THREADS), (size_t)0, s, (T*)eps, acc, n);
  });
  LAUNCHED();
  g_ew_last_kernel = vec ? "skip_add_kernel<vec>" : "skip_add_kernel<scalar>";
}

}  // namespace b2g
