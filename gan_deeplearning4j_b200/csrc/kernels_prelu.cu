// kernels_prelu.cu -- DL4J's PReLULayer (B2G_LAYER_PRELU; semantics and the slope gradient's summation order at B2G_LAYER_PRELU in
// include/b200gan.h): the forward, and a backward that writes the input gradient in place and the slope gradient's per-row-group partial sums,
// which the pass's reduce-list launch (kernels_ew.cu reduce_multi_kernel) folds into dalpha.
//
// Both kernels are memory-bound streams over the NHWC map.  Element j of a row (j = (h*W + w)*C + c) reads slope k(j) of alpha, stored in DL4J's
// [C][H][W] order with the shared axes of extent 1, and belongs to position s(j) among the positions sharing that slope.  VEC: 16-byte loads and
// stores of V = 16 / sizeof(T) consecutive elements (a row is a whole number of chunks and every operand is aligned); the scalar instantiation
// visits the same elements one by one.  Every element's arithmetic is the same fp32 expression on both paths, and the slope partials are summed
// over the same rows in the same order, so the bits do not depend on the path.
#include <algorithm>

#include "common.cuh"

namespace b2g {

namespace {

constexpr int PR_THREADS = 256;
constexpr int PR_ROW_ELEMS = 2048;      // row elements per block of the backward's group sizing (a constant: the order is fixed by the shape)
constexpr int PR_TARGET_BLOCKS = 1024, PR_MAX_GROUPS = 64;

// The position (c, h, w) of row element j (a row holds fewer than 2^31 elements: 32-bit arithmetic), found once per chunk and then advanced
// element by element; past the row's last element it wraps to the next row's first.
struct PreluPos { int c, h, w; };
__device__ __forceinline__ PreluPos prelu_pos(const PreluGeom& g, int j) { const int pix = j / g.C; return PreluPos{j - pix * g.C, pix / g.W, pix % g.W}; }
__device__ __forceinline__ void prelu_next(const PreluGeom& g, PreluPos& p) {
  if (++p.c == g.C) { p.c = 0; if (++p.w == g.W) { p.w = 0; if (++p.h == g.H) p.h = 0; } }
}
// slope k and sharing position s of the element at p
__device__ __forceinline__ int prelu_k(const PreluGeom& g, const PreluPos& p) {
  const bool cs = g.shared & 1, hs = g.shared & 2, ws = g.shared & 4;
  return ((cs ? 0 : p.c) * (hs ? 1 : g.H) + (hs ? 0 : p.h)) * (ws ? 1 : g.W) + (ws ? 0 : p.w);
}
__device__ __forceinline__ int prelu_s(const PreluGeom& g, const PreluPos& p) {
  const bool cs = g.shared & 1, hs = g.shared & 2, ws = g.shared & 4;
  return ((cs ? p.c : 0) * (hs ? g.H : 1) + (hs ? p.h : 0)) * (ws ? g.W : 1) + (ws ? p.w : 0);
}

template <typename T, bool VEC>
__global__ void __launch_bounds__(PR_THREADS) prelu_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, const float* __restrict__ alpha, size_t n,
                                                               PreluGeom g) {
  pdl_enter();
  constexpr int V = GVec<T>::V;
  const size_t M = (size_t)g.H * g.W * g.C, chunks = (n + V - 1) / V, stride = (size_t)gridDim.x * PR_THREADS;
  size_t j = (size_t)blockIdx.x * PR_THREADS + threadIdx.x;
  // the row position of the chunk's first element, advanced by the grid stride without a division per chunk (the grid is one wave, so its
  // first chunk and its stride are below 2^32 elements)
  long long jr = (unsigned)(j * V) % (unsigned)M;
  const long long step = (unsigned)(stride * V) % (unsigned)M;
  for (; j < chunks; j += stride) {
    float v[V];
    ld_chunk<T, VEC>(x, j * V, n, v);
    PreluPos p = prelu_pos(g, (int)jr);
#pragma unroll
    for (int q = 0; q < V; ++q) {
      if (v[q] < 0.f) v[q] = alpha[prelu_k(g, p)] * v[q];        // -0.0 and NaN are not negative: they pass
      prelu_next(g, p);
    }
    st_chunk<T, VEC>(y, j * V, n, v);
    jr += step; if (jr >= (long long)M) jr -= (long long)M;
  }
}

// Block (bx, grp): thread t takes the chunk of V elements at row position (bx * PR_THREADS + t) * V in every row of group grp, rows ascending.
template <typename T, bool VEC>
__global__ void __launch_bounds__(PR_THREADS) prelu_bwd_kernel(const T* __restrict__ x, T* __restrict__ eps, const float* __restrict__ alpha,
                                                               float* __restrict__ part, int write_dx, int rows, int rpg, PreluGeom g) {
  pdl_enter();
  constexpr int V = GVec<T>::V;
  const size_t M = (size_t)g.H * g.W * g.C, j0 = ((size_t)blockIdx.x * PR_THREADS + threadIdx.x) * V;
  if (j0 >= M) return;
  const int grp = blockIdx.y, r0 = grp * rpg, r1 = min(rows, r0 + rpg);
  int k[V], sp[V];
  PreluPos p = prelu_pos(g, (int)j0);
#pragma unroll
  for (int q = 0; q < V; ++q) { k[q] = prelu_k(g, p); sp[q] = prelu_s(g, p); prelu_next(g, p); }
  float acc[V];
#pragma unroll
  for (int q = 0; q < V; ++q) acc[q] = 0.f;
  for (int r = r0; r < r1; ++r) {
    const size_t e0 = (size_t)r * M + j0, end = (size_t)(r + 1) * M;
    float vx[V], ve[V];
    ld_chunk<T, VEC>(x, e0, end, vx); ld_chunk<T, VEC>(eps, e0, end, ve);
#pragma unroll
    for (int q = 0; q < V; ++q)
      if (vx[q] < 0.f) { acc[q] = acc[q] + __fmul_rn(vx[q], ve[q]); ve[q] = alpha[k[q]] * ve[q]; }
    if (write_dx) st_chunk<T, VEC>(eps, e0, end, ve);
  }
  if (part) {
    const long long K = (long long)prelu_slopes(g), S = (long long)M / K;
#pragma unroll
    for (int q = 0; q < V; ++q) if (j0 + q < M) part[((long long)grp * S + sp[q]) * K + k[q]] = acc[q];
  }
}

inline bool al16(const void* p) { return (uintptr_t)p % 16 == 0; }
inline size_t row_elems(const PreluGeom& g) { return (size_t)g.H * g.W * g.C; }

}  // namespace

// the group count a pass of many rows aims at
static int prelu_group_target(const PreluGeom& g) {
  const size_t bx = (row_elems(g) + PR_ROW_ELEMS - 1) / PR_ROW_ELEMS;
  return (int)std::max<size_t>(1, std::min<size_t>(PR_MAX_GROUPS, PR_TARGET_BLOCKS / bx));
}

void prelu_row_groups(int rows, const PreluGeom& g, int* groups, int* rows_per_group) {
  const int g0 = std::max(1, std::min(rows, prelu_group_target(g)));
  const int rpg = (rows + g0 - 1) / g0;
  *rows_per_group = rpg; *groups = (rows + rpg - 1) / rpg;
}

// G(rows) <= min(rows, want) but is not monotone in rows (65 rows make 33 groups of 2, 64 rows 64 groups of 1): the buffer holds
// min(max_rows, want) groups, the bound for every pass of 1 ... max_rows rows
size_t k_prelu_part_floats(int max_rows, const PreluGeom& g) {
  return (size_t)std::max(1, std::min(max_rows, prelu_group_target(g))) * row_elems(g);
}

void k_prelu_fwd(int prec, const void* x, void* y, const float* alpha, int rows, const PreluGeom& g, cudaStream_t s) {
  const size_t n = (size_t)rows * row_elems(g);
  const int V = prec == PREC_F32 ? 4 : 8;
  const bool vec = al16(x) && al16(y) && row_elems(g) % V == 0;
  const size_t chunks = (n + V - 1) / V, cap = (size_t)device_sm_count() * 8;
  const dim3 grid((unsigned)std::max<size_t>(1, std::min((chunks + PR_THREADS - 1) / PR_THREADS, cap)));
  DISPATCH_PREC(prec, T, {
    if (vec) launch_pdl(prelu_fwd_kernel<T, true>, grid, dim3(PR_THREADS), (size_t)0, s, (const T*)x, (T*)y, alpha, n, g);
    else launch_pdl(prelu_fwd_kernel<T, false>, grid, dim3(PR_THREADS), (size_t)0, s, (const T*)x, (T*)y, alpha, n, g);
  });
  LAUNCHED();
  g_ew_last_kernel = vec ? "prelu_fwd_kernel<vec>" : "prelu_fwd_kernel<scalar>";
}

void k_prelu_bwd(int prec, const void* x, void* eps, const float* alpha, float* part, int write_dx, int rows, const PreluGeom& g, cudaStream_t s) {
  const int V = prec == PREC_F32 ? 4 : 8;
  const bool vec = al16(x) && al16(eps) && row_elems(g) % V == 0;
  int G, rpg; prelu_row_groups(rows, g, &G, &rpg);
  const dim3 grid((unsigned)((row_elems(g) + (size_t)V * PR_THREADS - 1) / ((size_t)V * PR_THREADS)), (unsigned)G);
  DISPATCH_PREC(prec, T, {
    if (vec) launch_pdl(prelu_bwd_kernel<T, true>, grid, dim3(PR_THREADS), (size_t)0, s, (const T*)x, (T*)eps, alpha, part, write_dx, rows, rpg, g);
    else launch_pdl(prelu_bwd_kernel<T, false>, grid, dim3(PR_THREADS), (size_t)0, s, (const T*)x, (T*)eps, alpha, part, write_dx, rows, rpg, g);
  });
  LAUNCHED();
  g_ew_last_kernel = vec ? "prelu_bwd_kernel<vec>" : "prelu_bwd_kernel<scalar>";
}

void prelu_queue_reduce(ReduceList* rl, const float* part, float* dalpha, int rows, const PreluGeom& g) {
  int G, rpg; prelu_row_groups(rows, g, &G, &rpg);
  const int64_t K = (int64_t)prelu_slopes(g), S = (int64_t)(row_elems(g) / (size_t)K);
  reduce_list_push(rl, part, dalpha, K, (int)(G * S), K);
}

}  // namespace b2g
