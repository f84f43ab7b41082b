// kernels_cnnloss.cu -- CnnLossLayer's per-pixel losses (B2G_LAYER_CNN_LOSS; semantics in include/b200gan.h): sigmoid XENT over every
// element of an NHWC map, and a softmax MCXENT over the C channels of every pixel.  Codes 2-8 run kernels_ew.cu loss_kernel unchanged.
//
// Both kernels cut each group into k_loss_blocks() slices fixed by the shape (at most LOSS_MAX_GRID = 1024 blocks in all: one wave, so they
// let their successor in at once), sum their scores in double in a fixed order, write one partial per block, and the last block to finish
// (ticket word, 0 between launches) folds each group's partials in slice order, one warp per group, each lane a strided subset in slice order
// and then the warp's xor butterfly.  The loss sums do not depend on the order in which the blocks ran.
#include "common.cuh"

namespace b2g {

namespace {

constexpr int CL_THREADS = 256;

// LossBinaryXENT + sigmoid on one logit: the per-element formulas of kernels_ew.cu xent_kernel (clip > 0 DL4J-exact, 0 BCE-with-logits)
__device__ __forceinline__ float xent_elem(float zi, float yi, float clip, float* grad) {
  const float sg = 1.0f / (1.0f + expf(-zi));
  if (clip > 0.f) {
    const float p = fminf(fmaxf(sg, clip), 1.0f - clip);
    *grad = (p - yi) / (p * (1.0f - p)) * sg * (1.0f - sg);
    return -(yi * logf(p) + (1.0f - yi) * logf(1.0f - p));
  }
  *grad = sg - yi;
  return fmaxf(zi, 0.f) + log1pf(expf(-fabsf(zi))) - yi * zi;
}

// The last block of the launch folds partial[g * bpg + k] in slice order per group g (as kernels_ew.cu loss_kernel does) and resets the ticket.
__device__ __forceinline__ void fold_partials(double tot, int groups, int bpg, float* __restrict__ loss_sums, double* partial, unsigned* ticket) {
  __shared__ int last;
  if (threadIdx.x == 0) {
    partial[blockIdx.x] = tot;
    __threadfence();
    last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();      // every partial is visible: each writer fenced before taking its ticket
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int g = warp; g < groups; g += CL_THREADS / 32) {
    double s = 0.0;
    for (int k = lane; k < bpg; k += 32) s += __ldcg(partial + (size_t)g * bpg + k);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) loss_sums[g] = (float)s;
  }
  if (threadIdx.x == 0) { *ticket = 0u; __threadfence(); }
}

template <typename T> struct Vec;       // one 16-byte chunk of V elements
template <> struct Vec<float> {
  static constexpr int V = 4;
  static __device__ __forceinline__ void load(const float* p, float* v) { const float4 q = *reinterpret_cast<const float4*>(p); v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w; }
  static __device__ __forceinline__ void store(float* p, const float* v) { *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]); }
};
template <> struct Vec<__nv_bfloat16> {
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

// Sigmoid XENT over groups x n elements (z, y, dz [groups][n]).  Thread t of block b of group g owns the chunks j = b*256 + t + k*bpg*256
// (k = 0, 1, ...) of V = 16 / sizeof(T) elements each, [jV, jV + V) clipped to n; its double sum adds the elements' fp32 scores in element
// order, chunk after chunk.  VEC: 16-byte loads and stores of the full chunks (z, y, dz aligned and every group starting aligned); a partial
// chunk, and every chunk of the scalar instantiation, goes element by element in the same order -- the bits do not depend on the path.
// WM: element e (of the whole launch) is scaled by sc = loss_wm_scale(wm, e / C, e % C): its score enters as (double)score * (double)sc and its
// dz is grad * sc, in the same order.
template <typename T, bool VEC, bool WM>
__global__ void __launch_bounds__(CL_THREADS) cnn_xent_kernel(const T* __restrict__ z, const float* __restrict__ y, T* __restrict__ dz,
                                                              float* __restrict__ loss_sums, size_t n, int bpg, float clip, double* partial, unsigned* ticket,
                                                              LossWM wm) {
  pdl_enter();
  __shared__ double red[CL_THREADS / 32];
  constexpr int V = Vec<T>::V;
  const int g = blockIdx.x / bpg, b = blockIdx.x % bpg;
  const size_t base = (size_t)g * n, chunks = (n + V - 1) / V;
  double acc = 0.0;
  for (size_t j = (size_t)b * CL_THREADS + threadIdx.x; j < chunks; j += (size_t)bpg * CL_THREADS) {
    const size_t e0 = j * V;
    if (VEC && e0 + V <= n) {
      float zv[V], yv[V], gv[V];
      Vec<T>::load(z + base + e0, zv);
#pragma unroll
      for (int k = 0; k < V; k += 4) { const float4 q = *reinterpret_cast<const float4*>(y + base + e0 + k); yv[k] = q.x; yv[k + 1] = q.y; yv[k + 2] = q.z; yv[k + 3] = q.w; }
#pragma unroll
      for (int k = 0; k < V; ++k) {
        const float l = xent_elem(zv[k], yv[k], clip, &gv[k]);
        if (WM) { const size_t e = base + e0 + k; const float sc = loss_wm_scale(wm, e / wm.C, (int)(e % wm.C)); acc += __dmul_rn((double)l, (double)sc); gv[k] *= sc; }
        else acc += (double)l;
      }
      Vec<T>::store(dz + base + e0, gv);
    } else {
      const size_t e1 = e0 + V < n ? e0 + V : n;
      for (size_t e = e0; e < e1; ++e) {
        float gr; const float l = xent_elem(ldf(z, base + e), y[base + e], clip, &gr);
        if (WM) { const float sc = loss_wm_scale(wm, (base + e) / wm.C, (int)((base + e) % wm.C)); acc += __dmul_rn((double)l, (double)sc); gr *= sc; }
        else acc += (double)l;
        stf(dz, base + e, gr);
      }
    }
  }
  const double tot = block_sum(acc, red);
  fold_partials(tot, (int)(gridDim.x / bpg), bpg, loss_sums, partial, ticket);
}

// Softmax MCXENT per pixel: z, y, dz, p_out [groups][rows][C] (NHWC pixels).  One thread per pixel, thread t of block b of group g taking
// the pixels r = b*256 + t + k*bpg*256 of its group: m = max over c in channel order; den = sum over c of expf(z - m) in fp32, channel order;
// p_c = expf(z_c - m) / den; dz_c = p_c - y_c; the thread's double sum subtracts y_c * log((double)clamp(p_c, 1e-10, 1 - 1e-10)) channel after
// channel, pixel after pixel.  Without labels (y = null) it writes p_out only and sums nothing.  WM (labels given, a mask per pixel): the
// weighted softmax gradient of kernels_ew.cu softmax_xent_kernel, m_r the mask of pixel g*rows + r.
template <typename T, bool WM>
__global__ void __launch_bounds__(CL_THREADS) cnn_softmax_xent_kernel(const T* __restrict__ z, const float* __restrict__ y, T* __restrict__ dz, T* __restrict__ p_out,
                                                                      float* __restrict__ loss_sums, int rows, int C, int bpg, double* partial, unsigned* ticket,
                                                                      LossWM wm) {
  pdl_enter();
  __shared__ double red[CL_THREADS / 32];
  const int g = blockIdx.x / bpg, b = blockIdx.x % bpg;
  double acc = 0.0;
  for (int r = b * CL_THREADS + threadIdx.x; r < rows; r += bpg * CL_THREADS) {
    const size_t i0 = ((size_t)g * rows + r) * C;
    float m = -INFINITY; for (int c = 0; c < C; ++c) m = fmaxf(m, ldf(z, i0 + c));
    float den = 0.f; for (int c = 0; c < C; ++c) den += expf(ldf(z, i0 + c) - m);
    float sy = 0.f, mr = 1.f;
    if (WM) {
      if (wm.w) for (int c = 0; c < C; ++c) sy += __fmul_rn(wm.w[c], y[i0 + c]);
      if (wm.m) mr = wm.m[(size_t)g * rows + r];
    }
    for (int c = 0; c < C; ++c) {
      const float p = expf(ldf(z, i0 + c) - m) / den;
      if (p_out) stf(p_out, i0 + c, p);
      if (WM) {
        const float yc = y[i0 + c], wy = wm.w ? wm.w[c] * yc : yc;
        stf(dz, i0 + c, mr * (wm.w ? __fmul_rn(p, sy) - wy : p - yc)); acc -= __dmul_rn((double)(mr * wy), log((double)fminf(fmaxf(p, 1e-10f), 1.0f - 1e-10f)));
      }
      else if (y) { const float yc = y[i0 + c]; stf(dz, i0 + c, p - yc); acc -= (double)yc * log((double)fminf(fmaxf(p, 1e-10f), 1.0f - 1e-10f)); }
    }
  }
  if (!y) return;
  const double tot = block_sum(acc, red);
  fold_partials(tot, (int)(gridDim.x / bpg), bpg, loss_sums, partial, ticket);
}

}  // namespace

void k_cnn_xent(int prec, const void* z, const float* y, void* dz, float* loss_sums, size_t n_per_group, int groups, float clip, double* partial, unsigned* ticket,
                cudaStream_t s) {
  const int bpg = k_loss_blocks(n_per_group, groups);
  const int V = prec == PREC_F32 ? 4 : 8;     // elements per 16-byte chunk of z / dz
  const bool vec = (uintptr_t)z % 16 == 0 && (uintptr_t)dz % 16 == 0 && (uintptr_t)y % 16 == 0 && (groups == 1 || n_per_group % V == 0);
  DISPATCH_PREC(prec, T, {
    if (vec) { launch_pdl(cnn_xent_kernel<T, true, false>, dim3(groups * bpg), dim3(CL_THREADS), (size_t)0, s, (const T*)z, y, (T*)dz, loss_sums, n_per_group, bpg, clip, partial, ticket, LossWM{}); g_ew_last_kernel = "cnn_xent_kernel<vec>"; }
    else { launch_pdl(cnn_xent_kernel<T, false, false>, dim3(groups * bpg), dim3(CL_THREADS), (size_t)0, s, (const T*)z, y, (T*)dz, loss_sums, n_per_group, bpg, clip, partial, ticket, LossWM{}); g_ew_last_kernel = "cnn_xent_kernel<scalar>"; }
  });
  LAUNCHED();
}
void k_cnn_xent_wm(int prec, const void* z, const float* y, void* dz, float* loss_sums, size_t n_per_group, int groups, float clip, double* partial, unsigned* ticket,
                   const LossWM& wm, cudaStream_t s) {
  const int bpg = k_loss_blocks(n_per_group, groups);
  const int V = prec == PREC_F32 ? 4 : 8;
  const bool vec = (uintptr_t)z % 16 == 0 && (uintptr_t)dz % 16 == 0 && (uintptr_t)y % 16 == 0 && (groups == 1 || n_per_group % V == 0);
  DISPATCH_PREC(prec, T, {
    if (vec) { launch_pdl(cnn_xent_kernel<T, true, true>, dim3(groups * bpg), dim3(CL_THREADS), (size_t)0, s, (const T*)z, y, (T*)dz, loss_sums, n_per_group, bpg, clip, partial, ticket, wm); g_ew_last_kernel = "cnn_xent_kernel<vec,wm>"; }
    else { launch_pdl(cnn_xent_kernel<T, false, true>, dim3(groups * bpg), dim3(CL_THREADS), (size_t)0, s, (const T*)z, y, (T*)dz, loss_sums, n_per_group, bpg, clip, partial, ticket, wm); g_ew_last_kernel = "cnn_xent_kernel<scalar,wm>"; }
  });
  LAUNCHED();
}

int k_cnn_softmax_blocks(int rows_per_group, int groups) { return k_loss_blocks((size_t)rows_per_group * 4, groups); }

void k_cnn_softmax_xent(int prec, const void* z, const float* y, void* dz, void* p_out, float* loss_sums, int rows_per_group, int C, int groups, double* partial,
                        unsigned* ticket, cudaStream_t s) {
  const int bpg = k_cnn_softmax_blocks(rows_per_group, groups);
  DISPATCH_PREC(prec, T, (launch_pdl(cnn_softmax_xent_kernel<T, false>, dim3(groups * bpg), dim3(CL_THREADS), (size_t)0, s, (const T*)z, y, (T*)dz, (T*)p_out, loss_sums,
                                     rows_per_group, C, bpg, partial, ticket, LossWM{})));
  LAUNCHED();
  g_ew_last_kernel = "cnn_softmax_xent_kernel";
}
void k_cnn_softmax_xent_wm(int prec, const void* z, const float* y, void* dz, float* loss_sums, int rows_per_group, int C, int groups, double* partial,
                           unsigned* ticket, const LossWM& wm, cudaStream_t s) {
  const int bpg = k_cnn_softmax_blocks(rows_per_group, groups);
  DISPATCH_PREC(prec, T, (launch_pdl(cnn_softmax_xent_kernel<T, true>, dim3(groups * bpg), dim3(CL_THREADS), (size_t)0, s, (const T*)z, y, (T*)dz, (T*)nullptr, loss_sums,
                                     rows_per_group, C, bpg, partial, ticket, wm)));
  LAUNCHED();
  g_ew_last_kernel = "cnn_softmax_xent_kernel<wm>";
}

}  // namespace b2g
