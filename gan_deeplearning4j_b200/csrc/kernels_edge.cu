// kernels_edge.cu -- the "skinny" layers of the DCGAN stack, which are HBM/FMA-bound and not tensor-core shaped
// (SURVEY.md section 7 "skinny layers": D1 with K=48, G-last with 3 output channels, D-last with one output):
//
//   edge_deconv_small_c   Deconvolution2D 4x4 s2 p1 with <=4 output channels (G-last forward; D1's input gradient)
//   edge_conv_small_cin   ConvolutionLayer 4x4 s2 p1 with <=4 input channels (D1 forward; G-last's input gradient)
//   edge_wgrad_small_cin  its weight gradient (D1 / G-last), a [O x 48] result reduced over every pixel of the batch
//   dense_small_o_*       layers with <=4 output units (D-last 4x4 "valid" conv on a 4x4 map = a dot product per image;
//                         the reference's OutputLayer 1024->1, J:159-163): forward, input gradient, weight gradient
//
// All are direct (no GEMM tiles): weights live in shared memory as fp32 and are read as broadcasts, activations are
// read with 16-byte loads where the layout allows, every output element is written exactly once, reductions are
// fixed-order (partials + k_reduce_splits), so results are deterministic.
#include "kernels.h"
#include "common.cuh"

namespace b2g {

template <typename T> __device__ __forceinline__ void load8(const T* p, float (&v)[8]);
template <> __device__ __forceinline__ void load8<float>(const float* p, float (&v)[8]) {
  float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
template <> __device__ __forceinline__ void load8<__nv_bfloat16>(const __nv_bfloat16* p, float (&v)[8]) {
  uint4 u = *reinterpret_cast<const uint4*>(p);
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int j = 0; j < 4; ++j) { float2 f = __bfloat1622float2(h[j]); v[2 * j] = f.x; v[2 * j + 1] = f.y; }
}
template <typename TW> __device__ __forceinline__ float ldw(const TW* w, size_t i) { return ldf(w, i); }
// parameters sit at arbitrary element offsets of the flattened fp32 vector: vector loads only when 16-byte aligned
template <typename T> __device__ __forceinline__ void load8_any(const T* p, float (&v)[8]) {
  if ((reinterpret_cast<uintptr_t>(p) & 15) == 0) { load8(p, v); return; }
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = ldf(p, j);
}

// ------------------------------------------------------------------ (a) transposed conv, <=4 output channels ----
// dx[n, 2q+p] = bias + sum over the 2x2 taps of that parity class (sub-pixel phase form, as in kernels_tc.cu).
// One thread per dy-grid position (n,qy,qx): reads its 3x3 neighbourhood once, writes the 2x2 output block.
template <typename T, typename TW>
__global__ void __launch_bounds__(128) edge_deconv_small_c_kernel(const T* __restrict__ dy, const TW* __restrict__ w, const float* __restrict__ bias, T* __restrict__ dx,
                                                                   int N, int OH, int OW, int O, int C, int act, float alpha) { pdl_enter();
  extern __shared__ float4 ws4[];      // [16 taps][O] : (c0,c1,c2,c3)
  for (int i = threadIdx.x; i < 16 * O; i += blockDim.x) {
    int tap = i / O, o = i % O; float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    const size_t base = ((size_t)o * 16 + tap) * C;
    v.x = ldw(w, base); if (C > 1) v.y = ldw(w, base + 1); if (C > 2) v.z = ldw(w, base + 2); if (C > 3) v.w = ldw(w, base + 3);
    ws4[i] = v;
  }
  __syncthreads();
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < (long)N * OH * OW; idx += (long)gridDim.x * blockDim.x) {
  const int qx = idx % OW; long t = idx / OW; const int qy = t % OH; const int n = (int)(t / OH);
  float4 acc[2][2];
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 2; ++b) acc[a][b] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int dyr = -1; dyr <= 1; ++dyr) {
    const int iy = qy + dyr; if (iy < 0 || iy >= OH) continue;
#pragma unroll
    for (int dxc = -1; dxc <= 1; ++dxc) {
      const int ix = qx + dxc; if (ix < 0 || ix >= OW) continue;
      const T* src = dy + (((size_t)n * OH + iy) * OW + ix) * O;
      for (int o8 = 0; o8 < O; o8 += 8) {
        float v[8]; load8(src + o8, v);
        // row offset dyr serves: -1 -> (py=0, r=3); 0 -> (py=0, r=1) and (py=1, r=2); +1 -> (py=1, r=0)
#pragma unroll
        for (int py = 0; py < 2; ++py) {
          int r;
          if (dyr == -1) { if (py != 0) continue; r = 3; } else if (dyr == 0) { r = py == 0 ? 1 : 2; } else { if (py != 1) continue; r = 0; }
#pragma unroll
          for (int px = 0; px < 2; ++px) {
            int s;
            if (dxc == -1) { if (px != 0) continue; s = 3; } else if (dxc == 0) { s = px == 0 ? 1 : 2; } else { if (px != 1) continue; s = 0; }
            const float4* wt = ws4 + (r * 4 + s) * O + o8;
#pragma unroll
            for (int j = 0; j < 8; ++j) { const float4 ww = wt[j]; acc[py][px].x = fmaf(v[j], ww.x, acc[py][px].x); acc[py][px].y = fmaf(v[j], ww.y, acc[py][px].y);
              acc[py][px].z = fmaf(v[j], ww.z, acc[py][px].z); acc[py][px].w = fmaf(v[j], ww.w, acc[py][px].w); }
          }
        }
      }
    }
  }
  const int H = 2 * OH, W = 2 * OW;
#pragma unroll
  for (int py = 0; py < 2; ++py)
#pragma unroll
    for (int px = 0; px < 2; ++px) {
      T* dst = dx + (((size_t)n * H + 2 * qy + py) * W + 2 * qx + px) * C;
      const float a4[4] = {acc[py][px].x, acc[py][px].y, acc[py][px].z, acc[py][px].w};
#pragma unroll
      for (int c = 0; c < 4; ++c) if (c < C) stf(dst, c, act_fwd(act, a4[c] + (bias ? bias[c] : 0.f), alpha));
    }
  }
}

__device__ __forceinline__ void store16(float* dst, const float (&a)[16]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) reinterpret_cast<float4*>(dst)[j] = make_float4(a[4 * j], a[4 * j + 1], a[4 * j + 2], a[4 * j + 3]);
}
__device__ __forceinline__ void store16(__nv_bfloat16* dst, const float (&a)[16]) {
  uint32_t pk[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { __nv_bfloat162 h = __floats2bfloat162_rn(a[2 * j], a[2 * j + 1]); pk[j] = *reinterpret_cast<uint32_t*>(&h); }
  reinterpret_cast<uint4*>(dst)[0] = make_uint4(pk[0], pk[1], pk[2], pk[3]); reinterpret_cast<uint4*>(dst)[1] = make_uint4(pk[4], pk[5], pk[6], pk[7]);
}
// ------------------------------------------------------------------ (b) conv 4x4 s2 p1, <=4 input channels ------
// One thread per (output pixel, group of 16 output channels): 16 accumulators, the 48 inputs come from 4 contiguous
// 12-element row segments, weights from smem as [k][O] so a warp's reads are broadcasts / conflict-free.
template <typename T, typename TW>
__global__ void __launch_bounds__(128) edge_conv_small_cin_kernel(const T* __restrict__ x, const TW* __restrict__ w, const float* __restrict__ bias, T* __restrict__ out,
                                                                   int N, int H, int W, int C, int OH, int OW, int O, int act, float alpha) { pdl_enter();
  extern __shared__ float wsf[];      // [16*C][O]
  const int K = 16 * C;
  for (int i = threadIdx.x; i < K * O; i += blockDim.x) { int o = i / K, k = i % K; wsf[k * O + o] = ldw(w, (size_t)i); }   // coalesced global read
  __syncthreads();
  // work item = (4 adjacent output pixels of one row, 16 output channels): every weight vector fetched from smem feeds 4 pixels
  const int groups = O / 16, OW4 = OW / 4;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < (long)N * OH * OW4 * groups; idx += (long)gridDim.x * blockDim.x) {
    // og fastest: the 4 threads of a pixel quad share their input loads (L1 broadcast); measured faster than a warp-uniform og
    const int og = idx % groups; long q = idx / groups;
    const int ox0 = (int)(q % OW4) * 4; long t = q / OW4; const int oy = t % OH; const int n = (int)(t / OH);
    float acc[4][16];
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
      for (int j = 0; j < 16; ++j) acc[p][j] = bias ? bias[og * 16 + j] : 0.f;
    for (int r = 0; r < 4; ++r) {
      const int iy = 2 * oy - 1 + r; if (iy < 0 || iy >= H) continue;
      const T* row = x + ((size_t)n * H + iy) * W * C;
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        for (int c = 0; c < C; ++c) {
          float v[4];
#pragma unroll
          for (int p = 0; p < 4; ++p) { const int ix = 2 * (ox0 + p) - 1 + s; v[p] = (ix >= 0 && ix < W) ? ldf(row, (size_t)ix * C + c) : 0.f; }
          const float4* wr = reinterpret_cast<const float4*>(wsf + ((r * 4 + s) * C + c) * O + og * 16);
#pragma unroll
          for (int j = 0; j < 4; ++j) { const float4 ww = wr[j];
#pragma unroll
            for (int p = 0; p < 4; ++p) { acc[p][4 * j] = fmaf(v[p], ww.x, acc[p][4 * j]); acc[p][4 * j + 1] = fmaf(v[p], ww.y, acc[p][4 * j + 1]);
              acc[p][4 * j + 2] = fmaf(v[p], ww.z, acc[p][4 * j + 2]); acc[p][4 * j + 3] = fmaf(v[p], ww.w, acc[p][4 * j + 3]); } }
        }
      }
    }
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      T* dst = out + ((((size_t)n * OH + oy) * OW + ox0 + p)) * O + og * 16;
#pragma unroll
      for (int j = 0; j < 16; ++j) acc[p][j] = act_fwd(act, acc[p][j], alpha);
      store16(dst, acc[p]);
    }
  }
}

// ------------------------------------------------------------------ (c) its weight gradient ---------------------
// dw[o][r][s][c] = sum_pix dy[pix][o] * x[pix(r,s)][c].  CTA = 2*O threads: thread -> (pair of o, filter row r); per pixel it reads
// one dy pair and the 4*C contiguous x values of its filter row from smem and does 2*4*C FMAs.  Each CTA reduces a contiguous pixel range;
// partials [grid][O*16*C] are summed by k_reduce_splits.
template <typename T>
__global__ void edge_wgrad_small_cin_kernel(const T* __restrict__ x, const T* __restrict__ dy, float* __restrict__ part, int N, int H, int W, int C, int OH, int OW, int O, int pix_per_cta) { pdl_enter();
  extern __shared__ float sm[];
  const int TP = 64;                           // pixels per smem tile
  float* sdy = sm;                             // [TP][O]
  float* sx = sm + TP * O;                     // [TP][4 rows][4 taps][4 channels] (channels zero padded)
  const int o2 = threadIdx.x % (O / 2), r = threadIdx.x / (O / 2);
  const long P = (long)N * OH * OW;
  const long p_beg = (long)blockIdx.x * pix_per_cta, p_end = min(P, p_beg + pix_per_cta);
  float acc0[16], acc1[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) { acc0[j] = 0.f; acc1[j] = 0.f; }
  for (long p0 = p_beg; p0 < p_end; p0 += TP) {
    const int np = (int)min((long)TP, p_end - p0);
    // dy tile: 16-byte (bf16) / 32-byte (fp32) loads, 8 channels at a time
    for (int i = threadIdx.x; i < TP * (O / 8); i += blockDim.x) {
      const int pp = i / (O / 8), o8 = (i % (O / 8)) * 8; float v[8];
      if (pp < np) load8(dy + (size_t)(p0 + pp) * O + o8, v); else {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = 0.f; }
      *reinterpret_cast<float4*>(sdy + pp * O + o8) = make_float4(v[0], v[1], v[2], v[3]);
      *reinterpret_cast<float4*>(sdy + pp * O + o8 + 4) = make_float4(v[4], v[5], v[6], v[7]);
    }
    // x rows: one (pixel, filter row) pair per work item; its 4 taps x C channels are contiguous in memory
    for (int i = threadIdx.x; i < TP * 4; i += blockDim.x) {
      const int pp = i >> 2, rr = i & 3; float* dstx = sx + pp * 64 + rr * 16;
      float vals[16];
#pragma unroll
      for (int e = 0; e < 16; ++e) vals[e] = 0.f;
      if (pp < np) {
        const long pix = p0 + pp; const int ox = pix % OW; const long t = pix / OW; const int oy = t % OH; const int n = (int)(t / OH);
        const int iy = 2 * oy - 1 + rr;
        if (iy >= 0 && iy < H) {
          const T* row = x + ((size_t)n * H + iy) * W * C;
#pragma unroll
          for (int sx_ = 0; sx_ < 4; ++sx_) { const int ix = 2 * ox - 1 + sx_; if (ix < 0 || ix >= W) continue;
#pragma unroll
            for (int c = 0; c < 4; ++c) if (c < C) vals[sx_ * 4 + c] = ldf(row, (size_t)ix * C + c); }
        }
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) reinterpret_cast<float4*>(dstx)[e] = make_float4(vals[4 * e], vals[4 * e + 1], vals[4 * e + 2], vals[4 * e + 3]);
    }
    __syncthreads();
    for (int pp = 0; pp < np; ++pp) {
      const float2 d = *reinterpret_cast<const float2*>(sdy + pp * O + 2 * o2);
      const float4* xr = reinterpret_cast<const float4*>(sx + pp * 64 + r * 16);
#pragma unroll
      for (int j = 0; j < 4; ++j) { const float4 xv = xr[j];
        acc0[4 * j] = fmaf(d.x, xv.x, acc0[4 * j]); acc0[4 * j + 1] = fmaf(d.x, xv.y, acc0[4 * j + 1]); acc0[4 * j + 2] = fmaf(d.x, xv.z, acc0[4 * j + 2]); acc0[4 * j + 3] = fmaf(d.x, xv.w, acc0[4 * j + 3]);
        acc1[4 * j] = fmaf(d.y, xv.x, acc1[4 * j]); acc1[4 * j + 1] = fmaf(d.y, xv.y, acc1[4 * j + 1]); acc1[4 * j + 2] = fmaf(d.y, xv.z, acc1[4 * j + 2]); acc1[4 * j + 3] = fmaf(d.y, xv.w, acc1[4 * j + 3]); }
    }
    __syncthreads();
  }
  float* dst = part + (size_t)blockIdx.x * O * 16 * C;
#pragma unroll
  for (int sx_ = 0; sx_ < 4; ++sx_)
#pragma unroll
    for (int c = 0; c < 4; ++c) if (c < C) {       // dw[o][r][s][c]; smem rows are laid out [s][4] (channel-padded)
      dst[((size_t)(2 * o2) * 4 + r) * 4 * C + sx_ * C + c] = acc0[sx_ * 4 + c];
      dst[((size_t)(2 * o2 + 1) * 4 + r) * 4 * C + sx_ * C + c] = acc1[sx_ * 4 + c];
    }
}

// ------------------------------------------------------------------ (d) layers with <=4 output units -------------
template <typename T, typename TW>
__global__ void __launch_bounds__(128) dense_small_o_fwd_kernel(const T* __restrict__ x, const TW* __restrict__ w, const float* __restrict__ bias, T* __restrict__ out, int K, int O, int act, float alpha) { pdl_enter();
  const int n = blockIdx.x; __shared__ float red[4][4];
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  const T* xr = x + (size_t)n * K;
  for (int k = threadIdx.x * 8; k < K; k += blockDim.x * 8) {
    float v[8]; load8(xr + k, v);
    for (int o = 0; o < O; ++o) { float wv[8]; load8_any(w + (size_t)o * K + k, wv);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[o] = fmaf(v[j], wv[j], acc[o]); }
  }
  for (int o = 0; o < O; ++o) { float a = acc[o]; for (int m = 16; m; m >>= 1) a += __shfl_xor_sync(0xffffffffu, a, m); if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][o] = a; }
  __syncthreads();
  if (threadIdx.x < O) { float a = red[0][threadIdx.x] + red[1][threadIdx.x] + red[2][threadIdx.x] + red[3][threadIdx.x]; stf(out, (size_t)n * O + threadIdx.x, act_fwd(act, a + (bias ? bias[threadIdx.x] : 0.f), alpha)); }
}
__device__ __forceinline__ void store8(float* p, const float (&v)[8]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]); *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
}
__device__ __forceinline__ void store8(__nv_bfloat16* p, const float (&v)[8]) {
  uint4 u; __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
  for (int j = 0; j < 4; ++j) h[j] = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]);
  *reinterpret_cast<uint4*>(p) = u;
}
// dx[n][k] = sum_o dy[n][o] w[o][k]: pure streaming (one 16-byte store per 8 k), thread = 8 adjacent k of one image
template <typename T, typename TW>
__global__ void __launch_bounds__(256) dense_small_o_dgrad_kernel(const T* __restrict__ dy, const TW* __restrict__ w, T* __restrict__ dx, int N, int K, int O) { pdl_enter();
  const int kv = K >> 3; const size_t total = (size_t)N * kv;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t n = i / kv; const int k = (int)(i - n * kv) << 3;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int o = 0; o < O; ++o) {
      const float d = ldf(dy, n * O + o); float wv[8]; load8_any(w + (size_t)o * K + k, wv);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = fmaf(d, wv[j], acc[j]);
    }
    store8(dx + n * K + k, acc);
  }
}
// dw[o][k] = sum_n dy[n][o] x[n][k]: thread = 8 adjacent k, blockIdx.y = a slice of the batch (fixed-order partials, reduced by k_reduce_splits);
// eight row loads in flight per thread
template <typename T>
__global__ void __launch_bounds__(128) dense_small_o_wgrad_kernel(const T* __restrict__ x, const T* __restrict__ dy, float* __restrict__ part, int N, int K, int O, int rows_per_split) { pdl_enter();
  const int k = (blockIdx.x * blockDim.x + threadIdx.x) << 3; if (k >= K) return;
  const int n0 = blockIdx.y * rows_per_split, n1 = min(N, n0 + rows_per_split);
  float acc[4][8];
#pragma unroll
  for (int o = 0; o < 4; ++o)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[o][j] = 0.f;
  for (int nb = n0; nb < n1; nb += 8) {
    float v[8][8];
#pragma unroll
    for (int r = 0; r < 8; ++r) { if (nb + r < n1) load8(x + (size_t)(nb + r) * K + k, v[r]); else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[r][j] = 0.f; } }
#pragma unroll
    for (int r = 0; r < 8; ++r) if (nb + r < n1) {
#pragma unroll
      for (int o = 0; o < 4; ++o) if (o < O) { const float d = ldf(dy, (size_t)(nb + r) * O + o);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[o][j] = fmaf(d, v[r][j], acc[o][j]); }
    }
  }
  for (int o = 0; o < O; ++o) store8(part + (size_t)blockIdx.y * O * K + (size_t)o * K + k, acc[o]);
}

// ------------------------------------------------------------------ (e) 1x1 layers with a short reduction (G-first: z -> 4x4 map) -----
// Transposed conv of a 1x1 input = out[n][c] = sum_o z[n][o] * W[o][c] with O = nIn (100) and C = taps*nOut (8192): the reduction is too
// short (and not a multiple of 64) for the tensor-core tiles, the work is reading W / writing the map once.  Thread = 2 adjacent c
// (one 32-bit weight load per o), 8 rows of n per CTA with z staged in smem as fp32 and read as float4 broadcasts (4 o at a time).
template <typename T> __device__ __forceinline__ float2 ld2(const T* p);
template <> __device__ __forceinline__ float2 ld2<float>(const float* p) { if ((reinterpret_cast<uintptr_t>(p) & 7) == 0) return *reinterpret_cast<const float2*>(p); return make_float2(p[0], p[1]); }   // fp32 parameters sit at arbitrary offsets
template <> __device__ __forceinline__ float2 ld2<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p)); }
__device__ __forceinline__ void st2(float* p, float a, float b) { *reinterpret_cast<float2*>(p) = make_float2(a, b); }
__device__ __forceinline__ void st2(__nv_bfloat16* p, float a, float b) { *reinterpret_cast<__nv_bfloat162*>(p) = __floats2bfloat162_rn(a, b); }

// The thread's weights for 16 o are fetched together, one chunk ahead of the FMAs (register double buffer): one global latency per 16 o.
template <typename T, typename TW>
__global__ void __launch_bounds__(128) dense_small_k_dgrad_kernel(const T* __restrict__ dy, const TW* __restrict__ w, const float* __restrict__ bias, T* __restrict__ dx,
                                                                   int N, int C, int O, int act, float alpha) { pdl_enter();
  constexpr int OC = 16;                                  // o per chunk
  __shared__ __align__(16) float sz[8][128];             // [n][o], zero padded to a multiple of OC
  const int cb = blockIdx.x * 256, c = cb + threadIdx.x * 2, n0 = blockIdx.y * 8, OP = (O + OC - 1) / OC * OC;
#pragma unroll 8
  for (int i = threadIdx.x; i < 8 * OP; i += 128) { const int r = i / OP, o = i - r * OP; sz[r][o] = (o < O && n0 + r < N) ? ldf(dy, (size_t)(n0 + r) * O + o) : 0.f; }
  float acc[8][2];
#pragma unroll
  for (int r = 0; r < 8; ++r) { acc[r][0] = 0.f; acc[r][1] = 0.f; }
  float2 pre[OC];                                         // thread's pair of columns for each o of the next chunk
#pragma unroll
  for (int j = 0; j < OC; ++j) pre[j] = (j < O) ? ld2(w + (size_t)j * C + c) : make_float2(0.f, 0.f);
  __syncthreads();
  for (int o0 = 0; o0 < OP; o0 += OC) {
    float2 cur[OC];
#pragma unroll
    for (int j = 0; j < OC; ++j) { cur[j] = pre[j]; pre[j] = (o0 + OC + j < O) ? ld2(w + (size_t)(o0 + OC + j) * C + c) : make_float2(0.f, 0.f); }
#pragma unroll
    for (int j4 = 0; j4 < OC / 4; ++j4) {
      const float2* wv = cur + 4 * j4;
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const float4 z = *reinterpret_cast<const float4*>(&sz[r][o0 + 4 * j4]);
        acc[r][0] = fmaf(z.x, wv[0].x, acc[r][0]); acc[r][1] = fmaf(z.x, wv[0].y, acc[r][1]);
        acc[r][0] = fmaf(z.y, wv[1].x, acc[r][0]); acc[r][1] = fmaf(z.y, wv[1].y, acc[r][1]);
        acc[r][0] = fmaf(z.z, wv[2].x, acc[r][0]); acc[r][1] = fmaf(z.z, wv[2].y, acc[r][1]);
        acc[r][0] = fmaf(z.w, wv[3].x, acc[r][0]); acc[r][1] = fmaf(z.w, wv[3].y, acc[r][1]);
      }
    }
  }
  const float b0 = bias ? bias[c] : 0.f, b1 = bias ? bias[c + 1] : 0.f;
#pragma unroll
  for (int r = 0; r < 8; ++r) if (n0 + r < N) st2(dx + (size_t)(n0 + r) * C + c, act_fwd(act, acc[r][0] + b0, alpha), act_fwd(act, acc[r][1] + b1, alpha));
}
// dw[o][c] = sum_n dy[n][o] * x[n][c]: thread = 2 adjacent c x 16 o, the whole batch reduced in the CTA (no split, deterministic);
// rows are consumed 8 at a time so that eight global loads are in flight per thread.  dw is a layer's slice of the flattened gradient vector,
// at any element offset: ST2 (dw 8-byte aligned; C and c are even) stores each pair as one float2, otherwise as two floats.
template <typename T, bool ST2>
__global__ void __launch_bounds__(128) dense_small_k_wgrad_kernel(const T* __restrict__ x, const T* __restrict__ dy, float* __restrict__ dw, int N, int C, int O) { pdl_enter();
  __shared__ __align__(16) float sd[128][16];            // [n][o local]
  const int c = (blockIdx.x * 128 + threadIdx.x) * 2, o0 = blockIdx.y * 16;
  float acc[16][2];
#pragma unroll
  for (int j = 0; j < 16; ++j) { acc[j][0] = 0.f; acc[j][1] = 0.f; }
  for (int nb = 0; nb < N; nb += 128) {
    __syncthreads();
    for (int i = threadIdx.x; i < 128 * 16; i += 128) { const int r = i >> 4, o = i & 15; sd[r][o] = (nb + r < N && o0 + o < O) ? ldf(dy, (size_t)(nb + r) * O + o0 + o) : 0.f; }
    __syncthreads();
    const int rows = min(128, N - nb);
    for (int r0 = 0; r0 < rows; r0 += 8) {
      float2 xv[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) xv[q] = (r0 + q < rows) ? ld2(x + (size_t)(nb + r0 + q) * C + c) : make_float2(0.f, 0.f);
#pragma unroll
      for (int q = 0; q < 8; ++q) {
#pragma unroll
        for (int j4 = 0; j4 < 4; ++j4) {
          const float4 d = *reinterpret_cast<const float4*>(&sd[r0 + q][4 * j4]);
          acc[4 * j4][0] = fmaf(d.x, xv[q].x, acc[4 * j4][0]); acc[4 * j4][1] = fmaf(d.x, xv[q].y, acc[4 * j4][1]);
          acc[4 * j4 + 1][0] = fmaf(d.y, xv[q].x, acc[4 * j4 + 1][0]); acc[4 * j4 + 1][1] = fmaf(d.y, xv[q].y, acc[4 * j4 + 1][1]);
          acc[4 * j4 + 2][0] = fmaf(d.z, xv[q].x, acc[4 * j4 + 2][0]); acc[4 * j4 + 2][1] = fmaf(d.z, xv[q].y, acc[4 * j4 + 2][1]);
          acc[4 * j4 + 3][0] = fmaf(d.w, xv[q].x, acc[4 * j4 + 3][0]); acc[4 * j4 + 3][1] = fmaf(d.w, xv[q].y, acc[4 * j4 + 3][1]);
        }
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 16; ++j) if (o0 + j < O) {
    float* p = dw + (size_t)(o0 + j) * C + c;
    if constexpr (ST2) st2(p, acc[j][0], acc[j][1]); else { p[0] = acc[j][0]; p[1] = acc[j][1]; }
  }
}


// ------------------------------------------------------------------ (e') the same two GEMMs on warp-level tensor-core MMAs (bf16 operands) ---
// out[n][c] = sum_o z[n][o] W[o][c] (N x 100 x 8192) and dW[o][c] = sum_n z[n][o] dOut[n][c] (100 x N x 8192) are 0.2 GFLOP each: the
// SIMT kernels above spend ~18 us on instruction issue (ncu: 43 % issue-slot busy at 25 % occupancy).  mma.sync.m16n8k16 with ldmatrix
// fragments cuts the instruction count ~10x; the tensor-core path does not apply (reduction of 100 is not a multiple of 64 and the operand
// rows are not 16-byte multiples for TMA).  Operands are staged once per CTA in shared memory, rows padded so that every ldmatrix
// phase touches 8 distinct 16-byte bank groups.
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"((uint32_t)__cvta_generic_to_shared(p)));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"((uint32_t)__cvta_generic_to_shared(p)));
}
__device__ __forceinline__ void ldsm_x2_t(uint32_t& r0, uint32_t& r1, const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];" : "=r"(r0), "=r"(r1) : "r"((uint32_t)__cvta_generic_to_shared(p)));
}
static constexpr int DK_AP = 136, DK_BP = 72;     // shared-memory row pitches (bf16 elements): 272 B and 144 B, both 16-byte multiples
// forward: CTA = 64 images x 64 columns, warp = 16 images x 64 columns; the reduction (O <= 128, zero padded to a multiple of 16) is resident
// z tile [ROWS images][O] -> shared [ROWS][DK_AP], zero padded to OP columns and past the batch; four loads in flight per thread
template <int ROWS, int OP>
__device__ __forceinline__ void dk_fill_z(const __nv_bfloat16* __restrict__ z, __nv_bfloat16* sA, int n0, int N, int O, int tid) {
  constexpr int HALF = OP / 2, TOTAL = ROWS * HALF;
#pragma unroll 1
  for (int i0 = tid; i0 < TOTAL; i0 += 128 * 16) {
    __nv_bfloat162 v[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int i = i0 + u * 128, r = i / HALF, o = (i - r * HALF) * 2, n = n0 + r;
      v[u] = __floats2bfloat162_rn(0.f, 0.f);
      if (i < TOTAL && n < N) {
        if (!(O & 1)) { if (o < O) v[u] = *reinterpret_cast<const __nv_bfloat162*>(z + (size_t)n * O + o); }
        else { if (o < O) v[u].x = z[(size_t)n * O + o]; if (o + 1 < O) v[u].y = z[(size_t)n * O + o + 1]; }
      }
    }
#pragma unroll
    for (int u = 0; u < 16; ++u) { const int i = i0 + u * 128, r = i / HALF, o = (i - r * HALF) * 2; if (i < TOTAL) *reinterpret_cast<__nv_bfloat162*>(sA + r * DK_AP + o) = v[u]; }
  }
}
template <int KT>
__global__ void __launch_bounds__(128) dense_k_fwd_mma_kernel(const __nv_bfloat16* __restrict__ z, const __nv_bfloat16* __restrict__ w, const float* __restrict__ bias,
                                                              __nv_bfloat16* __restrict__ out, int N, int C, int O, int act, float alpha) { pdl_enter();
  __shared__ __align__(16) __nv_bfloat16 sA[64 * DK_AP];      // [image][o]
  __shared__ __align__(16) __nv_bfloat16 sB[128 * DK_BP];     // [o][column]
  constexpr int OP = KT * 16;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, c0 = blockIdx.x * 64, n0 = blockIdx.y * 64;
  dk_fill_z<64, OP>(z, sA, n0, N, O, tid);
#pragma unroll
  for (int i = tid; i < OP * 8; i += 128) {                   // 8 x 16 B per weight row, all loads of a thread in flight together
    const int o = i >> 3, j = i & 7;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (o < O) v = __ldg(reinterpret_cast<const uint4*>(w + (size_t)o * C + c0) + j);
    *reinterpret_cast<uint4*>(sB + o * DK_BP + j * 8) = v;
  }
  __syncthreads();
  float acc[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j) { acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f; }
  // ldmatrix row addresses: A (x4, no transpose) matrices = (rows 0-7 | 8-15) x (k 0-7 | 8-15); B (x2, transposed) = k 0-7 | 8-15 of one 8-column block
  const __nv_bfloat16* aptr = sA + (warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * DK_AP + (lane >> 4) * 8;
  const __nv_bfloat16* bptr = sB + ((lane & 7) + ((lane >> 3) & 1) * 8) * DK_BP;
#pragma unroll
  for (int k0 = 0; k0 < OP; k0 += 16) {
    uint32_t a[4]; ldsm_x4(a, aptr + k0);
#pragma unroll
    for (int j = 0; j < 8; ++j) { uint32_t b0, b1; ldsm_x2_t(b0, b1, bptr + k0 * DK_BP + j * 8); mma_bf16_16816(acc[j], a, b0, b1); }
  }
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = c0 + j * 8 + 2 * t; const float b0 = bias ? bias[c] : 0.f, b1 = bias ? bias[c + 1] : 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int n = n0 + warp * 16 + g + h * 8;
      if (n < N) *reinterpret_cast<__nv_bfloat162*>(out + (size_t)n * C + c) = __floats2bfloat162_rn(act_fwd(act, acc[j][2 * h] + b0, alpha), act_fwd(act, acc[j][2 * h + 1] + b1, alpha));
    }
  }
}
// weight gradient: CTA = all O (<= 128, padded to OP) x 64 columns, warp = OP x 16 columns; the batch is consumed 64 images at a time in a
// fixed order (deterministic, no split).  A = z^T comes out of the [image][o] tile through transposing ldmatrix.
template <int KT>
__global__ void __launch_bounds__(128) dense_k_wgrad_mma_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ z, float* __restrict__ dw, int N, int C, int O) { pdl_enter();
  __shared__ __align__(16) __nv_bfloat16 sZ[64 * DK_AP];     // [image][o]
  __shared__ __align__(16) __nv_bfloat16 sX[64 * DK_BP];     // [image][column]
  constexpr int OP = KT * 16, MT = KT;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, c0 = blockIdx.x * 64;
  float acc[MT][2][4];
#pragma unroll
  for (int m = 0; m < MT; ++m)
#pragma unroll
    for (int j = 0; j < 2; ++j) { acc[m][j][0] = acc[m][j][1] = acc[m][j][2] = acc[m][j][3] = 0.f; }
  for (int nb = 0; nb < N; nb += 64) {
    __syncthreads();
    dk_fill_z<64, OP>(z, sZ, nb, N, O, tid);
#pragma unroll
    for (int i = tid; i < 64 * 8; i += 128) {
      const int r = i >> 3, j = i & 7; const int n = nb + r;
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if (n < N) v = __ldg(reinterpret_cast<const uint4*>(x + (size_t)n * C + c0) + j);
      *reinterpret_cast<uint4*>(sX + r * DK_BP + j * 8) = v;
    }
    __syncthreads();
    // A^T tile stored [k = image][m = o]: x4.trans matrices = (m 0-7 | 8-15) x (k 0-7 | 8-15) -> a0..a3
    const __nv_bfloat16* aptr = sZ + ((lane & 7) + (lane >> 4) * 8) * DK_AP + ((lane >> 3) & 1) * 8;
    const __nv_bfloat16* bptr = sX + ((lane & 7) + ((lane >> 3) & 1) * 8) * DK_BP + warp * 16;
#pragma unroll
    for (int k0 = 0; k0 < 64; k0 += 16) {
      uint32_t b[2][2];
#pragma unroll
      for (int j = 0; j < 2; ++j) ldsm_x2_t(b[j][0], b[j][1], bptr + k0 * DK_BP + j * 8);
#pragma unroll
      for (int m = 0; m < MT; ++m) {
        uint32_t a[4]; ldsm_x4_t(a, aptr + k0 * DK_AP + m * 16);
#pragma unroll
        for (int j = 0; j < 2; ++j) mma_bf16_16816(acc[m][j], a, b[j][0], b[j][1]);
      }
    }
  }
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int m = 0; m < MT; ++m)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int o = m * 16 + g + h * 8;
        if (o < O) *reinterpret_cast<float2*>(dw + (size_t)o * C + c0 + warp * 16 + j * 8 + 2 * t) = make_float2(acc[m][j][2 * h], acc[m][j][2 * h + 1]);
      }
}

// ------------------------------------------------------------------ host wrappers ---------------------------------
static bool is_k4s2p1(const ConvGeom& g) { return g.KH == 4 && g.KW == 4 && g.SH == 2 && g.SW == 2 && g.PH == 1 && g.PW == 1 && g.H == 2 * g.OH && g.W == 2 * g.OW; }
bool edge_deconv_small_c_supported(const ConvGeom& g) { return is_k4s2p1(g) && g.C <= 4 && g.O % 8 == 0 && g.O <= 128; }
bool edge_conv_small_cin_supported(const ConvGeom& g) { return is_k4s2p1(g) && g.C <= 4 && g.O % 16 == 0 && g.OW % 4 == 0 && 16 * g.C * g.O * 4 <= 48 * 1024; }
bool edge_wgrad_small_cin_supported(const ConvGeom& g) { return is_k4s2p1(g) && g.C <= 4 && g.O % 8 == 0 && g.O <= 256; }
bool dense_small_o_supported(const ConvGeom& g) { return g.KH == 1 && g.KW == 1 && g.H == 1 && g.W == 1 && g.O <= 4 && g.C % 8 == 0; }

template <typename T, typename TW>
static void launch_deconv_small_c(const ConvGeom& g, const void* dy, const void* w, const float* bias, void* dx, int act, float alpha, cudaStream_t s) {
  long tot = (long)g.N * g.OH * g.OW; long blocks = (tot + 127) / 128; if (blocks > device_sm_count() * 8) blocks = device_sm_count() * 8;
  launch_pdl(edge_deconv_small_c_kernel<T, TW>, dim3((unsigned)blocks), dim3(128), (size_t)(16 * g.O * sizeof(float4)), s, (const T*)dy, (const TW*)w, bias, (T*)dx, g.N, g.OH, g.OW, g.O, g.C, act, alpha);
  g_gemm_last_kernel = "edge_deconv_small_c_kernel"; g_gemm_last_splits = 1;
}
void k_edge_deconv_small_c(int prec, int wprec, const ConvGeom& g, const void* dy, const void* w, const float* bias, void* dx, int act, float alpha, cudaStream_t s) {
  if (prec == PREC_F32) launch_deconv_small_c<float, float>(g, dy, w, bias, dx, act, alpha, s);
  else if (wprec == PREC_F32) launch_deconv_small_c<__nv_bfloat16, float>(g, dy, w, bias, dx, act, alpha, s);
  else launch_deconv_small_c<__nv_bfloat16, __nv_bfloat16>(g, dy, w, bias, dx, act, alpha, s);
  LAUNCHED();
}
template <typename T, typename TW>
static void launch_conv_small_cin(const ConvGeom& g, const void* x, const void* w, const float* bias, void* out, int act, float alpha, cudaStream_t s) {
  long tot = (long)g.N * g.OH * (g.OW / 4) * (g.O / 16); long blocks = (tot + 127) / 128; if (blocks > device_sm_count() * 8) blocks = device_sm_count() * 8;
  launch_pdl(edge_conv_small_cin_kernel<T, TW>, dim3((unsigned)blocks), dim3(128), (size_t)(16 * g.C * g.O * sizeof(float)), s, (const T*)x, (const TW*)w, bias, (T*)out, g.N, g.H, g.W, g.C, g.OH, g.OW, g.O, act, alpha);
  g_gemm_last_kernel = "edge_conv_small_cin_kernel"; g_gemm_last_splits = 1;
}
void k_edge_conv_small_cin(int prec, int wprec, const ConvGeom& g, const void* x, const void* w, const float* bias, void* out, int act, float alpha, cudaStream_t s) {
  if (prec == PREC_F32) launch_conv_small_cin<float, float>(g, x, w, bias, out, act, alpha, s);
  else if (wprec == PREC_F32) launch_conv_small_cin<__nv_bfloat16, float>(g, x, w, bias, out, act, alpha, s);
  else launch_conv_small_cin<__nv_bfloat16, __nv_bfloat16>(g, x, w, bias, out, act, alpha, s);
  LAUNCHED();
}
static int edge_wgrad_ctas(const ConvGeom& g) { long P = (long)g.N * g.OH * g.OW; long c = device_sm_count() * 2; long cap = (P + 63) / 64; if (c > cap) c = cap; if (c < 1) c = 1; return (int)c; }
size_t k_edge_wgrad_scratch_floats(const ConvGeom& g) { return edge_wgrad_small_cin_supported(g) ? (size_t)edge_wgrad_ctas(g) * g.O * 16 * g.C : 0; }
// (64*O + 64*64) floats of dynamic shared memory: past the 48 KB default for O > 128.  The kernel is opted into the amount the largest
// supported O (256) needs, once per (instantiation, device) -- the attribute is per device -- and only by a launch that needs more than 48 KB.
static size_t edge_wgrad_smem(int O) { return (64 * (size_t)O + 64 * 64) * sizeof(float); }
template <typename T> static void edge_wgrad_opt_in() {
  static bool set_[64] = {}; int d = 0; cudaGetDevice(&d); if (d < 0 || d >= 64) d = 0;
  if (!set_[d] && cudaFuncSetAttribute(edge_wgrad_small_cin_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)edge_wgrad_smem(256)) == cudaSuccess) set_[d] = true;
}
void k_edge_wgrad_small_cin(int prec, const ConvGeom& g, const void* x, const void* dy, float* dw, float* scratch, int accumulate, cudaStream_t s) {
  const int ctas = edge_wgrad_ctas(g); const long P = (long)g.N * g.OH * g.OW; const int ppc = (int)((P + ctas - 1) / ctas);
  const size_t n = (size_t)g.O * 16 * g.C; const size_t smem = edge_wgrad_smem(g.O);
  if (smem > 48 * 1024) DISPATCH_PREC(prec, T, (edge_wgrad_opt_in<T>()));
  DISPATCH_PREC(prec, T, (launch_pdl(edge_wgrad_small_cin_kernel<T>, dim3(ctas), dim3(2 * g.O), (size_t)(smem), s, (const T*)x, (const T*)dy, scratch, g.N, g.H, g.W, g.C, g.OH, g.OW, g.O, ppc))); LAUNCHED();
  k_reduce_splits(scratch, dw, n, ctas, n, accumulate, s);
  g_gemm_last_kernel = "edge_wgrad_small_cin_kernel"; g_gemm_last_splits = ctas;
}
bool dense_small_k_supported(const ConvGeom& g) { return g.KH == 1 && g.KW == 1 && g.H == 1 && g.W == 1 && g.O >= 1 && g.O <= 128 && g.C % 256 == 0 && g.C >= 256; }
void k_dense_small_k_dgrad(int prec, int wprec, const ConvGeom& g, const void* dy, const void* w, const float* bias, void* dx, int act, float alpha, cudaStream_t s) {
  dim3 grid(g.C / 256, (g.N + 7) / 8);
  g_gemm_last_kernel = "dense_small_k_dgrad_kernel"; g_gemm_last_splits = 1;
  if (prec == PREC_F32) launch_pdl(dense_small_k_dgrad_kernel<float, float>, grid, dim3(128), (size_t)0, s, (const float*)dy, (const float*)w, bias, (float*)dx, g.N, g.C, g.O, act, alpha);
  else if (wprec == PREC_F32) launch_pdl(dense_small_k_dgrad_kernel<__nv_bfloat16, float>, grid, dim3(128), (size_t)0, s, (const __nv_bfloat16*)dy, (const float*)w, bias, (__nv_bfloat16*)dx, g.N, g.C, g.O, act, alpha);
  else if ((reinterpret_cast<uintptr_t>(w) & 15) == 0 && (reinterpret_cast<uintptr_t>(dy) & 3) == 0 && (reinterpret_cast<uintptr_t>(dx) & 3) == 0) {
    g_gemm_last_kernel = "dense_k_fwd_mma_kernel";
    switch ((g.O + 15) / 16) {
#define B2G_DK_FWD(KT) case KT: launch_pdl(dense_k_fwd_mma_kernel<KT>, dim3(g.C / 64, (g.N + 63) / 64), dim3(128), (size_t)0, s, (const __nv_bfloat16*)dy, (const __nv_bfloat16*)w, bias, (__nv_bfloat16*)dx, g.N, g.C, g.O, act, alpha); break;
      B2G_DK_FWD(1) B2G_DK_FWD(2) B2G_DK_FWD(3) B2G_DK_FWD(4) B2G_DK_FWD(5) B2G_DK_FWD(6) B2G_DK_FWD(7) B2G_DK_FWD(8)
#undef B2G_DK_FWD
    }
  }
  else launch_pdl(dense_small_k_dgrad_kernel<__nv_bfloat16, __nv_bfloat16>, grid, dim3(128), (size_t)0, s, (const __nv_bfloat16*)dy, (const __nv_bfloat16*)w, bias, (__nv_bfloat16*)dx, g.N, g.C, g.O, act, alpha);
  LAUNCHED();
}
void k_dense_small_k_wgrad(int prec, const ConvGeom& g, const void* x, const void* dy, float* dw, cudaStream_t s) {
  dim3 grid(g.C / 256, (g.O + 15) / 16);
  if (prec == PREC_BF16 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(dy) & 3) == 0 && (reinterpret_cast<uintptr_t>(dw) & 7) == 0 && (((size_t)g.C * 4) & 7) == 0) {
    switch ((g.O + 15) / 16) {
#define B2G_DK_WG(KT) case KT: launch_pdl(dense_k_wgrad_mma_kernel<KT>, dim3(g.C / 64), dim3(128), (size_t)0, s, (const __nv_bfloat16*)x, (const __nv_bfloat16*)dy, dw, g.N, g.C, g.O); break;
      B2G_DK_WG(1) B2G_DK_WG(2) B2G_DK_WG(3) B2G_DK_WG(4) B2G_DK_WG(5) B2G_DK_WG(6) B2G_DK_WG(7) B2G_DK_WG(8)
#undef B2G_DK_WG
    }
    LAUNCHED(); g_gemm_last_kernel = "dense_k_wgrad_mma_kernel"; g_gemm_last_splits = 1; return;
  }
  if ((reinterpret_cast<uintptr_t>(dw) & 7) == 0) {
    DISPATCH_PREC(prec, T, (launch_pdl(dense_small_k_wgrad_kernel<T, true>, grid, dim3(128), (size_t)0, s, (const T*)x, (const T*)dy, dw, g.N, g.C, g.O)));
    g_gemm_last_kernel = "dense_small_k_wgrad_kernel<st2>";
  } else {
    DISPATCH_PREC(prec, T, (launch_pdl(dense_small_k_wgrad_kernel<T, false>, grid, dim3(128), (size_t)0, s, (const T*)x, (const T*)dy, dw, g.N, g.C, g.O)));
    g_gemm_last_kernel = "dense_small_k_wgrad_kernel<st1>";
  }
  LAUNCHED(); g_gemm_last_splits = 1;
}
void k_dense_small_o_fwd(int prec, int wprec, const ConvGeom& g, const void* x, const void* w, const float* bias, void* out, int act, float alpha, cudaStream_t s) {
  if (prec == PREC_F32) launch_pdl(dense_small_o_fwd_kernel<float, float>, dim3(g.N), dim3(128), (size_t)(0), s, (const float*)x, (const float*)w, bias, (float*)out, g.C, g.O, act, alpha);
  else if (wprec == PREC_F32) launch_pdl(dense_small_o_fwd_kernel<__nv_bfloat16, float>, dim3(g.N), dim3(128), (size_t)(0), s, (const __nv_bfloat16*)x, (const float*)w, bias, (__nv_bfloat16*)out, g.C, g.O, act, alpha);
  else launch_pdl(dense_small_o_fwd_kernel<__nv_bfloat16, __nv_bfloat16>, dim3(g.N), dim3(128), (size_t)(0), s, (const __nv_bfloat16*)x, (const __nv_bfloat16*)w, bias, (__nv_bfloat16*)out, g.C, g.O, act, alpha);
  LAUNCHED(); g_gemm_last_kernel = "dense_small_o_fwd_kernel"; g_gemm_last_splits = 1;
}
void k_dense_small_o_dgrad(int prec, int wprec, const ConvGeom& g, const void* dy, const void* w, void* dx, cudaStream_t s) {
  size_t tot = (size_t)g.N * (g.C / 8); int blocks = (int)((tot + 255) / 256); if (blocks > device_sm_count() * 8) blocks = device_sm_count() * 8;
  if (prec == PREC_F32) launch_pdl(dense_small_o_dgrad_kernel<float, float>, dim3(blocks), dim3(256), (size_t)(0), s, (const float*)dy, (const float*)w, (float*)dx, g.N, g.C, g.O);
  else if (wprec == PREC_F32) launch_pdl(dense_small_o_dgrad_kernel<__nv_bfloat16, float>, dim3(blocks), dim3(256), (size_t)(0), s, (const __nv_bfloat16*)dy, (const float*)w, (__nv_bfloat16*)dx, g.N, g.C, g.O);
  else launch_pdl(dense_small_o_dgrad_kernel<__nv_bfloat16, __nv_bfloat16>, dim3(blocks), dim3(256), (size_t)(0), s, (const __nv_bfloat16*)dy, (const __nv_bfloat16*)w, (__nv_bfloat16*)dx, g.N, g.C, g.O);
  LAUNCHED(); g_gemm_last_kernel = "dense_small_o_dgrad_kernel"; g_gemm_last_splits = 1;
}
static int dense_wgrad_splits(const ConvGeom& g) { int sp = (g.N + 7) / 8; if (sp > 32) sp = 32; if (sp < 1) sp = 1; return sp; }
size_t k_dense_small_o_wgrad_scratch_floats(const ConvGeom& g) { return dense_small_o_supported(g) ? (size_t)dense_wgrad_splits(g) * g.O * g.C : 0; }
void k_dense_small_o_wgrad(int prec, const ConvGeom& g, const void* x, const void* dy, float* dw, float* scratch, int accumulate, cudaStream_t s) {
  const int sp = dense_wgrad_splits(g), rps = (g.N + sp - 1) / sp; const size_t n = (size_t)g.O * g.C;
  dim3 grid((g.C / 8 + 127) / 128, sp);
  DISPATCH_PREC(prec, T, (launch_pdl(dense_small_o_wgrad_kernel<T>, dim3(grid), dim3(128), (size_t)(0), s, (const T*)x, (const T*)dy, scratch, g.N, g.C, g.O, rps))); LAUNCHED();
  k_reduce_splits(scratch, dw, n, sp, n, accumulate, s);
  g_gemm_last_kernel = "dense_small_o_wgrad_kernel"; g_gemm_last_splits = sp;
}

}  // namespace b2g
