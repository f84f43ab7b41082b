// kernels_simt.cu -- implicit-GEMM convolution kernels on the fp32 FMA pipe (no tensor cores).
//
// These are (1) the fp32 "DL4J-parity" path (activations, weights and accumulation all fp32 -- the mode in
// which whole-step activations/gradients are compared with the oracle to 1e-3 relative) and (2) the
// correctness reference every tensor-core kernel in kernels_tc.cu is checked against on the device, and
// (3) the kernels for shapes the tensor-core path does not cover (5x5 reference convs, dense layers).
//
// One 64x64x16 tiled kernel, three gather rules (SURVEY.md section 8a rows a1, a2, a7):
//   fprop  out[(n,oy,ox)][o]   = sum_{r,s,c} x[n, oy*SH-PH+r, ox*SW-PW+s, c] * w[o][r][s][c]        (ConvolutionLayer.preOutput)
//   dgrad  dx[(n,iy,ix)][c]    = sum_{r,s,o} dy[n, (iy+PH-r)/SH, (ix+PW-s)/SW, o] * w[o][r][s][c]   (backprop eps; Deconvolution2D forward)
//   wgrad  dw[o][(r,s,c)]      = sum_{n,oy,ox} dy[n,oy,ox,o] * x[n, oy*SH-PH+r, ox*SW-PW+s, c]      (weight gradient, minibatch SUM)
// No im2col buffer is materialised (DL4J's nd4j-native path writes a 25x blow-up of the input, SURVEY.md 8a).
#include "kernels.h"
#include "common.cuh"

namespace b2g {

static const int TM = 64, TN = 64, TK = 16;
const char* g_gemm_last_kernel = "";
int g_gemm_last_splits = 0;

template <typename T, typename TW>
struct FpropProb {
  ConvGeom g; const T* x; const TW* w; const float* bias; const float* scale; T* out; int act; float alpha;
  int M, Ncols, K;
  __device__ __forceinline__ void load(float (*As)[TM + 4], float (*Bs)[TN + 4], int m0, int n0, int k0, int kend) const {
    int t = threadIdx.x;
    int row = t >> 2, kq = (t & 3) * 4;
    int m = m0 + row;
    int n = 0, oy = 0, ox = 0; bool mv = m < M;
    if (mv) { ox = m % g.OW; int tt = m / g.OW; oy = tt % g.OH; n = tt / g.OH; }
    int o = n0 + row; bool ov = o < Ncols;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int k = k0 + kq + i; float a = 0.f, b = 0.f;
      if (k < kend) {
        int c = k % g.C, tap = k / g.C, s = tap % g.KW, r = tap / g.KW;
        if (mv) { int iy = oy * g.SH - g.PH + r, ix = ox * g.SW - g.PW + s;
          if (iy >= 0 && iy < g.H && ix >= 0 && ix < g.W) a = ldf(x, (((size_t)n * g.H + iy) * g.W + ix) * g.C + c); }
        if (ov) b = ldf(w, (size_t)o * K + k);
      }
      As[kq + i][row] = a; Bs[kq + i][row] = b;
    }
  }
  __device__ __forceinline__ void store(float acc[4][4], int m0, int n0, int ty, int tx) const {
#pragma unroll
    for (int i = 0; i < 4; ++i) { int m = m0 + ty * 4 + i; if (m >= M) continue;
#pragma unroll
      for (int j = 0; j < 4; ++j) { int o = n0 + tx * 4 + j; if (o >= Ncols) continue;
        stf(out, (size_t)m * Ncols + o, act_fwd(act, acc[i][j] * (scale ? scale[o] : 1.f) + (bias ? bias[o] : 0.f), alpha)); } }
  }
};

template <typename T, typename TW>
struct DgradProb {
  ConvGeom g; const T* dy; const TW* w; const float* bias; const float* scale; T* dx; int act; float alpha;
  int M, Ncols, K;   // M = N*H*W, Ncols = C, K = KH*KW*O
  __device__ __forceinline__ void load(float (*As)[TM + 4], float (*Bs)[TN + 4], int m0, int n0, int k0, int kend) const {
    int t = threadIdx.x;
    { // A: row = input pixel, k = (r,s,o)
      int row = t >> 2, kq = (t & 3) * 4; int m = m0 + row; bool mv = m < M;
      int n = 0, iy = 0, ix = 0;
      if (mv) { ix = m % g.W; int tt = m / g.W; iy = tt % g.H; n = tt / g.H; }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        int k = k0 + kq + i; float a = 0.f;
        if (k < kend && mv) {
          int o = k % g.O, tap = k / g.O, s = tap % g.KW, r = tap / g.KW;
          int ty = iy + g.PH - r, tx = ix + g.PW - s;
          if (ty >= 0 && tx >= 0 && ty % g.SH == 0 && tx % g.SW == 0) {
            int oy = ty / g.SH, ox = tx / g.SW;
            if (oy < g.OH && ox < g.OW) a = ldf(dy, (((size_t)n * g.OH + oy) * g.OW + ox) * g.O + o);
          }
        }
        As[kq + i][row] = a;
      }
    }
    { // B: k = (r,s,o), col = c ; w[(o*taps + tap)*C + c]  (c contiguous)
      int kk = t >> 4, cq = (t & 15) * 4; int k = k0 + kk;
      int taps = g.KH * g.KW;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        int c = n0 + cq + j; float b = 0.f;
        if (k < kend && c < Ncols) { int o = k % g.O, tap = k / g.O; b = ldf(w, ((size_t)o * taps + tap) * g.C + c); }
        Bs[kk][cq + j] = b;
      }
    }
  }
  __device__ __forceinline__ void store(float acc[4][4], int m0, int n0, int ty, int tx) const {
#pragma unroll
    for (int i = 0; i < 4; ++i) { int m = m0 + ty * 4 + i; if (m >= M) continue;
#pragma unroll
      for (int j = 0; j < 4; ++j) { int c = n0 + tx * 4 + j; if (c >= Ncols) continue;
        stf(dx, (size_t)m * Ncols + c, act_fwd(act, acc[i][j] * (scale ? scale[c] : 1.f) + (bias ? bias[c] : 0.f), alpha)); } }
  }
};

template <typename T>
struct WgradProb {
  ConvGeom g; const T* x; const T* dy; float* out; size_t split_stride;
  int M, Ncols, K;   // M = O, Ncols = KH*KW*C, K = N*OH*OW
  __device__ __forceinline__ void load(float (*As)[TM + 4], float (*Bs)[TN + 4], int m0, int n0, int k0, int kend) const {
    int t = threadIdx.x;
    int col = t & 63, kq = (t >> 6) * 4;
    int o = m0 + col; bool ov = o < M;
    int j = n0 + col; bool jv = j < Ncols;
    int c = 0, r = 0, s = 0;
    if (jv) { c = j % g.C; int tap = j / g.C; s = tap % g.KW; r = tap / g.KW; }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int k = k0 + kq + i; float a = 0.f, b = 0.f;
      if (k < kend) {
        if (ov) a = ldf(dy, (size_t)k * g.O + o);
        if (jv) { int ox = k % g.OW; int tt = k / g.OW; int oy = tt % g.OH; int n = tt / g.OH;
          int iy = oy * g.SH - g.PH + r, ix = ox * g.SW - g.PW + s;
          if (iy >= 0 && iy < g.H && ix >= 0 && ix < g.W) b = ldf(x, (((size_t)n * g.H + iy) * g.W + ix) * g.C + c); }
      }
      As[kq + i][col] = a; Bs[kq + i][col] = b;
    }
  }
  __device__ __forceinline__ void store(float acc[4][4], int m0, int n0, int ty, int tx) const {
    float* dst = out + (size_t)blockIdx.z * split_stride;
#pragma unroll
    for (int i = 0; i < 4; ++i) { int m = m0 + ty * 4 + i; if (m >= M) continue;
#pragma unroll
      for (int j = 0; j < 4; ++j) { int c = n0 + tx * 4 + j; if (c >= Ncols) continue; dst[(size_t)m * Ncols + c] = acc[i][j]; } }
  }
};

template <class Prob>
__global__ void __launch_bounds__(256) simt_gemm_kernel(Prob p, int k_per_split) { pdl_enter();
  __shared__ float As[TK][TM + 4];
  __shared__ float Bs[TK][TN + 4];
  const int m0 = blockIdx.y * TM, n0 = blockIdx.x * TN;
  const int kbeg = blockIdx.z * k_per_split, kend = min(p.K, kbeg + k_per_split);
  const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = kbeg; k0 < kend; k0 += TK) {
    p.load(As, Bs, m0, n0, k0, kend);
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < TK; ++kk) {
      float a[4], b[4];
      *reinterpret_cast<float4*>(a) = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      *reinterpret_cast<float4*>(b) = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  p.store(acc, m0, n0, ty, tx);
}

template <typename T, typename TW>
static void launch_fprop(const ConvGeom& g, const void* x, const void* w, const float* bias, const float* scale, void* out, int act, float alpha, cudaStream_t s) {
  FpropProb<T, TW> p{g, (const T*)x, (const TW*)w, bias, scale, (T*)out, act, alpha, g.N * g.OH * g.OW, g.O, g.KH * g.KW * g.C};
  dim3 grid((p.Ncols + TN - 1) / TN, (p.M + TM - 1) / TM, 1);
  launch_pdl(simt_gemm_kernel<FpropProb<T, TW>>, dim3(grid), dim3(256), (size_t)(0), s, p, p.K); LAUNCHED();
  g_gemm_last_kernel = "simt_gemm_kernel<FpropProb>"; g_gemm_last_splits = 1;
}
template <typename T, typename TW>
static void launch_dgrad(const ConvGeom& g, const void* dy, const void* w, const float* bias, const float* scale, void* dx, int act, float alpha, cudaStream_t s) {
  DgradProb<T, TW> p{g, (const T*)dy, (const TW*)w, bias, scale, (T*)dx, act, alpha, g.N * g.H * g.W, g.C, g.KH * g.KW * g.O};
  dim3 grid((p.Ncols + TN - 1) / TN, (p.M + TM - 1) / TM, 1);
  launch_pdl(simt_gemm_kernel<DgradProb<T, TW>>, dim3(grid), dim3(256), (size_t)(0), s, p, p.K); LAUNCHED();
  g_gemm_last_kernel = "simt_gemm_kernel<DgradProb>"; g_gemm_last_splits = 1;
}

void k_simt_fprop(int prec, int wprec, const ConvGeom& g, const void* x, const void* w, const float* bias, void* out, int act, float alpha, cudaStream_t s, const float* scale) {
  if (prec == PREC_F32) launch_fprop<float, float>(g, x, w, bias, scale, out, act, alpha, s);
  else if (wprec == PREC_F32) launch_fprop<__nv_bfloat16, float>(g, x, w, bias, scale, out, act, alpha, s);
  else launch_fprop<__nv_bfloat16, __nv_bfloat16>(g, x, w, bias, scale, out, act, alpha, s);
}
void k_simt_dgrad(int prec, int wprec, const ConvGeom& g, const void* dy, const void* w, const float* bias, void* dx, int act, float alpha, cudaStream_t s, const float* scale) {
  if (prec == PREC_F32) launch_dgrad<float, float>(g, dy, w, bias, scale, dx, act, alpha, s);
  else if (wprec == PREC_F32) launch_dgrad<__nv_bfloat16, float>(g, dy, w, bias, scale, dx, act, alpha, s);
  else launch_dgrad<__nv_bfloat16, __nv_bfloat16>(g, dy, w, bias, scale, dx, act, alpha, s);
}

static int wgrad_splits(const ConvGeom& g) {
  long tiles = (long)((g.O + TM - 1) / TM) * ((g.KH * g.KW * g.C + TN - 1) / TN);
  long P = (long)g.N * g.OH * g.OW;
  long sp = (296 + tiles - 1) / tiles; if (sp > 64) sp = 64; long cap = P / 256; if (cap < 1) cap = 1; if (sp > cap) sp = cap; if (sp < 1) sp = 1;
  return (int)sp;
}
size_t k_simt_wgrad_scratch_floats(const ConvGeom& g) {
  int sp = wgrad_splits(g); return (size_t)sp * g.O * g.KH * g.KW * g.C;   // also covers accumulate with one split
}
void k_simt_wgrad(int prec, const ConvGeom& g, const void* x, const void* dy, float* dw, float* scratch, size_t scratch_floats, int accumulate, cudaStream_t s) {
  int sp = wgrad_splits(g);
  size_t n = (size_t)g.O * g.KH * g.KW * g.C;
  if (sp > 1 && scratch_floats < (size_t)sp * n) sp = 1;
  int P = g.N * g.OH * g.OW;
  int kps = ((P + sp - 1) / sp + TK - 1) / TK * TK;
  float* dst = (sp > 1 || accumulate) ? scratch : dw;
  if (sp == 1 && accumulate && scratch_floats < n) { dst = dw; accumulate = 0; }   // caller guarantees scratch when accumulating
  dim3 grid((int)((g.KH * g.KW * g.C + TN - 1) / TN), (g.O + TM - 1) / TM, sp);
  DISPATCH_PREC(prec, T, (launch_pdl(simt_gemm_kernel<WgradProb<T>>, dim3(grid), dim3(256), (size_t)(0), s, WgradProb<T>{g, (const T*)x, (const T*)dy, dst, n, g.O, g.KH * g.KW * g.C, P}, kps))); LAUNCHED();
  if (dst != dw) k_reduce_splits(dst, dw, n, sp, n, accumulate, s);
  g_gemm_last_kernel = "simt_gemm_kernel<WgradProb>"; g_gemm_last_splits = sp;
}

}  // namespace b2g
