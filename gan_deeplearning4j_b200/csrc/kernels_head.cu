// kernels_head.cu -- few-output conv kernels for BF16 nets: a k x k conv (KH*KW > 1, KH, KW <= 7, stride 1 or 2, 0 <= pad < kernel) from
// C % 8 == 0 channels onto O <= 4 channels on a map wider than one pixel: the PatchGAN discriminator's head (and the same geometry in any BF16
// net).  The tensor-core kernels need >= 64 output columns and the skinny-layer kernels take <= 4 INPUT channels or the 1x1 / full-window
// geometry, so without these the three GEMMs of such a layer ran on simt_gemm_kernel.
//
// All three read the bf16 weight copy [O][KH*KW][C] and the NHWC activations with 16-byte channel vectors, accumulate in fp32 in a fixed
// order and use no atomics:
//   forward      one warp per output pixel: lane l takes the channel vectors l, l+32, ... of every in-range tap (taps in row-major order), the
//                O sums fold with the warp's xor butterfly; lane o adds the bias, applies the activation (codes 0-4) and stores output o.
//   input grad   the gather form: one thread per (input pixel, 8-channel vector) sums dy[o] * W[o][tap][c] over the taps that cover the pixel
//                (filter row, then column, ascending; o ascending), then bias / activation (a transposed conv's forward uses them).
//   weight grad  one thread per (tap, 8-channel vector) column and pixel range: O x 8 fp32 sums over the range's output pixels in order into
//                partial [split][O][taps][C]; the splits are summed by one reduce_multi job (the backward pass's deferred list) or at once.
#include <algorithm>

#include "common.cuh"

namespace b2g {

namespace {

constexpr int HW_THREADS = 128;      // weight-gradient block: 128 columns

__device__ __forceinline__ void unpack8(const uint4& q, float* f) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&q);
#pragma unroll
  for (int k = 0; k < 4; ++k) { const float2 v = __bfloat1622float2(h[k]); f[2 * k] = v.x; f[2 * k + 1] = v.y; }
}

template <int O>
__global__ void __launch_bounds__(256) head_conv_fwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w, const float* __restrict__ bias,
                                                            __nv_bfloat16* __restrict__ out, const ConvGeom g, int act, float alpha) {
  pdl_wait();
  const int lane = threadIdx.x & 31, C8 = g.C / 8, taps = g.KH * g.KW;
  const int P = g.N * g.OH * g.OW;
  for (int pix = blockIdx.x * 8 + (threadIdx.x >> 5); pix < P; pix += gridDim.x * 8) {
    const int n = pix / (g.OH * g.OW), r = pix % (g.OH * g.OW), oy = r / g.OW, ox = r % g.OW;
    float acc[O];
#pragma unroll
    for (int o = 0; o < O; ++o) acc[o] = 0.f;
    for (int ky = 0; ky < g.KH; ++ky) {
      const int iy = oy * g.SH - g.PH + ky;
      if (iy < 0 || iy >= g.H) continue;
      for (int kx = 0; kx < g.KW; ++kx) {
        const int ix = ox * g.SW - g.PW + kx;
        if (ix < 0 || ix >= g.W) continue;
        const int tap = ky * g.KW + kx;
        const uint4* xp = reinterpret_cast<const uint4*>(x + (((size_t)n * g.H + iy) * g.W + ix) * g.C);
        for (int v = lane; v < C8; v += 32) {
          float xf[8]; unpack8(__ldg(xp + v), xf);
#pragma unroll
          for (int o = 0; o < O; ++o) {
            float wf[8]; unpack8(__ldg(reinterpret_cast<const uint4*>(w + ((size_t)o * taps + tap) * g.C) + v), wf);
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[o] = fmaf(xf[k], wf[k], acc[o]);
          }
        }
      }
    }
#pragma unroll
    for (int o = 0; o < O; ++o)
#pragma unroll
      for (int s = 16; s > 0; s >>= 1) acc[o] += __shfl_xor_sync(0xffffffffu, acc[o], s);
    float a = acc[0];      // every lane holds the O sums: lane o stores output o
#pragma unroll
    for (int o = 1; o < O; ++o) a = lane == o ? acc[o] : a;
    if (lane < O) out[(size_t)pix * O + lane] = __float2bfloat16_rn(act_fwd(act, a + (bias ? bias[lane] : 0.f), alpha));
  }
}

template <int O>
__global__ void __launch_bounds__(256) head_conv_dgrad_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ w, const float* __restrict__ bias,
                                                              __nv_bfloat16* __restrict__ dx, const ConvGeom g, int act, float alpha) {
  pdl_wait();
  const int C8 = g.C / 8, taps = g.KH * g.KW;
  const size_t total = (size_t)g.N * g.H * g.W * C8;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % C8); const size_t pix = i / C8;
    const int n = (int)(pix / ((size_t)g.H * g.W)), r = (int)(pix % ((size_t)g.H * g.W)), iy = r / g.W, ix = r % g.W;
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    for (int ky = 0; ky < g.KH; ++ky) {
      const int ty = iy + g.PH - ky;
      if (ty < 0 || ty % g.SH) continue;
      const int oy = ty / g.SH;
      if (oy >= g.OH) continue;
      for (int kx = 0; kx < g.KW; ++kx) {
        const int tx = ix + g.PW - kx;
        if (tx < 0 || tx % g.SW) continue;
        const int ox = tx / g.SW;
        if (ox >= g.OW) continue;
        const int tap = ky * g.KW + kx;
        const __nv_bfloat16* dp = dy + (((size_t)n * g.OH + oy) * g.OW + ox) * O;
#pragma unroll
        for (int o = 0; o < O; ++o) {
          const float d = __bfloat162float(dp[o]);
          float wf[8]; unpack8(__ldg(reinterpret_cast<const uint4*>(w + ((size_t)o * taps + tap) * g.C) + c8), wf);
#pragma unroll
          for (int k = 0; k < 8; ++k) acc[k] = fmaf(d, wf[k], acc[k]);
        }
      }
    }
    uint4 q; __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&q);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = c8 * 8 + 2 * k;
      h[k] = __floats2bfloat162_rn(act_fwd(act, acc[2 * k] + (bias ? bias[c] : 0.f), alpha), act_fwd(act, acc[2 * k + 1] + (bias ? bias[c + 1] : 0.f), alpha));
    }
    reinterpret_cast<uint4*>(dx)[i] = q;
  }
}

template <int O>
__global__ void __launch_bounds__(HW_THREADS) head_conv_wgrad_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy, float* __restrict__ part,
                                                                     const ConvGeom g, int per) {
  pdl_wait();
  const int C8 = g.C / 8, taps = g.KH * g.KW, col = blockIdx.x * HW_THREADS + threadIdx.x;
  if (col >= taps * C8) return;
  const int tap = col / C8, c8 = col % C8, ky = tap / g.KW, kx = tap % g.KW;
  const int P = g.N * g.OH * g.OW, p0 = min(P, blockIdx.y * per), p1 = min(P, p0 + per);
  float acc[O][8];
#pragma unroll
  for (int o = 0; o < O; ++o)
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[o][k] = 0.f;
  for (int pix = p0; pix < p1; ++pix) {
    const int n = pix / (g.OH * g.OW), r = pix % (g.OH * g.OW), oy = r / g.OW, ox = r % g.OW;
    const int iy = oy * g.SH - g.PH + ky, ix = ox * g.SW - g.PW + kx;
    if (iy < 0 || iy >= g.H || ix < 0 || ix >= g.W) continue;
    float xf[8]; unpack8(__ldg(reinterpret_cast<const uint4*>(x + (((size_t)n * g.H + iy) * g.W + ix) * g.C) + c8), xf);
#pragma unroll
    for (int o = 0; o < O; ++o) {
      const float d = __bfloat162float(dy[(size_t)pix * O + o]);
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[o][k] = fmaf(d, xf[k], acc[o][k]);
    }
  }
  const size_t nw = (size_t)O * taps * g.C;
#pragma unroll
  for (int o = 0; o < O; ++o) {
    float4* dst = reinterpret_cast<float4*>(part + blockIdx.y * nw + ((size_t)o * taps + tap) * g.C + c8 * 8);
    dst[0] = make_float4(acc[o][0], acc[o][1], acc[o][2], acc[o][3]);
    dst[1] = make_float4(acc[o][4], acc[o][5], acc[o][6], acc[o][7]);
  }
}

inline int col_blocks(const ConvGeom& g) { return (g.KH * g.KW * (g.C / 8) + HW_THREADS - 1) / HW_THREADS; }
// the production split target: two waves of weight-gradient blocks
inline int target_splits(const ConvGeom& g) { return std::max(1, (2 * device_sm_count() + col_blocks(g) - 1) / col_blocks(g)); }

#define HEAD_DISPATCH_O(O_, ...) \
  do { switch (O_) { case 1: { constexpr int OO = 1; __VA_ARGS__; } break; case 2: { constexpr int OO = 2; __VA_ARGS__; } break; \
                     case 3: { constexpr int OO = 3; __VA_ARGS__; } break; default: { constexpr int OO = 4; __VA_ARGS__; } break; } } while (0)

}  // namespace

bool head_conv_supported(const ConvGeom& g) {
  return g.O >= 1 && g.O <= 4 && g.C >= 8 && g.C % 8 == 0 && g.KH * g.KW > 1 && g.KH <= 7 && g.KW <= 7 && (g.SH == 1 || g.SH == 2) && (g.SW == 1 || g.SW == 2) &&
         g.PH >= 0 && g.PH < g.KH && g.PW >= 0 && g.PW < g.KW && g.OH * g.OW > 1 &&
         g.OH == (g.H + 2 * g.PH - g.KH) / g.SH + 1 && g.OW == (g.W + 2 * g.PW - g.KW) / g.SW + 1;
}

size_t k_head_wgrad_scratch_floats(const ConvGeom& g) {
  return head_conv_supported(g) ? (size_t)target_splits(g) * g.O * g.KH * g.KW * g.C : 0;
}

void k_head_fwd(const ConvGeom& g, const __nv_bfloat16* x, const __nv_bfloat16* w, const float* bias, __nv_bfloat16* out, int act, float alpha, cudaStream_t s) {
  const int P = g.N * g.OH * g.OW, blocks = std::max(1, std::min((P + 7) / 8, 8 * device_sm_count()));
  HEAD_DISPATCH_O(g.O, (launch_pdl(head_conv_fwd_kernel<OO>, dim3(blocks), dim3(256), (size_t)0, s, x, w, bias, out, g, act, alpha)));
  LAUNCHED(); g_gemm_last_kernel = "head_conv_fwd_kernel"; g_gemm_last_splits = 1;
}

void k_head_dgrad(const ConvGeom& g, const __nv_bfloat16* dy, const __nv_bfloat16* w, const float* bias, __nv_bfloat16* dx, int act, float alpha, cudaStream_t s) {
  const size_t total = (size_t)g.N * g.H * g.W * (g.C / 8);
  const int blocks = (int)std::max<size_t>(1, std::min<size_t>((total + 255) / 256, (size_t)16 * device_sm_count()));
  HEAD_DISPATCH_O(g.O, (launch_pdl(head_conv_dgrad_kernel<OO>, dim3(blocks), dim3(256), (size_t)0, s, dy, w, bias, dx, g, act, alpha)));
  LAUNCHED(); g_gemm_last_kernel = "head_conv_dgrad_kernel"; g_gemm_last_splits = 1;
}

int k_head_wgrad(const ConvGeom& g, const __nv_bfloat16* x, const __nv_bfloat16* dy, float* dw, float* part, size_t part_floats, int force_splits, cudaStream_t s,
                 ReduceList* defer) {
  const int P = g.N * g.OH * g.OW;
  const int splits = force_splits > 0 ? force_splits : std::max(1, std::min(target_splits(g), (P + 31) / 32));
  const int per = (P + splits - 1) / splits;
  const size_t nw = (size_t)g.O * g.KH * g.KW * g.C;
  if ((size_t)splits * nw > part_floats) return -1;
  HEAD_DISPATCH_O(g.O, (launch_pdl(head_conv_wgrad_kernel<OO>, dim3(col_blocks(g), splits), dim3(HW_THREADS), (size_t)0, s, x, dy, part, g, per)));
  LAUNCHED(); g_gemm_last_kernel = "head_conv_wgrad_kernel"; g_gemm_last_splits = splits;
  if (defer) reduce_list_push(defer, part, dw, (int64_t)nw, splits, (int64_t)nw);
  else k_reduce_splits(part, dw, nw, splits, nw, 0, s);
  return 0;
}

}  // namespace b2g
