// kernels_init.cu -- weight initialization (DL4J WeightInit / Distribution / biasInit): a layer's W drawn on the device from the counter-based
// generator, element by element at its DL4J view index, and its bias filled.  Definitions: include/b200gan.h b2g_weight_init; restatement:
// oracle/dl4j_oracle.py (weight_init_draw).  A translation unit of its own, so that no other kernel's generated code changes.
#include <stdint.h>
#include <algorithm>
#include "kernels.h"
#include "common.cuh"

namespace b2g {

// One thread per group of 4 consecutive view indices j = 4g .. 4g + 3, which share the Philox counter g of every round; each value is stored
// at its internal [A][taps][B] slot.  Threads g < n_bias also write bias element g.
__global__ void __launch_bounds__(256) weight_init_kernel(float* __restrict__ w, int64_t n, int taps, int B, const WiDraw d, float* __restrict__ bias,
                                                          int n_bias, float bias_init, uint32_t k0, uint32_t k1, uint32_t tag) { pdl_enter();
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (bias && g < n_bias) bias[g] = bias_init;
  const int64_t j0 = 4 * g;
  if (j0 >= n) return;
  const int m = n - j0 < 4 ? (int)(n - j0) : 4;
  const uint32_t c0 = (uint32_t)g;
  float v[4];
  switch (d.kind) {
    case WI_NORMAL: case WI_LOG_NORMAL: {
      float z[4]; normals4(philox4x32_10(c0, 0u, 0u, tag, k0, k1), z);
#pragma unroll
      for (int e = 0; e < 4; ++e) { v[e] = fmaf(d.b, z[e], d.a); if (d.kind == WI_LOG_NORMAL) v[e] = expf(v[e]); }
    } break;
    case WI_UNIFORM: {
      const Philox4 r = philox4x32_10(c0, 0u, 0u, tag, k0, k1);
      const float span = d.b - d.a;
#pragma unroll
      for (int e = 0; e < 4; ++e) v[e] = fmaf(span, (float)(r.x[e] >> 8) * 0x1p-24f, d.a);
    } break;
    case WI_TRUNCATED_NORMAL: {      // the first of 16 rounds with |z| <= 2; none: round 15's z clamped
      float z[4] = {0.f, 0.f, 0.f, 0.f}; unsigned todo = (1u << m) - 1u;
      for (uint32_t k = 0; k < 16 && todo; ++k) {
        float t[4]; normals4(philox4x32_10(c0, k, 0u, tag, k0, k1), t);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if (!((todo >> e) & 1u)) continue;
          if (fabsf(t[e]) <= 2.f) { z[e] = t[e]; todo &= ~(1u << e); }
          else if (k == 15) z[e] = fminf(fmaxf(t[e], -2.f), 2.f);
        }
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) v[e] = fmaf(d.b, z[e], d.a);
    } break;
    case WI_BINOMIAL: {              // round t is trial t: a success when its word is below floor(p 2^32)
      int c[4] = {0, 0, 0, 0};
      for (int t = 0; t < d.trials; ++t) {
        const Philox4 r = philox4x32_10(c0, (uint32_t)t, 0u, tag, k0, k1);
#pragma unroll
        for (int e = 0; e < 4; ++e) c[e] += (uint64_t)r.x[e] < d.thr ? 1 : 0;
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) v[e] = (float)c[e];
    } break;
    case WI_IDENTITY: {              // a square DENSE / OUTPUT W: j = o * nIn + i, one on the diagonal
#pragma unroll
      for (int e = 0; e < 4; ++e) { const int64_t j = j0 + e; v[e] = j / B == j % B ? 1.f : 0.f; }
    } break;
    default: {                       // CONSTANT (ZERO, ONES)
#pragma unroll
      for (int e = 0; e < 4; ++e) v[e] = d.a;
    }
  }
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    if (e >= m) break;
    const int64_t j = j0 + e;
    int64_t i = j;
    if (taps > 1) {                  // j = (a*B + b)*taps + t  ->  i = (a*taps + t)*B + b
      const int64_t ab = j / taps, a = ab / B, b = ab - a * B, t = j - ab * taps;
      i = (a * taps + t) * B + b;
    }
    w[i] = v[e];
  }
}

void k_weight_init(float* w, int A, int taps, int B, const WiDraw& d, float* bias, int n_bias, float bias_init, uint64_t seed, int layer, cudaStream_t s) {
  const int64_t n = (int64_t)A * taps * B, threads = std::max((n + 3) / 4, (int64_t)(bias ? n_bias : 0));
  if (threads <= 0) return;
  launch_pdl(weight_init_kernel, dim3((unsigned)((threads + 255) / 256)), dim3(256), (size_t)0, s, w, n, taps, B, d, bias, n_bias, bias_init,
             (uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)layer | 0x80000000u); LAUNCHED();
}

}  // namespace b2g
