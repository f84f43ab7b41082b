// kernels_gradnorm.cu -- DL4J's L2 gradient normalization (GradientNormalization.RenormalizeL2PerLayer / PerParamType, ClipL2PerLayer /
// PerParamType): the per-group L2 norms of the minibatch-divided gradient, and from them one multiplier per updater segment, which the
// updater kernel (kernels_ew.cu, SCALED instantiation) applies right after its minibatch division.  Semantics: include/b200gan.h
// (b2g_net_set_gradient_normalization); oracle restatement: tests/gradnorm_ref.py.
//
// A translation unit of its own, like kernels_dropout.cu: the unscaled updater kernel keeps the code nvcc generates for it without this kernel.
#include <stdint.h>
#include "kernels.h"
#include "common.cuh"

namespace b2g {

__device__ __forceinline__ double sq(float g, float gscale) { const double v = (double)(g * gscale); return v * v; }

__global__ void __launch_bounds__(256) gradnorm_kernel(const float* __restrict__ grads, const UpdSeg* __restrict__ segs, const int32_t* __restrict__ chunk_seg,
                                                       const int64_t* __restrict__ chunk_off, const GnGroup* __restrict__ groups, int ngroups, int clip,
                                                       float threshold, float inv_mb, float inv_world, double* partial, unsigned* ticket, float* __restrict__ mult) {
  pdl_enter();
  __shared__ double red[8];
  __shared__ int last;
  const UpdSeg& sg = segs[chunk_seg[blockIdx.x]];
  const int64_t base = chunk_off[blockIdx.x];
  const int64_t end = min(base + (int64_t)UPD_CHUNK, sg.off + sg.len);
  const float gscale = sg.div_mb ? inv_mb : inv_world;
  double acc = 0.0;
  if (((base | end) & 3) == 0) {      // 16-byte loads: a full chunk is four float4 per thread
    for (int64_t i = base + 4 * (int64_t)threadIdx.x; i < end; i += 4 * (int64_t)blockDim.x) {
      const float4 g = *reinterpret_cast<const float4*>(grads + i);
      acc += sq(g.x, gscale); acc += sq(g.y, gscale); acc += sq(g.z, gscale); acc += sq(g.w, gscale);
    }
  } else {
    for (int64_t i = base + threadIdx.x; i < end; i += blockDim.x) acc += sq(grads[i], gscale);
  }
  const double tot = block_sum(acc, red);
  if (threadIdx.x == 0) {
    partial[blockIdx.x] = tot;
    __threadfence();
    last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  // the last block: every partial is visible (each writer fenced before taking its ticket).  One warp per group; each lane sums a strided
  // subset of the group's partials in chunk order, then the warp's xor butterfly: lane 0's sum is the group's, the same on every run.
  __threadfence();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int gi = warp; gi < ngroups; gi += (int)(blockDim.x >> 5)) {
    const GnGroup gr = groups[gi];
    double s = 0.0;
    for (int c = gr.chunk_begin + lane; c < gr.chunk_end; c += 32) s += __ldcg(partial + c);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    s = __shfl_sync(0xffffffffu, s, 0);
    const double norm = sqrt(s);
    float m;
    if (clip) m = norm > (double)threshold ? (float)((double)threshold / norm) : 1.0f;
    else m = (float)(1.0 / (norm == 0.0 ? 1e-5 : norm));
    for (int k = gr.seg_begin + lane; k < gr.seg_end; k += 32) mult[k] = m;
  }
  if (threadIdx.x == 0) { *ticket = 0u; __threadfence(); }
}

void k_gradnorm(const float* grads, const UpdSeg* segs, const int32_t* chunk_seg, const int64_t* chunk_off, int nchunks, const GnGroup* groups, int ngroups,
                int clip, float threshold, float inv_mb, float inv_world, double* partial, unsigned* ticket, float* mult, cudaStream_t s) {
  if (!nchunks) return;
  launch_pdl(gradnorm_kernel, dim3(nchunks), dim3(256), (size_t)0, s, grads, segs, chunk_seg, chunk_off, groups, ngroups, clip, threshold, inv_mb, inv_world,
             partial, ticket, mult); LAUNCHED();
}

}  // namespace b2g
