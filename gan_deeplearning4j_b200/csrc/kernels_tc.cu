// kernels_tc.cu -- the tensor-core hot path: implicit-GEMM convolution / transposed convolution on sm_90a
// with TMA-staged shared-memory tiles and warpgroup MMAs (wgmma.mma_async: bf16 x bf16 -> fp32 accumulators in
// registers).  Hand-written PTX; no CUTLASS, no cuDNN.
//
// Replaces DL4J's ConvolutionLayer.preOutput / backpropGradient (im2col buffer + OpenBLAS sgemm + separate bias
// and activation passes; SURVEY.md section 8a rows a1, a2; reference call sites J:135-150, 203-219) for the
// DCGAN shapes of SURVEY.md Appendix B.
//
// A persistent, warp-specialised CTA of five warpgroups (one per SM) walks 128 x BN output tiles:
//   producer        one elected lane issues, per K-block, one 4-D tensor-map box for the activations (the im2col gather is done by the
//                   TMA unit: traversal strides give the stride-2 sampling, out-of-bounds coordinates give the zero padding) and the
//                   weight box(es), both landing 128B-swizzled in a STAGES-deep smem ring (mbarrier expect_tx), tile after tile
//   2 consumers     each owns 64 accumulator rows and issues 4 x wgmma m64nNk16 per K-block straight from the swizzled tiles via
//                   matrix descriptors, keeping one K-block in flight; at the end of a tile the accumulators are parked as fp32 in a
//                   park buffer and the consumers go on with the next tile
//   2 epilogue      one thread = one output pixel of the parked tile: + bias, activation, BatchNorm statistics, convert to bf16, 16-byte
//                   stores of the contiguous NHWC channel run -- overlapping the next tile's MMAs
// Modes: fprop (conv forward; also the input-gradient of a transposed conv) and dgrad (conv input-gradient = transposed
// conv forward) in sub-pixel phase form: a 4x4 stride-2 pad-1 transposed conv is four 2x2 stride-1 convs, one per output
// parity class, so no MAC is spent on inserted zeros and nothing is scattered.
#include <cuda.h>
#include <stdio.h>
#include <stdlib.h>
#include <algorithm>

#include "common.cuh"
#include "kernels.h"

namespace b2g {

// ------------------------------------------------------------------ driver entry point (no -lcuda) ------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled g_encode = nullptr;

int tc_init() {
  if (g_encode) return 0;
  void* fn = nullptr; cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess || !fn || q != cudaDriverEntryPointSuccess) return -1;
  g_encode = (PFN_encodeTiled)fn; return 0;
}

static int make_map_bf16(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes, const cuuint32_t* box, const cuuint32_t* estr) {
  if (!g_encode) return -1;
  CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), dims, strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { fprintf(stderr, "[b200gan] cuTensorMapEncodeTiled failed: %d (rank %d)\n", (int)r, rank); return -1; }
  return 0;
}

// ------------------------------------------------------------------ PTX wrappers --------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count)); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ int g_tc_timeout_flag = 0;
// bounded wait: a wrong expect_tx byte count or a bad descriptor must not hang the GPU -- trap instead
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  for (uint32_t it = 0; it < (1u << 26); ++it) {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    if (done) return;
  }
  g_tc_timeout_flag = 1; __trap();
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
               ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
               ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
// One lane of a CONVERGED warp (elect.sync): the producer loop is written as "whole warp runs the loop, the elected lane issues", so that
// the TMA instructions are emitted once, predicated, instead of inside a divergent branch.
__device__ __forceinline__ bool elect_one_sync() {
  uint32_t pred = 0;
  asm volatile("{\n\t.reg .pred P1;\n\t.reg .b32 rx;\n\telect.sync rx|P1, %1;\n\t@P1 mov.s32 %0, 1;\n\t}" : "+r"(pred) : "r"(0xffffffffu));
  return pred != 0;
}
__device__ __forceinline__ void prefetch_map(const CUtensorMap* map) { asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory"); }
// generic-proxy writes to shared memory (tiles built by the threads themselves) become visible to wgmma, which reads through the async proxy
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// Shared-memory matrix descriptor of wgmma (sm_90): start address >> 4 in [0,14), leading byte offset >> 4 in [16,30), stride byte
// offset >> 4 in [32,46), base offset in [49,52) (0: tiles are 1024-byte aligned), layout type in [62,64) (1 = SWIZZLE_128B).
//   K-major tile (rows of 128 B = 64 bf16 of the reduction): 8-row groups 1024 B apart (SBO), LBO unused.  A K step of 16 inside the
//   128-byte swizzle atom is +32 B = +2 in the start-address field.
//   MN-major tile ([K rows][64 MN elements], 128 B per row): 8-K-row groups 1024 B apart (SBO), 64-element MN blocks `lbo` apart (LBO);
//   a K step of 16 is 16 rows = +2048 B.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
__device__ __forceinline__ uint64_t desc_kmajor_sw128(uint32_t saddr) { return gmma_desc(saddr, 16); }
__device__ __forceinline__ uint64_t desc_mnmajor_sw128(uint32_t saddr, uint32_t lbo_bytes) { return gmma_desc(saddr, lbo_bytes); }

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x 64] += A[64 x 16] B[16 x 64], both operands in shared memory; TA / TB = 1: that operand is MN-major.
// Accumulator fragment (thread t of the warpgroup, w = t / 32, l = t % 32): d[4j + 2i + k] = D[16w + l/4 + 8i][8j + 2(l%4) + k].
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t da, uint64_t db) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, 1, 1, 1, %34, %35;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
        "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]),
        "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "n"(TA), "n"(TB));
}
// the same with N = 16 (pixel-shuffle tile): d[4j + 2i + k], j < 2
__device__ __forceinline__ void wgmma_n16(float (&d)[8], uint64_t da, uint64_t db) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, 1, 1, 1, 0, 0;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(da), "l"(db));
}


// ------------------------------------------------------------------ conv fprop / dgrad-phase kernels -------
// Epilogue modes (runtime, warp-uniform):
//   EPI_PLAIN   out = act(acc * scale[c] + bias[c])                 (scale / bias optional: inference-mode BatchNorm folded in)
//   EPI_STATS   EPI_PLAIN + per-(group, channel) sum / sum of squares of the bf16-rounded outputs: the train-mode BatchNorm
//               statistics of the layer that follows come out of the producing GEMM (SURVEY section 7 step 5, J:132-134,197-199)
//   EPI_BNBWD   the GEMM produces the epsilon w.r.t. the OUTPUT y of a BatchNorm(+activation) layer; the epilogue reads y and that
//               layer's input z at the same pixel, out = eps * act'(y) (derivative from the stored output: no per-channel
//               coefficients in the epilogue) and accumulates sum(out), sum(out * z): the two reductions of BatchNorm backward fall
//               out of the dgrad epilogue (the consumer turns sum(out*z) into sum(out*xhat) = invstd*(sum(out*z) - mean*sum(out)) in double)
//   EPI_ACTBWD  out = eps * act'(a) with a = the forward output of the layer below (D1's LeakyReLU, G-last's tanh)
// Statistics: 32 rows x 32 columns per warp are column-reduced by a shuffle butterfly (31 shuffles per statistic), the four row
// quadrants are folded through shared memory in fixed order, and one value per (tile, channel) is added into a 128-bit
// fixed-point accumulator with two 64-bit integer atomics (common.cuh sacc_add): integer addition commutes, so the result is
// bit-reproducible whatever order the CTAs arrive in, and there is no partial buffer and no finalise kernel.

struct TcConvParams {
  int mode;                 // 0 = fprop, 1 = dgrad in sub-pixel phase form (4x4 s2 p1)
  int Nt, Ht, Wt;           // A-tile rows = Nt images x Ht rows x Wt cols of the row grid (Nt*Ht*Wt = 128)
  int GH, GW;               // row grid: conv output (fprop) / phase grid = dy spatial dims (dgrad)
  int tiles_y;              // GH / Ht
  int taps_h, taps_w;       // K-loop taps: KH,KW (fprop) / 2,2 (dgrad phase)
  int chunks;               // reduction channels / 64
  int KW, SH, SW, PH, PW;
  int OC;                   // output channels = row length of `out`
  int outH, outW;           // spatial dims of `out`
  int b_mn;                 // 1: the weight tile is MN-major (rows = reduction index, 64 output channels contiguous): the straight
                            //    [O][taps][C] copy serves the dgrad form too, no transposed weight copy exists
  const float* bias; const float* scale; int act; float alpha;     // EPI_PLAIN / EPI_STATS
  __nv_bfloat16* out;
  int epi;
  unsigned long long* acc;  // EPI_STATS / EPI_BNBWD: [groups][2][2][OC] (statistic, hi | lo, channel)
  int imgs_per_group;
  const __nv_bfloat16* aux; // EPI_BNBWD / EPI_ACTBWD: the forward output whose act' multiplies the result   (same NHWC shape as `out`)
  const __nv_bfloat16* aux2;// EPI_BNBWD: the BatchNorm input z
  int tiles_m, tiles_n, phases;   // work items: tile t = ((phase * tiles_n) + n tile) * tiles_m + m tile
};

static constexpr int TC_THREADS = 384;       // tc_wgrad_kernel: producer warpgroup + two consumer warpgroups
static constexpr int TC_CONV_THREADS = 640;  // tc_conv_kernel: two MMA consumer warpgroups, two epilogue warpgroups, a producer warpgroup
template <int BN, int STAGES, int EPI = EPI_PLAIN>
struct TcSmem {
  static constexpr int A_BYTES = 128 * 128;        // 128 rows x 64 bf16
  static constexpr int B_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int RING_BYTES = STAGES * STAGE_BYTES;
  static constexpr int ACC_PITCH = BN + 4;         // floats per parked accumulator row: 16-byte row reads by 8 lanes hit 8 different bank groups
  static constexpr int PARK_BYTES = 128 * ACC_PITCH * 4;
  static constexpr int PARKS = BN >= 128 ? 1 : 2;  // accumulator park slots: two where shared memory allows (a 128-column tile has one)
  static constexpr int PARK_OFF = RING_BYTES;
  static constexpr int BAR_OFF = PARK_OFF + PARKS * PARK_BYTES;
  static constexpr int STAT_OFF = BAR_OFF + 256;
  static constexpr int STG_OFF = STAT_OFF + ((EPI == EPI_STATS || EPI == EPI_BNBWD) ? 4 * 2 * BN * 4 : 0);
  static constexpr int TOTAL = STG_OFF + (BN >= 32 ? 8 * 2048 : 0) + 1024;   // + barriers + statistics + epilogue staging + alignment slack
  static_assert(TOTAL <= 227 * 1024, "one CTA per SM must fit the shared memory of an sm_90 SM");
};

__device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }    // the eight epilogue warps only
template <int N> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

// column sums over the 32 lanes of a warp: on return lane l holds sum_lanes a[l] in a[0].  One butterfly level per template instance, so
// that every index into `a` is a compile-time constant and the array stays in registers (a runtime loop over the level puts it on the stack).
template <int OFF>
__device__ __forceinline__ void warp_colsum_level(float (&a)[32], int lane) {
  const bool up = (lane & OFF) != 0;
#pragma unroll
  for (int j = 0; j < OFF; ++j) {
    const float lo = a[j], hi = a[j + OFF];
    const float send = up ? lo : hi, keep = up ? hi : lo;
    a[j] = keep + __shfl_xor_sync(0xffffffffu, send, OFF);
  }
  if constexpr (OFF > 1) warp_colsum_level<OFF / 2>(a, lane);
}
__device__ __forceinline__ void warp_colsum32(float (&a)[32], int lane) { warp_colsum_level<16>(a, lane); }

// Columns [c_beg, c_end) of one 128-row accumulator tile: parked fp32 row -> registers -> epilogue arithmetic -> bf16 -> global.
// srow = this thread's parked accumulator row; roff = element offset of (pixel, first channel of the tile) in `out`.
// A thread owns one accumulator row, but a warp instruction in which every lane touches its own row costs the load/store unit 32
// wavefronts of 16 B each.  Global traffic therefore goes through a per-warp 2 KB staging area `stg` ([32 rows][4 x 16 B], XOR-swizzled so
// that both access patterns are bank-conflict free): four lanes cover the 64 B of one row, a warp instruction covers 8 rows = 16 full
// sectors.  The same transposition brings the auxiliary operands (forward output y, BN input z) in, 32 columns at a time (loading the next
// 32 ahead would keep 32 more registers live than the epilogue warpgroups have; their latency overlaps the next tile's MMAs instead).
template <int BN, int EPI, bool AFFINE>
__device__ __forceinline__ void epi_tile(const TcConvParams& p, const float* srow, size_t roff, int nb0, int group, float* sst, uint4* stg, int q, int lane, int ep_tid,
                                         int c_beg, int c_end) {
  constexpr bool stats = EPI == EPI_STATS || EPI == EPI_BNBWD;
  const bool has_bias = p.bias != nullptr;
  const int sub = lane >> 2, cq = lane & 3, sx = (lane >> 1) & 3;
  size_t roff_i[4];                      // element offsets of the rows this lane serves in the transposed pattern: row i*8 + lane/4
#pragma unroll
  for (int i = 0; i < 4; ++i) roff_i[i] = __shfl_sync(0xffffffffu, (unsigned long long)roff, i * 8 + sub) + cq * 8;
#pragma unroll 1
  for (int c0 = c_beg; c0 < c_end; c0 += 32) {
    uint32_t v[32];
    uint4 gy[4], gz[4], ax[4], az[4];
    if constexpr (EPI >= EPI_BNBWD) {
#pragma unroll
      for (int i = 0; i < 4; ++i) gy[i] = *reinterpret_cast<const uint4*>(p.aux + roff_i[i] + c0);
    }
    if constexpr (EPI == EPI_BNBWD) {
#pragma unroll
      for (int i = 0; i < 4; ++i) gz[i] = *reinterpret_cast<const uint4*>(p.aux2 + roff_i[i] + c0);
    }
    if constexpr (EPI >= EPI_BNBWD) {
#pragma unroll
      for (int i = 0; i < 4; ++i) { const int r = i * 8 + sub; stg[r * 4 + (cq ^ ((r >> 1) & 3))] = gy[i]; }
      __syncwarp();
#pragma unroll
      for (int j = 0; j < 4; ++j) ax[j] = stg[lane * 4 + (j ^ sx)];
      __syncwarp();
    }
    if constexpr (EPI == EPI_BNBWD) {
#pragma unroll
      for (int i = 0; i < 4; ++i) { const int r = i * 8 + sub; stg[r * 4 + (cq ^ ((r >> 1) & 3))] = gz[i]; }
      __syncwarp();
#pragma unroll
      for (int j = 0; j < 4; ++j) az[j] = stg[lane * 4 + (j ^ sx)];
      __syncwarp();
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) { const uint4 t = reinterpret_cast<const uint4*>(srow + c0)[j]; v[4 * j] = t.x; v[4 * j + 1] = t.y; v[4 * j + 2] = t.z; v[4 * j + 3] = t.w; }
    float o[32], s2[32];
    if constexpr (EPI == EPI_BNBWD) {
      const __nv_bfloat162* yb = reinterpret_cast<const __nv_bfloat162*>(ax);
      const __nv_bfloat162* zb = reinterpret_cast<const __nv_bfloat162*>(az);
#define B2G_BNBWD_LOOP(ACTC)                                                                                                   \
  _Pragma("unroll") for (int j = 0; j < 16; ++j) {                                                                             \
    const float2 y2 = __bfloat1622float2(yb[j]), z2 = __bfloat1622float2(zb[j]);                                               \
    o[2 * j] = __uint_as_float(v[2 * j]) * act_grad_from_out(ACTC, y2.x, p.alpha);                                             \
    o[2 * j + 1] = __uint_as_float(v[2 * j + 1]) * act_grad_from_out(ACTC, y2.y, p.alpha);                                     \
    s2[2 * j] = z2.x; s2[2 * j + 1] = z2.y;                                                                                    \
  }
      if (p.act == ACT_LRELU) { B2G_BNBWD_LOOP(ACT_LRELU) }
      else if (p.act == ACT_RELU) { B2G_BNBWD_LOOP(ACT_RELU) }
      else { B2G_BNBWD_LOOP(p.act) }
#undef B2G_BNBWD_LOOP
    } else if constexpr (EPI == EPI_ACTBWD) {
      const __nv_bfloat162* ab = reinterpret_cast<const __nv_bfloat162*>(ax);
#define B2G_ACTBWD_LOOP(ACTC)                                                                                                  \
  _Pragma("unroll") for (int j = 0; j < 16; ++j) {                                                                             \
    const float2 a2 = __bfloat1622float2(ab[j]);                                                                               \
    o[2 * j] = __uint_as_float(v[2 * j]) * act_grad_from_out(ACTC, a2.x, p.alpha);                                             \
    o[2 * j + 1] = __uint_as_float(v[2 * j + 1]) * act_grad_from_out(ACTC, a2.y, p.alpha);                                     \
  }
      if (p.act == ACT_LRELU) { B2G_ACTBWD_LOOP(ACT_LRELU) }
      else if (p.act == ACT_TANH) { B2G_ACTBWD_LOOP(ACT_TANH) }
      else { B2G_ACTBWD_LOOP(p.act) }
#undef B2G_ACTBWD_LOOP
    } else {
      // the activation switch is hoisted out of the 32-column loop: one uniform branch per chunk instead of one per element
#define B2G_EPI_LOOP(ACTC)                                                                                                     \
  _Pragma("unroll") for (int j = 0; j < 32; ++j) {                                                                             \
    float a = __uint_as_float(v[j]);                                                                                           \
    if (AFFINE) a = fmaf(a, p.scale[nb0 + c0 + j], p.bias[nb0 + c0 + j]);                                                      \
    else if (has_bias) a += p.bias[nb0 + c0 + j];                                                                              \
    o[j] = act_fwd(ACTC, a, p.alpha);                                                                                          \
  }
      if (p.act == ACT_IDENTITY) { B2G_EPI_LOOP(ACT_IDENTITY) }
      else if (p.act == ACT_LRELU) { B2G_EPI_LOOP(ACT_LRELU) }
      else if (p.act == ACT_RELU) { B2G_EPI_LOOP(ACT_RELU) }
      else { B2G_EPI_LOOP(p.act) }
#undef B2G_EPI_LOOP
    }
    uint32_t packed[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      __nv_bfloat162 h = __floats2bfloat162_rn(o[2 * j], o[2 * j + 1]);
      packed[j] = *reinterpret_cast<uint32_t*>(&h);
      if constexpr (stats) { const float2 r = __bfloat1622float2(h); o[2 * j] = r.x; o[2 * j + 1] = r.y; }      // statistics of what is stored
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) stg[lane * 4 + (j ^ sx)] = make_uint4(packed[4 * j], packed[4 * j + 1], packed[4 * j + 2], packed[4 * j + 3]);
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 4; ++i) { const int r = i * 8 + sub; *reinterpret_cast<uint4*>(p.out + roff_i[i] + c0) = stg[r * 4 + (cq ^ ((r >> 1) & 3))]; }
    __syncwarp();
    if constexpr (stats) {
      if constexpr (EPI == EPI_STATS) {
#pragma unroll
        for (int j = 0; j < 32; ++j) s2[j] = o[j] * o[j];
      } else {
#pragma unroll
        for (int j = 0; j < 32; ++j) s2[j] = o[j] * s2[j];
      }
      warp_colsum32(o, lane); warp_colsum32(s2, lane);
      sst[(q * 2 + 0) * BN + c0 + lane] = o[0];
      sst[(q * 2 + 1) * BN + c0 + lane] = s2[0];
    }
  }
  if constexpr (stats) {
    epi_bar_sync();
    for (int col = ep_tid; col < BN; col += 256) {
#pragma unroll
      for (int st = 0; st < 2; ++st) {
        const float s = ((sst[(0 * 2 + st) * BN + col] + sst[(1 * 2 + st) * BN + col]) + sst[(2 * 2 + st) * BN + col]) + sst[(3 * 2 + st) * BN + col];
        sacc_add(p.acc + (size_t)(group * 2 + st) * 2 * p.OC, (size_t)p.OC, (size_t)(nb0 + col), s);
      }
    }
  }
}

// weight tile of one K-block: K-major = one 3-D box {64 k, 1 tap, BN rows}; MN-major = BN/64 boxes {64 n, 1 tap, 64 k rows}
template <int BN>
__device__ __forceinline__ void load_b_tile(const TcConvParams& p, const CUtensorMap* tmB, uint32_t dst, uint32_t bar, int ch, int wtap, int nb0) {
  if (!p.b_mn) tma_load_3d(dst, tmB, bar, ch * 64, wtap, nb0);
  else {
#pragma unroll
    for (int j = 0; j < (BN >= 64 ? BN / 64 : 1); ++j) tma_load_3d(dst + j * 8192, tmB, bar, nb0 + j * 64, wtap, ch * 64);
  }
}
// the 4 x (K = 16) MMAs of one K-block for one consumer warpgroup: its 64 A rows start at a_smem; N = 64 per instruction (16 for the
// pixel-shuffle tile), the n-th 64-column block of the weight tile 8 KB further in both layouts
template <int BN, int NB, int NACC>
__device__ __forceinline__ void mma_kblock(float (&acc)[NB][NACC], uint32_t a_smem, uint32_t b_smem, int b_mn) {
  const uint64_t adesc = desc_kmajor_sw128(a_smem);
  if constexpr (BN < 64) {
    const uint64_t bdesc = desc_kmajor_sw128(b_smem);
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_n16(acc[0], adesc + 2 * k, bdesc + 2 * k);
  } else if (!b_mn) {
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int nb = 0; nb < NB; ++nb) wgmma_n64<0, 0>(acc[nb], adesc + 2 * k, desc_kmajor_sw128(b_smem + nb * 8192) + 2 * k);
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int nb = 0; nb < NB; ++nb) wgmma_n64<0, 1>(acc[nb], adesc + 2 * k, desc_mnmajor_sw128(b_smem + nb * 8192 + k * 2048, 8192));
  }
}
__device__ __forceinline__ void tap_coords(const TcConvParams& p, int ta, int tb, int py, int px, int& ax, int& dy_, int& wtap) {
  if (p.mode == 0) { dy_ = -p.PH + ta; ax = -p.PW + tb; wtap = ta * p.KW + tb; }
  else {
    // output row 2*q+py takes filter rows r with (py+1-r) even: py=0 -> r=1 (dy row q), r=3 (q-1); py=1 -> r=0 (q+1), r=2 (q)
    const int r = py == 0 ? (ta == 0 ? 1 : 3) : (ta == 0 ? 0 : 2), dyr = py == 0 ? (ta == 0 ? 0 : -1) : (ta == 0 ? 1 : 0);
    const int sx = px == 0 ? (tb == 0 ? 1 : 3) : (tb == 0 ? 0 : 2), dxc = px == 0 ? (tb == 0 ? 0 : -1) : (tb == 0 ? 1 : 0);
    dy_ = dyr; ax = dxc; wtap = r * 4 + sx;
  }
}

// Persistent and warp-specialised: CTA b walks the work items t = b, b + gridDim.x, ... (one 128 x BN output tile of one phase each).
//   warpgroups 0-1  MMA consumers: 64 accumulator rows each; at the end of a tile's K loop they park the fp32 fragments in a park slot (not the
//                   ring), arrive on "park full" and go straight on to the next tile
//   warpgroups 2-3  epilogue: wait on "park full", run epi_tile (or the pixel-shuffle scatter) from the slot, arrive on "park empty"
//   warpgroup 4     TMA producer (one warp): the K-blocks of all of the CTA's tiles as one stream through the ring, so the next tile's loads are in flight
//                   before the current tile's K loop ends
// so the epilogue of tile i runs while the MMAs of tile i+1 are issued.  The per-tile arithmetic and summation order are those of a
// one-tile CTA: results do not depend on the grid size.
// PS ("pixel shuffle", BN = 16): the 4x4 stride-2 pad-1 transposed conv onto <= 4 image channels (G-last forward, D1 input gradient) as ONE
// 3x3 stride-1 pad-1 convolution whose 16 output columns are (py, px, c) = the 2x2 output block x 4 (padded) channels: the four
// sub-pixel phases share every activation load (9 taps instead of 4 x 4), the packed weight [16][9][O] holds zeros where a
// (tap, phase) pair does not meet; the epilogue scatters its 16 values to the 2x2 block of the NHWC image.
// Registers per thread after setmaxnreg.  Each SM sub-partition holds one warp of every warpgroup and 64 KB of registers, so the launch
// gives 96 per thread (16384 / (5 x 32), in steps of 8) and PRODUCER + 2 MMA + 2 EPI must stay within 5 x 96.  128 accumulator columns
// need 96 in the MMA warpgroups (at 88 ptxas serialises the wgmmas).
template <int BN>
struct TcConvRegs {
  static constexpr int LAUNCH = 96, PRODUCER = 24, MMA = BN >= 128 ? 96 : 64, EPI = BN >= 128 ? 128 : 160;
  static_assert(PRODUCER + 2 * MMA + 2 * EPI <= 5 * LAUNCH, "setmaxnreg budget exceeds the launch allocation");
};
template <int BN, int STAGES, int EPI, bool AFFINE, bool PS = false>
__global__ void __launch_bounds__(TC_CONV_THREADS, 1) tc_conv_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const TcConvParams p) {
  using S = TcSmem<BN, STAGES, EPI>;
  using R = TcConvRegs<BN>;
  constexpr int NB = BN >= 64 ? BN / 64 : 1, NACC = BN >= 64 ? 32 : BN / 2;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  const uint32_t bar_full = smem_base + S::BAR_OFF;                 // STAGES x 8 B
  const uint32_t bar_empty = bar_full + 8 * STAGES;                 // STAGES x 8 B
  const uint32_t park_full = bar_empty + 8 * STAGES;                // PARKS x 8 B
  const uint32_t park_empty = park_full + 8 * S::PARKS;             // PARKS x 8 B
  float* sst = reinterpret_cast<float*>(smem_gen + S::STAT_OFF);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_kb = p.taps_h * p.taps_w * p.chunks;
  const int tiles = p.tiles_m * p.tiles_n * p.phases;
  // work item -> first output channel, phase, and the first image / row of its 128-row tile
  auto tile_coords = [&](int t, int& nb0, int& phase, int& n0, int& y0) {
    const int mt = t % p.tiles_m, r = t / p.tiles_m;
    nb0 = (r % p.tiles_n) * BN; phase = r / p.tiles_n;
    if (p.Nt > 1) { n0 = mt * p.Nt; y0 = 0; } else { n0 = mt / p.tiles_y; y0 = (mt % p.tiles_y) * p.Ht; }
  };

  if (threadIdx.x == 0) {
    prefetch_map(&tmA); prefetch_map(&tmB);
    for (int s = 0; s < STAGES; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, 8); }    // 8 consumer warps release a stage
    for (int k = 0; k < S::PARKS; ++k) { mbar_init(park_full + 8 * k, 256); mbar_init(park_empty + 8 * k, 256); }   // every consumer / epilogue thread
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();         // barrier init above overlaps the predecessor's tail; global memory is touched only below

  if (warp >= 16) {
    setmaxnreg_dec<R::PRODUCER>();
    if (warp == 16) {
      // ===== TMA producer (converged warp, elected lane issues): no integer division inside the K loop -- ring slot, channel chunk and tap advance as counters =====
      int s = 0; uint32_t ph = 0;
      for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
        int nb0, phase, n0, y0; tile_coords(t, nb0, phase, n0, y0);
        const int py = phase >> 1, px = phase & 1;
        const int ybase = p.mode == 0 ? y0 * p.SH : y0;
        int ch = 0, ta = 0, tb = 0;
        int ax, dy_, wtap; tap_coords(p, 0, 0, py, px, ax, dy_, wtap);
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(bar_empty + 8 * s, ph ^ 1);
          if (elect_one_sync()) {
            mbar_expect_tx(bar_full + 8 * s, S::STAGE_BYTES);
            tma_load_4d(smem_base + s * S::STAGE_BYTES, &tmA, bar_full + 8 * s, ch * 64, ax, ybase + dy_, n0);
            load_b_tile<BN>(p, &tmB, smem_base + s * S::STAGE_BYTES + S::A_BYTES, bar_full + 8 * s, ch, wtap, nb0);
          }
          __syncwarp();
          if (++s == STAGES) { s = 0; ph ^= 1; }
          if (++ch == p.chunks) { ch = 0; if (++tb == p.taps_w) { tb = 0; ++ta; } tap_coords(p, ta, tb, py, px, ax, dy_, wtap); }
        }
      }
    }
  } else if (warp < 8) {
    if constexpr (R::MMA < R::LAUNCH) setmaxnreg_dec<R::MMA>();
    // ===== MMA consumers: warpgroup wg owns accumulator rows [64 wg, 64 wg + 64) =====
    const int wg = warp >> 2;
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    int s = 0, k = 0; uint32_t ph = 0, kph = 0;
    for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
      float acc[NB][NACC];
#pragma unroll
      for (int nb = 0; nb < NB; ++nb)
#pragma unroll
        for (int j = 0; j < NACC; ++j) acc[nb][j] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(bar_full + 8 * s, ph);
        wg_fence();
        const uint32_t st = smem_base + s * S::STAGE_BYTES;
        mma_kblock<BN, NB, NACC>(acc, st + wg * 8192, st + S::A_BYTES, PS ? 0 : p.b_mn);
        wg_commit();
        wg_wait<1>();                                   // the previous K-block's MMAs are done: its stage goes back to the producer
        if (prev >= 0 && lane == 0) mbar_arrive(bar_empty + 8 * prev);
        prev = s;
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
      wg_wait<0>();
      if (lane == 0) mbar_arrive(bar_empty + 8 * prev);
      mbar_wait(park_empty + 8 * k, kph ^ 1);           // the epilogue is done with the tile parked in this slot before
      float* park = reinterpret_cast<float*>(smem_gen + S::PARK_OFF + k * S::PARK_BYTES);
#pragma unroll
      for (int nb = 0; nb < NB; ++nb)
#pragma unroll
        for (int j = 0; j < NACC / 4; ++j) {
          const int col = nb * 64 + j * 8 + 2 * (lane & 3);
          *reinterpret_cast<float2*>(park + r0 * S::ACC_PITCH + col) = make_float2(acc[nb][4 * j], acc[nb][4 * j + 1]);
          *reinterpret_cast<float2*>(park + (r0 + 8) * S::ACC_PITCH + col) = make_float2(acc[nb][4 * j + 2], acc[nb][4 * j + 3]);
        }
      mbar_arrive(park_full + 8 * k);
      if (++k == S::PARKS) { k = 0; kph ^= 1; }
    }
  } else {
    setmaxnreg_inc<R::EPI>();
    // ===== epilogue: warp ew serves parked rows [32 q, 32 q + 32) (q = ew % 4), column half ew / 4 =====
    const int ew = warp - 8, q = ew & 3, half = ew >> 2;
    const int row = q * 32 + lane;
    const int img = row / (p.Ht * p.Wt), rem = row % (p.Ht * p.Wt), yy = rem / p.Wt, xx = rem % p.Wt;
    int k = 0; uint32_t kph = 0;
    for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
      int nb0, phase, n0, y0; tile_coords(t, nb0, phase, n0, y0);
      const int py = phase >> 1, px = phase & 1;
      const int n = n0 + img, gy = y0 + yy, gx = xx;
      mbar_wait(park_full + 8 * k, kph);
      const float* srow = reinterpret_cast<const float*>(smem_gen + S::PARK_OFF + k * S::PARK_BYTES) + row * S::ACC_PITCH;
      if constexpr (PS) {
        if (half == 0) {
          const int C = p.OC;
#pragma unroll
          for (int ppy = 0; ppy < 2; ++ppy) {
            const size_t doff = (((size_t)n * p.outH + 2 * gy + ppy) * p.outW + 2 * gx) * C;
            __nv_bfloat16* dst = p.out + doff;
            float o[8];
#pragma unroll
            for (int ppx = 0; ppx < 2; ++ppx)
#pragma unroll
              for (int c = 0; c < 4; ++c) {
                float a = srow[(ppy * 2 + ppx) * 4 + c];
                if constexpr (EPI == EPI_ACTBWD) { if (c < C) a *= act_grad_from_out(p.act, __bfloat162float(p.aux[doff + ppx * C + c]), p.alpha); }
                else { if (p.bias && c < C) a += p.bias[c]; a = act_fwd(p.act, a, p.alpha); }
                o[ppx * 4 + c] = a;
              }
            if (C == 3) {         // 6 contiguous bf16 = three aligned 32-bit stores
              __nv_bfloat162 h0 = __floats2bfloat162_rn(o[0], o[1]), h1 = __floats2bfloat162_rn(o[2], o[4]), h2 = __floats2bfloat162_rn(o[5], o[6]);
              uint32_t* d32 = reinterpret_cast<uint32_t*>(dst);
              d32[0] = *reinterpret_cast<uint32_t*>(&h0); d32[1] = *reinterpret_cast<uint32_t*>(&h1); d32[2] = *reinterpret_cast<uint32_t*>(&h2);
            } else {
#pragma unroll
              for (int ppx = 0; ppx < 2; ++ppx)
#pragma unroll
                for (int c = 0; c < 4; ++c) if (c < C) dst[ppx * C + c] = __float2bfloat16(o[ppx * 4 + c]);
            }
          }
        }
      } else {
        size_t pix;
        if (p.mode == 0) pix = ((size_t)n * p.outH + gy) * p.outW + gx;
        else pix = ((size_t)n * p.outH + 2 * gy + py) * p.outW + 2 * gx + px;
        const int group = p.imgs_per_group > 0 ? n0 / p.imgs_per_group : 0;
        epi_tile<BN, EPI, AFFINE>(p, srow, pix * p.OC + nb0, nb0, group, sst, reinterpret_cast<uint4*>(smem_gen + S::STG_OFF) + ew * 128, q, lane,
                                  (int)threadIdx.x - 256, half * (BN / 2), (half + 1) * (BN / 2));
        if constexpr (EPI == EPI_STATS || EPI == EPI_BNBWD) epi_bar_sync();   // every epilogue warp has read sst before the next tile rewrites it
      }
      mbar_arrive(park_empty + 8 * k);
      if (++k == S::PARKS) { k = 0; kph ^= 1; }
    }
  }
}

// ------------------------------------------------------------------ host side ------------------------------
const char* g_tc_last_kernel = "";       // name of the tensor-core kernel the most recent k_tc_* call dispatched (parity tests assert it)
int g_tc_test_bn = 0, g_tc_test_max_ctas = 0;   // test-hook schedule overrides (kernels.h); production code never sets them
static int tc_device() { int dev = 0; cudaGetDevice(&dev); return dev < 0 || dev >= 64 ? 0 : dev; }
// cudaFuncAttributeMaxDynamicSharedMemorySize is per device: one flag per (kernel, device)
#define TC_SET_SMEM_ONCE(kernel, bytes)                                                                                            \
  do { static bool set_[64] = {}; const int d_ = tc_device();                                                                       \
       if (!set_[d_]) { if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes)) != cudaSuccess) return -2; set_[d_] = true; } } while (0)

static bool pick_row_tile(int N, int GH, int GW, int rows, int* Nt, int* Ht, int* Wt) {
  const int P = GH * GW;
  if (GW > rows || rows % GW) return false;
  if (P >= rows) { if (P % rows) return false; *Nt = 1; *Ht = rows / GW; *Wt = GW; return GH % *Ht == 0; }
  if (rows % P || N % (rows / P)) return false;
  *Nt = rows / P; *Ht = GH; *Wt = GW; return true;
}
// N tiles of at most 128 columns: two consumer warpgroups x 64 rows x 128 fp32 accumulators = 64 registers per thread
static int pick_bn(int OC) { return OC % 128 == 0 ? 128 : OC % 64 == 0 ? 64 : 0; }
// Small layers (few M tiles) are latency-bound per CTA, not bandwidth-bound: prefer narrower N tiles until the grid covers the SMs.
static int pick_bn_fill(int OC, long m_tiles_x_phases) {
  if (g_tc_test_bn) return g_tc_test_bn;
  static int min_ctas = -1; if (min_ctas < 0) { const char* e = getenv("B2G_BN_MIN_CTAS"); min_ctas = e ? atoi(e) : 0; }
  const int target = min_ctas >= 1 ? min_ctas : device_sm_count();
  int bn = pick_bn(OC);
  while (bn > 64 && m_tiles_x_phases * (OC / bn) < target) bn /= 2;
  return bn;
}

bool tc_fprop_supported(const ConvGeom& g) {
  int a, b, c;
  return g.C % 64 == 0 && pick_bn(g.O) != 0 && g.SH >= 1 && g.SH <= 2 && g.SW == g.SH && g.KH * g.KW * (g.C / 64) >= 1 &&
         pick_row_tile(g.N, g.OH, g.OW, 128, &a, &b, &c) && c * g.SW <= 256 && b * g.SH <= 256 && g.N >= 1;
}
bool tc_dgrad_supported(const ConvGeom& g) {
  int a, b, c;
  return g.KH == 4 && g.KW == 4 && g.SH == 2 && g.SW == 2 && g.PH == 1 && g.PW == 1 && g.O % 64 == 0 && pick_bn(g.C) != 0 && g.H == 2 * g.OH && g.W == 2 * g.OW &&
         pick_row_tile(g.N, g.OH, g.OW, 128, &a, &b, &c);
}
// the fused BatchNorm epilogues need every 128-row tile inside one statistics group
static bool tc_epi_ok(const TcEpi* e, int Nt) { return !e || e->mode == EPI_PLAIN || e->mode == EPI_ACTBWD || (e->imgs_per_group > 0 && e->imgs_per_group % Nt == 0 && e->acc); }

// persistent grid: one CTA per SM, or one per work item when there are fewer (a test may cap it at g_tc_test_max_ctas instead)
template <int BN, int STAGES, int EPI, bool AFFINE, bool PS = false>
static int launch_conv_e(const CUtensorMap& tmA, const CUtensorMap& tmB, const TcConvParams& p, cudaStream_t s) {
  using S = TcSmem<BN, STAGES, EPI>;
  TC_SET_SMEM_ONCE((tc_conv_kernel<BN, STAGES, EPI, AFFINE, PS>), S::TOTAL);
  const long tiles = (long)p.tiles_m * p.tiles_n * p.phases;
  const unsigned grid = (unsigned)std::min<long>(tiles, g_tc_test_max_ctas > 0 ? g_tc_test_max_ctas : device_sm_count());
  launch_pdl(tc_conv_kernel<BN, STAGES, EPI, AFFINE, PS>, dim3(grid), dim3(TC_CONV_THREADS), (size_t)(S::TOTAL), s, tmA, tmB, p);
  LAUNCHED();
  return cudaPeekAtLastError() == cudaSuccess ? 0 : -3;
}
template <int BN, int STAGES>
static int launch_conv(const CUtensorMap& tmA, const CUtensorMap& tmB, const TcConvParams& p, cudaStream_t s, const char* name) {
  g_tc_last_kernel = name;
  switch (p.epi) {
    case EPI_STATS: return launch_conv_e<BN, STAGES, EPI_STATS, false>(tmA, tmB, p, s);
    case EPI_BNBWD: return launch_conv_e<BN, STAGES, EPI_BNBWD, false>(tmA, tmB, p, s);
    case EPI_ACTBWD: return launch_conv_e<BN, STAGES, EPI_ACTBWD, false>(tmA, tmB, p, s);
  }
  return (p.scale && p.bias) ? launch_conv_e<BN, STAGES, EPI_PLAIN, true>(tmA, tmB, p, s) : launch_conv_e<BN, STAGES, EPI_PLAIN, false>(tmA, tmB, p, s);
}
static int dispatch_conv(int BN, const CUtensorMap& tmA, const CUtensorMap& tmB, const TcConvParams& p, cudaStream_t s) {
  switch (BN) {
    case 64: return launch_conv<64, 4>(tmA, tmB, p, s, "tc_conv_kernel<64,4>");
    case 128: return launch_conv<128, 4>(tmA, tmB, p, s, "tc_conv_kernel<128,4>");
  }
  return -4;
}

// weights as a 3-D tensor [rows][taps][inner] (bf16, inner contiguous)
static int weight_map(CUtensorMap* m, const __nv_bfloat16* w, int rows, int taps, int inner, int box_rows) {
  cuuint64_t dims[3] = {(cuuint64_t)inner, (cuuint64_t)taps, (cuuint64_t)rows};
  cuuint64_t strides[2] = {(cuuint64_t)inner * 2, (cuuint64_t)taps * inner * 2};
  cuuint32_t box[3] = {64, 1, (cuuint32_t)box_rows}; cuuint32_t es[3] = {1, 1, 1};
  return make_map_bf16(m, w, 3, dims, strides, box, es);
}
static void fill_epi(TcConvParams& p, const float* bias, int act, float alpha, const TcEpi* e) {
  p.bias = bias; p.act = act; p.alpha = alpha; p.epi = EPI_PLAIN;
  if (!e) return;
  p.scale = e->scale; p.epi = e->mode; p.acc = e->acc; p.imgs_per_group = e->mode == EPI_STATS || e->mode == EPI_BNBWD ? e->imgs_per_group : 0;
  p.aux = e->aux; p.aux2 = e->aux2;
  if (e->mode == EPI_BNBWD || e->mode == EPI_ACTBWD) { p.act = e->act; p.alpha = e->alpha; p.bias = nullptr; p.scale = nullptr; }
}

// w_mn = 0: w is [O][taps][C] (reduction contiguous).  w_mn = 1 (1x1 geometry only): w is [C][O] -- the dense layer's own [nOut][nIn] weight
// read as the operand of its input-gradient GEMM (reduction over nOut), no transposed copy.
int k_tc_fprop(const ConvGeom& g, const __nv_bfloat16* x, const __nv_bfloat16* w, const float* bias, __nv_bfloat16* out, int act, float alpha, cudaStream_t s, const TcEpi* epi, int w_mn) {
  TcConvParams p{}; p.mode = 0;
  if (!pick_row_tile(g.N, g.OH, g.OW, 128, &p.Nt, &p.Ht, &p.Wt) || !tc_epi_ok(epi, p.Nt)) return -1;
  if (w_mn && (g.KH != 1 || g.KW != 1)) return -1;
  const int BN = pick_bn_fill(g.O, (long)g.N * g.OH * g.OW / 128);
  p.GH = g.OH; p.GW = g.OW; p.tiles_y = g.OH / p.Ht; p.taps_h = g.KH; p.taps_w = g.KW; p.chunks = g.C / 64; p.KW = g.KW;
  p.SH = g.SH; p.SW = g.SW; p.PH = g.PH; p.PW = g.PW; p.OC = g.O; p.outH = g.OH; p.outW = g.OW; p.out = out; p.b_mn = w_mn;
  fill_epi(p, bias, act, alpha, epi);
  CUtensorMap tmA, tmB;
  cuuint64_t dims[4] = {(cuuint64_t)g.C, (cuuint64_t)g.W, (cuuint64_t)g.H, (cuuint64_t)g.N};
  cuuint64_t strides[3] = {(cuuint64_t)g.C * 2, (cuuint64_t)g.W * g.C * 2, (cuuint64_t)g.H * g.W * g.C * 2};
  cuuint32_t box[4] = {64, (cuuint32_t)(p.Wt * g.SW), (cuuint32_t)(p.Ht * g.SH), (cuuint32_t)p.Nt};
  cuuint32_t es[4] = {1, (cuuint32_t)g.SW, (cuuint32_t)g.SH, 1};
  if (make_map_bf16(&tmA, x, 4, dims, strides, box, es)) return -1;
  p.tiles_m = g.N * g.OH * g.OW / 128; p.tiles_n = g.O / BN; p.phases = 1;
  if (w_mn ? weight_map(&tmB, w, g.C, 1, g.O, 64) : weight_map(&tmB, w, g.O, g.KH * g.KW, g.C, BN)) return -1;
  return dispatch_conv(BN, tmA, tmB, p, s);
}

// conv input gradient = transposed-conv forward, 4x4 s2 p1, in sub-pixel phase form.  w is the STRAIGHT copy [O][16][C]: the reduction runs
// over O, so the weight tile is MN-major ({64 c, 1 tap, 64 o} boxes).
int k_tc_dgrad(const ConvGeom& g, const __nv_bfloat16* dy, const __nv_bfloat16* w, const float* bias, __nv_bfloat16* dx, int act, float alpha, cudaStream_t s, const TcEpi* epi) {
  TcConvParams p{}; p.mode = 1;
  if (!pick_row_tile(g.N, g.OH, g.OW, 128, &p.Nt, &p.Ht, &p.Wt) || !tc_epi_ok(epi, p.Nt)) return -1;
  const int BN = pick_bn_fill(g.C, (long)g.N * g.OH * g.OW / 128 * 4);
  p.GH = g.OH; p.GW = g.OW; p.tiles_y = g.OH / p.Ht; p.taps_h = 2; p.taps_w = 2; p.chunks = g.O / 64; p.KW = 4;
  p.SH = 1; p.SW = 1; p.PH = 0; p.PW = 0; p.OC = g.C; p.outH = g.H; p.outW = g.W; p.out = dx; p.b_mn = 1;
  fill_epi(p, bias, act, alpha, epi);
  CUtensorMap tmA, tmB;
  cuuint64_t dims[4] = {(cuuint64_t)g.O, (cuuint64_t)g.OW, (cuuint64_t)g.OH, (cuuint64_t)g.N};
  cuuint64_t strides[3] = {(cuuint64_t)g.O * 2, (cuuint64_t)g.OW * g.O * 2, (cuuint64_t)g.OH * g.OW * g.O * 2};
  cuuint32_t box[4] = {64, (cuuint32_t)p.Wt, (cuuint32_t)p.Ht, (cuuint32_t)p.Nt};
  cuuint32_t es[4] = {1, 1, 1, 1};
  if (weight_map(&tmB, w, g.O, 16, g.C, 64)) return -1;
  if (make_map_bf16(&tmA, dy, 4, dims, strides, box, es)) return -1;
  p.tiles_m = g.N * g.OH * g.OW / 128; p.tiles_n = g.C / BN; p.phases = 4;
  return dispatch_conv(BN, tmA, tmB, p, s);
}

// ------------------------------------------------------------------ transposed conv onto <= 4 channels ------
static bool is_k4s2p1_geom(const ConvGeom& g) { return g.KH == 4 && g.KW == 4 && g.SH == 2 && g.SW == 2 && g.PH == 1 && g.PW == 1 && g.H == 2 * g.OH && g.W == 2 * g.OW; }
bool tc_deconv_ps_shape(const ConvGeom& g) { return is_k4s2p1_geom(g) && g.C >= 1 && g.C <= 4 && g.O % 64 == 0; }
bool tc_deconv_ps_supported(const ConvGeom& g) { int a, b, c; return tc_deconv_ps_shape(g) && pick_row_tile(g.N, g.OH, g.OW, 128, &a, &b, &c); }
size_t k_tc_deconv_ps_weight_elems(const ConvGeom& g) { return tc_deconv_ps_shape(g) ? (size_t)16 * 9 * g.O : 0; }
// w [O][4][4][C] fp32 master -> wps [(py,px,c4)][(dyr,dxc)][O] bf16; dy row offset dyr serves (py, filter row r): -1 -> (0,3); 0 -> (0,1),(1,2); +1 -> (1,0)
__global__ void pack_deconv_ps_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ wps, int O, int C) { pdl_wait();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x; if (idx >= 16 * 9 * O) return;
  const int o = idx % O, t = (idx / O) % 9, n = idx / (9 * O);
  const int py = n >> 3, px = (n >> 2) & 1, c = n & 3, dyr = t / 3 - 1, dxc = t % 3 - 1;
  const int r = dyr == -1 ? (py == 0 ? 3 : -1) : dyr == 0 ? (py == 0 ? 1 : 2) : (py == 1 ? 0 : -1);
  const int sx = dxc == -1 ? (px == 0 ? 3 : -1) : dxc == 0 ? (px == 0 ? 1 : 2) : (px == 1 ? 0 : -1);
  wps[idx] = __float2bfloat16((r >= 0 && sx >= 0 && c < C) ? w[((size_t)o * 16 + r * 4 + sx) * C + c] : 0.f);
}
void k_pack_deconv_ps(const float* w, __nv_bfloat16* wps, int O, int C, cudaStream_t s) {
  launch_pdl(pack_deconv_ps_kernel, dim3((16 * 9 * O + 255) / 256), dim3(256), (size_t)(0), s, w, wps, O, C); LAUNCHED();
}
int k_tc_deconv_ps(const ConvGeom& g, const __nv_bfloat16* dy, const __nv_bfloat16* wps, const float* bias, __nv_bfloat16* dx, int act, float alpha, cudaStream_t s, const TcEpi* epi) {
  TcConvParams p{}; p.mode = 0;
  if (!tc_deconv_ps_shape(g) || !pick_row_tile(g.N, g.OH, g.OW, 128, &p.Nt, &p.Ht, &p.Wt)) return -1;
  if (epi && epi->mode != EPI_PLAIN && epi->mode != EPI_ACTBWD) return -1;
  p.GH = g.OH; p.GW = g.OW; p.tiles_y = g.OH / p.Ht; p.taps_h = 3; p.taps_w = 3; p.chunks = g.O / 64; p.KW = 3;
  p.SH = 1; p.SW = 1; p.PH = 1; p.PW = 1; p.OC = g.C; p.outH = g.H; p.outW = g.W; p.out = dx;
  fill_epi(p, bias, act, alpha, epi);
  CUtensorMap tmA, tmB;
  cuuint64_t dims[4] = {(cuuint64_t)g.O, (cuuint64_t)g.OW, (cuuint64_t)g.OH, (cuuint64_t)g.N};
  cuuint64_t strides[3] = {(cuuint64_t)g.O * 2, (cuuint64_t)g.OW * g.O * 2, (cuuint64_t)g.OH * g.OW * g.O * 2};
  cuuint32_t box[4] = {64, (cuuint32_t)p.Wt, (cuuint32_t)p.Ht, (cuuint32_t)p.Nt}; cuuint32_t es[4] = {1, 1, 1, 1};
  if (make_map_bf16(&tmA, dy, 4, dims, strides, box, es)) return -1;
  if (weight_map(&tmB, wps, 16, 9, g.O, 16)) return -1;
  p.tiles_m = (int)((long)g.N * g.OH * g.OW / 128); p.tiles_n = 1; p.phases = 1;
  g_tc_last_kernel = "tc_conv_kernel<16,4,PS>";
  return p.epi == EPI_ACTBWD ? launch_conv_e<16, 4, EPI_ACTBWD, false, true>(tmA, tmB, p, s) : launch_conv_e<16, 4, EPI_PLAIN, false, true>(tmA, tmB, p, s);
}

// ------------------------------------------------------------------ conv 4x4 s2 p1 FROM <= 4 image channels ------
// D1 forward / G-last input gradient (fprop form) and their weight gradient.  K = 16 taps x C <= 64 is ONE 128-byte swizzle row per
// output pixel, but a 3-channel NHWC image cannot be gathered by TMA (6-byte pixels), so the im2col tile is built by the CTA itself:
// the (2*Ht+2) input rows a 128-pixel tile touches are one contiguous slab of the image; 128 threads copy it to shared memory with
// 16-byte loads, each thread then writes its pixel's 4 x (4*C) window as the 128B-swizzled K-major row wgmma expects
// (fence.proxy.async makes the generic-proxy writes visible to the tensor core), and the CTA -- one warpgroup -- issues the MMAs.
// Many short CTAs per SM (31 KB smem each) overlap each other's load / transform / MMA / store phases.
struct TcEdgeParams {
  const __nv_bfloat16* x; const __nv_bfloat16* w; const __nv_bfloat16* dy; const float* bias; __nv_bfloat16* out; float* part; float* part_b;
  int N, H, W, C, OH, OW, O, Ht, tiles_y, tiles_total, tiles_per_cta, act; float alpha;
};
static constexpr int EDGE_SLAB_BYTES = 6144;
__device__ __forceinline__ uint32_t swz128(int row, int byte) { return (uint32_t)(row * 128 + ((((byte >> 4) ^ (row & 7)) << 4) | (byte & 15))); }

// rows 2*oy0-1 .. 2*(oy0+Ht-1)+2 of image n (zero rows outside the image), <= 3 x 16 B per thread: fetched into registers one tile ahead so
// that the global-memory latency overlaps the previous tile's transform / MMA / epilogue, then parked in the slab
struct EdgeSlabRegs { uint4 v[3]; };
__device__ __forceinline__ void edge_fetch_slab(const TcEdgeParams& p, int n, int oy0, EdgeSlabRegs& r) {
  const int WC = p.W * p.C, cpr = WC >> 3, total = (2 * p.Ht + 2) * cpr;
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    const int i = threadIdx.x + q * 128; r.v[q] = make_uint4(0u, 0u, 0u, 0u);
    if (i < total) { const int j = i / cpr, cc = i - j * cpr, iy = 2 * oy0 - 1 + j;
      if (iy >= 0 && iy < p.H) r.v[q] = __ldg(reinterpret_cast<const uint4*>(p.x + ((size_t)n * p.H + iy) * WC) + cc); }
  }
}
__device__ __forceinline__ void edge_store_slab(const TcEdgeParams& p, const EdgeSlabRegs& r, uint8_t* slab) {
  const int total = (2 * p.Ht + 2) * ((p.W * p.C) >> 3);
#pragma unroll
  for (int q = 0; q < 3; ++q) { const int i = threadIdx.x + q * 128; if (i < total) reinterpret_cast<uint4*>(slab)[i] = r.v[q]; }
}
// thread = output pixel (oy_l, ox) of the tile: k = (r*4 + s)*C + c  <-  slab row 2*oy_l + r, elements (2*ox-1)*C + s*C + c, i.e. 4*C contiguous
// bf16 per filter row.  The window starts 2 bytes off a 32-bit boundary when C is odd: aligned 32-bit loads + a 16-bit funnel shift.  The
// whole 128-byte row (zero padded past k = 16*C) is assembled in registers and written as eight conflict-free 16-byte swizzled stores.
template <int C>
__device__ __forceinline__ void edge_build_row_c(const TcEdgeParams& p, const uint8_t* slab, uint8_t* tile, int row, bool ones) {
  const int WC = p.W * C, oy_l = row / p.OW, ox = row - oy_l * p.OW;
  const int lo = ox == 0 ? C : 0, hi = ox == p.OW - 1 ? 3 * C : 4 * C;       // window elements outside [lo, hi) fall left / right of the image
  uint32_t out[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) out[i] = 0u;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int b0 = ((2 * oy_l + r) * WC + (2 * ox - 1) * C) * 2;
    if (C & 1) {
      const uint32_t* wp = reinterpret_cast<const uint32_t*>(slab + b0 - 2);
      uint32_t w[2 * C + 1];
#pragma unroll
      for (int i = 0; i <= 2 * C; ++i) w[i] = wp[i];
#pragma unroll
      for (int i = 0; i < 2 * C; ++i) out[r * 2 * C + i] = __funnelshift_r(w[i], w[i + 1], 16);
    } else {
      const uint32_t* wp = reinterpret_cast<const uint32_t*>(slab + b0);
#pragma unroll
      for (int i = 0; i < 2 * C; ++i) out[r * 2 * C + i] = wp[i];
    }
#pragma unroll
    for (int i = 0; i < 2 * C; ++i) {
      const uint32_t m = ((2 * i >= lo && 2 * i < hi) ? 0xFFFFu : 0u) | ((2 * i + 1 >= lo && 2 * i + 1 < hi) ? 0xFFFF0000u : 0u);
      out[r * 2 * C + i] &= m;
    }
  }
  if (C < 4 && ones) out[8 * C] = 0x3F80u;       // column 16*C = 1.0 (bf16): the weight-gradient MMA then also yields sum_pix dy[pix][o] = the bias gradient
#pragma unroll
  for (int cc = 0; cc < 8; ++cc) *reinterpret_cast<uint4*>(tile + row * 128 + ((cc ^ (row & 7)) << 4)) = make_uint4(out[4 * cc], out[4 * cc + 1], out[4 * cc + 2], out[4 * cc + 3]);
}
__device__ __forceinline__ void edge_build_row(const TcEdgeParams& p, const uint8_t* slab, uint8_t* tile, int row, bool ones = false) {
  switch (p.C) { case 1: edge_build_row_c<1>(p, slab, tile, row, ones); break; case 2: edge_build_row_c<2>(p, slab, tile, row, ones); break;
                 case 3: edge_build_row_c<3>(p, slab, tile, row, ones); break; default: edge_build_row_c<4>(p, slab, tile, row, ones); break; }
}


__global__ void __launch_bounds__(128) tc_edge_conv_kernel(const TcEdgeParams p) { pdl_wait();
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* sm = smem_raw + (smem_base - smem_u32(smem_raw));
  uint8_t* sA = sm; uint8_t* sB = sm + 16384; uint8_t* slab = sm + 24576;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nb0 = blockIdx.y * 64, K = 16 * p.C;
  const int t_beg = blockIdx.x * p.tiles_per_cta, t_end = min(p.tiles_total, t_beg + p.tiles_per_cta);
  EdgeSlabRegs pre;
  if (t_beg < t_end) edge_fetch_slab(p, t_beg / p.tiles_y, (t_beg % p.tiles_y) * p.Ht, pre);
  {   // weight tile [64 o][64 k] K-major, once per CTA: row o = 16*C contiguous bf16 of the shadow = 2*C 16-byte chunks, zero padded to 8
    uint4 wv[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) { const int i = tid + q * 128, o = i >> 3, cc = i & 7;
      wv[q] = cc < 2 * p.C ? __ldg(reinterpret_cast<const uint4*>(p.w + (size_t)(nb0 + o) * K) + cc) : make_uint4(0u, 0u, 0u, 0u); }
#pragma unroll
    for (int q = 0; q < 4; ++q) { const int i = tid + q * 128, o = i >> 3, cc = i & 7; *reinterpret_cast<uint4*>(sB + o * 128 + ((cc ^ (o & 7)) << 4)) = wv[q]; }
  }
  const bool has_bias = p.bias != nullptr;
  const int r0 = warp * 16 + (lane >> 2), cq = lane & 3;       // accumulator fragment rows r0 (+8) of each 64-row half, columns 8j + 2cq
  for (int t = t_beg; t < t_end; ++t) {
    const int n = t / p.tiles_y, oy0 = (t % p.tiles_y) * p.Ht;
    edge_store_slab(p, pre, slab);
    __syncthreads();            // slab complete; the previous tile's output staging in sA has been copied out
    if (t + 1 < t_end) edge_fetch_slab(p, (t + 1) / p.tiles_y, ((t + 1) % p.tiles_y) * p.Ht, pre);
    edge_build_row(p, slab, sA, tid);
    fence_proxy_async_smem();
    __syncthreads();
    float acc[2][32];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < 32; ++j) acc[h][j] = 0.f;
    wg_fence();
    {
      const uint64_t bdesc = desc_kmajor_sw128(smem_base + 16384);
#pragma unroll
      for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int h = 0; h < 2; ++h) wgmma_n64<0, 0>(acc[h], desc_kmajor_sw128(smem_base + h * 8192) + 2 * k, bdesc + 2 * k);
    }
    wg_commit();
    wg_wait<0>();
    __syncthreads();            // every MMA has consumed sA: it becomes the bf16 output staging [128 pixels][64 channels], 16-byte chunks XOR-swizzled
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int row = h * 64 + r0 + 8 * i;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int col = j * 8 + 2 * cq;
          float a = acc[h][4 * j + 2 * i], b = acc[h][4 * j + 2 * i + 1];
          if (has_bias) { a += p.bias[nb0 + col]; b += p.bias[nb0 + col + 1]; }
          __nv_bfloat162 v = __floats2bfloat162_rn(act_fwd(p.act, a, p.alpha), act_fwd(p.act, b, p.alpha));
          *reinterpret_cast<__nv_bfloat162*>(sA + row * 128 + ((j ^ (row & 7)) << 4) + cq * 4) = v;
        }
      }
    __syncthreads();
    // the tile's 128 pixels are consecutive in NHWC: 16-byte pieces, eight lanes per 128-byte pixel row
    __nv_bfloat16* obase = p.out + ((size_t)n * p.OH + oy0) * p.OW * p.O + nb0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int idx = tid + i * 128, r = idx >> 3, cc = idx & 7;
      *reinterpret_cast<uint4*>(obase + (size_t)r * p.O + cc * 8) = *reinterpret_cast<const uint4*>(sA + r * 128 + ((cc ^ (r & 7)) << 4));
    }
  }
}

// weight gradient of the same layers: dw[o][k] = sum_pix dy[pix][o] * xcol[pix][k].  Both operands are MN-major tiles [128 pixel rows][128 B]:
// dy rows are copied as they are (64 channels = 128 B), xcol rows are built as above; one m64n64 MMA per 16 pixel rows.
// Each CTA walks tiles_per_cta consecutive tiles (split over pixels), accumulating in registers, and writes one fp32 partial.
__global__ void __launch_bounds__(128) tc_edge_wgrad_kernel(const TcEdgeParams p) { pdl_wait();
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* sm = smem_raw + (smem_base - smem_u32(smem_raw));
  uint8_t* sDy = sm; uint8_t* sX = sm + 16384; uint8_t* slab = sm + 32768;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, K = 16 * p.C;
  const int t_beg = blockIdx.x * p.tiles_per_cta, t_end = min(p.tiles_total, t_beg + p.tiles_per_cta);
  float acc[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) acc[j] = 0.f;
  EdgeSlabRegs pre; uint4 dyr[8];
  auto fetch = [&](int t) {
    const int n = t / p.tiles_y, oy0 = (t % p.tiles_y) * p.Ht;
    edge_fetch_slab(p, n, oy0, pre);
    const uint4* dyt = reinterpret_cast<const uint4*>(p.dy + (((size_t)n * p.OH + oy0) * p.OW) * 64);     // the tile's 128 pixels are contiguous: 16 KB
#pragma unroll
    for (int i = 0; i < 8; ++i) dyr[i] = __ldg(dyt + tid + i * 128);
  };
  if (t_beg < t_end) fetch(t_beg);
  for (int t = t_beg; t < t_end; ++t) {
    edge_store_slab(p, pre, slab);
#pragma unroll
    for (int i = 0; i < 8; ++i) { const int idx = tid + i * 128, r = idx >> 3, cc = idx & 7; *reinterpret_cast<uint4*>(sDy + r * 128 + ((cc ^ (r & 7)) << 4)) = dyr[i]; }
    __syncthreads();
    if (t + 1 < t_end) fetch(t + 1);      // next tile's global loads fly during this tile's transform + MMAs
    edge_build_row(p, slab, sX, tid, p.part_b != nullptr);
    fence_proxy_async_smem();
    __syncthreads();
    wg_fence();
#pragma unroll
    for (int k = 0; k < 8; ++k)       // 16 pixel rows per MMA
      wgmma_n64<1, 1>(acc, desc_mnmajor_sw128(smem_base + k * 2048, 8192), desc_mnmajor_sw128(smem_base + 16384 + k * 2048, 8192));
    wg_commit();
    wg_wait<0>();
    __syncthreads();                      // the MMAs have consumed both tiles: shared memory may be overwritten
  }
  // accumulator row = output channel o, column = k (column K: the ones column = sum_pix dy = the bias gradient); an empty split writes zeros
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int o = warp * 16 + (lane >> 2) + 8 * i;
    float* orow = p.part + ((size_t)blockIdx.x * 64 + o) * K;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = j * 8 + 2 * (lane & 3);
      if (col < K) *reinterpret_cast<float2*>(orow + col) = make_float2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
      else if (col == K && p.part_b) p.part_b[(size_t)blockIdx.x * 64 + o] = acc[4 * j + 2 * i];
    }
  }
}

static bool edge_tile(const ConvGeom& g, int* Ht) {
  if (!is_k4s2p1_geom(g) || g.C < 1 || g.C > 4 || g.OW > 128 || 128 % g.OW) return false;
  const int ht = 128 / g.OW;
  if (g.OH % ht || (g.W * g.C) % 8 || (2 * ht + 2) * g.W * g.C * 2 > EDGE_SLAB_BYTES) return false;
  *Ht = ht; return true;
}
bool tc_edge_conv_supported(const ConvGeom& g) { int ht; return edge_tile(g, &ht) && g.O % 64 == 0; }
bool tc_edge_wgrad_supported(const ConvGeom& g) { int ht; return edge_tile(g, &ht) && g.O == 64; }
// CTA targets of the edge kernels: two waves for the weight gradient (split-K partials, fixed-order sum), eight for the forward
static int tc_edge_wgrad_target() {
  static int env = -1; if (env < 0) { const char* e = getenv("B2G_EDGE_WGRAD_CTAS"); env = e ? atoi(e) : 0; }
  const int cap = 8 * device_sm_count(); return env >= 1 && env <= cap ? env : 2 * device_sm_count();
}
static int tc_edge_wgrad_ctas(const ConvGeom& g, int* tpc) {
  int ht = 1; edge_tile(g, &ht);
  const int tiles = g.N * (g.OH / ht), target = tc_edge_wgrad_target();
  const int per = (tiles + target - 1) / target; *tpc = per < 1 ? 1 : per;
  return (tiles + *tpc - 1) / *tpc;
}
size_t k_tc_edge_wgrad_scratch_floats(const ConvGeom& g) { return tc_edge_wgrad_supported(g) ? (size_t)tc_edge_wgrad_target() * (64 * 16 * g.C + 64) : 0; }
int k_tc_edge_conv(const ConvGeom& g, const __nv_bfloat16* x, const __nv_bfloat16* w, const float* bias, __nv_bfloat16* out, int act, float alpha, cudaStream_t s) {
  TcEdgeParams p{}; if (!edge_tile(g, &p.Ht) || g.O % 64) return -1;
  if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(w) & 15) || (reinterpret_cast<uintptr_t>(out) & 15)) return -1;
  p.x = x; p.w = w; p.bias = bias; p.out = out; p.N = g.N; p.H = g.H; p.W = g.W; p.C = g.C; p.OH = g.OH; p.OW = g.OW; p.O = g.O; p.tiles_y = g.OH / p.Ht;
  p.tiles_total = g.N * p.tiles_y; p.act = act; p.alpha = alpha;
  const size_t smem = 1024 + 24576 + EDGE_SLAB_BYTES;
  TC_SET_SMEM_ONCE(tc_edge_conv_kernel, smem);
  static int env = -1; if (env < 0) { const char* e = getenv("B2G_EDGE_CONV_CTAS"); env = e ? atoi(e) : 0; }
  const int target = env >= 1 ? env : 8 * device_sm_count();
  p.tiles_per_cta = (p.tiles_total + target - 1) / target;
  launch_pdl(tc_edge_conv_kernel, dim3(dim3((unsigned)((p.tiles_total + p.tiles_per_cta - 1) / p.tiles_per_cta), (unsigned)(g.O / 64))), dim3(128), (size_t)(smem), s, p);
  LAUNCHED(); g_tc_last_kernel = "tc_edge_conv_kernel";
  return cudaPeekAtLastError() == cudaSuccess ? 0 : -3;
}
static void reduce_or_defer(ReduceList* defer, const float* src, float* dst, size_t n, int splits, size_t stride, int accumulate, cudaStream_t s);
int k_tc_edge_wgrad(const ConvGeom& g, const __nv_bfloat16* x, const __nv_bfloat16* dy, float* dw, float* db, float* scratch, size_t scratch_floats, int accumulate, cudaStream_t s, ReduceList* defer) {
  TcEdgeParams p{}; if (!edge_tile(g, &p.Ht) || g.O != 64) return -1;
  if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(dy) & 15)) return -1;
  p.x = x; p.dy = dy; p.part = scratch; p.N = g.N; p.H = g.H; p.W = g.W; p.C = g.C; p.OH = g.OH; p.OW = g.OW; p.O = g.O; p.tiles_y = g.OH / p.Ht;
  p.tiles_total = g.N * p.tiles_y;
  const int ctas = tc_edge_wgrad_ctas(g, &p.tiles_per_cta); const size_t n = (size_t)64 * 16 * g.C;
  if ((size_t)ctas * (n + 64) > scratch_floats) return -5;
  if (db && g.C < 4) p.part_b = scratch + (size_t)ctas * n;
  const size_t smem = 1024 + 32768 + EDGE_SLAB_BYTES;
  TC_SET_SMEM_ONCE(tc_edge_wgrad_kernel, smem);
  launch_pdl(tc_edge_wgrad_kernel, dim3(dim3((unsigned)ctas)), dim3(128), (size_t)(smem), s, p);
  LAUNCHED(); g_tc_last_kernel = "tc_edge_wgrad_kernel";
  if (cudaPeekAtLastError() != cudaSuccess) return -3;
  reduce_or_defer(defer, scratch, dw, n, ctas, n, accumulate, s);
  if (p.part_b) reduce_or_defer(defer, p.part_b, db, 64, ctas, 64, accumulate, s);
  return p.part_b ? 1 : 0;      // 1: the bias gradient (column sums of dy) was produced as well
}

// ------------------------------------------------------------------ wgrad: MN-major operands --------------
// dW[o][tap][c] = sum over pixels of dy[pix][o] * x[pix shifted by tap][c].  The reduction index (pixels) is the
// slow dimension of both NHWC operands, so both are fed to wgmma as MN-major tiles: a TMA box of
// {64 channels, 64 pixels} lands as [pixel rows][128 B], which IS the canonical 128B-swizzled MN-major layout
// (8-pixel groups 1024 B apart = SBO, 64-channel blocks one box apart = LBO).  No transposes anywhere.
// CTA tile: 128 output channels (o, 64 per consumer warpgroup) x BNW columns of the flattened (tap, c) axis -- i.e. BNW/64
// sixty-four-channel blocks that may belong to different filter taps, so one dy tile in smem feeds several taps (halves the L2
// traffic of dy) -- over a split of the pixel range; fp32 partials go to scratch[split] and are summed in fixed order (deterministic).
struct TcWgradParams {
  int Nt, Ht, Wt;          // K-block = 64 pixels of the dy grid = Nt images x Ht rows x Wt cols
  int tiles_y;             // OH / Ht
  int KW, SH, SW, PH, PW;
  int taps, C;             // row length of dw = taps*C
  int kb_total, kb_per_split;
  float* out; size_t split_stride;
};

template <int BNW, int STAGES>
struct TcWgradSmem {
  static constexpr int A_BYTES = 2 * 64 * 128;            // two 64-channel blocks of dy
  static constexpr int B_BYTES = (BNW / 64) * 64 * 128;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int BAR_OFF = STAGES * STAGE_BYTES;
  static constexpr int TOTAL = BAR_OFF + 256 + 1024;
};

template <int BNW, int STAGES>
__global__ void __launch_bounds__(TC_THREADS, 1) tc_wgrad_kernel(const __grid_constant__ CUtensorMap tmDy, const __grid_constant__ CUtensorMap tmX, const TcWgradParams p) {
  using S = TcWgradSmem<BNW, STAGES>;
  constexpr int NB = BNW / 64;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_full = smem_base + S::BAR_OFF, bar_empty = bar_full + 8 * STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int split = blockIdx.x, col0 = blockIdx.y * BNW, o0 = blockIdx.z * 128;     // col = tap*C + c
  const int kb_beg = split * p.kb_per_split, kb_end = min(p.kb_total, kb_beg + p.kb_per_split);
  const int num_kb = max(0, kb_end - kb_beg);

  if (threadIdx.x == 0) {
    prefetch_map(&tmDy); prefetch_map(&tmX);
    for (int s = 0; s < STAGES; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, 8); }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_trigger();      // single-wave grid: the successor may be scheduled behind us right away
  pdl_wait();         // barrier init above overlaps the predecessor's tail; global memory is touched only below

  if (warp == 0) {
    // producer (converged warp, elected lane issues).  The (tap, channel) origin of each 64-column block is fixed for the CTA; ring slot and
    // pixel-block origin advance as counters (an integer division per step is time the loads wait for)
    int xc[NB], xw[NB], xh[NB];
#pragma unroll
    for (int j = 0; j < NB; ++j) { const int col = col0 + j * 64, tap = col / p.C; xc[j] = col % p.C; xw[j] = -p.PW + tap % p.KW; xh[j] = -p.PH + tap / p.KW; }
    int n0, y0;
    if (p.Nt > 1) { n0 = kb_beg * p.Nt; y0 = 0; } else { n0 = kb_beg / p.tiles_y; y0 = (kb_beg % p.tiles_y) * p.Ht; }
    int s = 0; uint32_t ph = 0;
    for (int i = 0; i < num_kb; ++i) {
      const int kb = kb_beg + i;
      mbar_wait(bar_empty + 8 * s, ph ^ 1);
      if (elect_one_sync()) {
        mbar_expect_tx(bar_full + 8 * s, S::STAGE_BYTES);
        const uint32_t a = smem_base + s * S::STAGE_BYTES, b = a + S::A_BYTES;
        tma_load_2d(a, &tmDy, bar_full + 8 * s, o0, kb * 64);
        tma_load_2d(a + 8192, &tmDy, bar_full + 8 * s, o0 + 64, kb * 64);
#pragma unroll
        for (int j = 0; j < NB; ++j) tma_load_4d(b + j * 8192, &tmX, bar_full + 8 * s, xc[j], xw[j], y0 * p.SH + xh[j], n0);
      }
      __syncwarp();
      if (++s == STAGES) { s = 0; ph ^= 1; }
      if (p.Nt > 1) n0 += p.Nt; else { y0 += p.Ht; if (y0 >= p.tiles_y * p.Ht) { y0 = 0; ++n0; } }
    }
  } else if (warp >= 4) {
    // consumers: warpgroup wg owns output channels [o0 + 64 wg, o0 + 64 wg + 64)
    const int wg = (warp >> 2) - 1;
    float acc[NB][32];
#pragma unroll
    for (int nb = 0; nb < NB; ++nb)
#pragma unroll
      for (int j = 0; j < 32; ++j) acc[nb][j] = 0.f;
    int s = 0, prev = -1; uint32_t ph = 0;
    for (int i = 0; i < num_kb; ++i) {
      mbar_wait(bar_full + 8 * s, ph);
      wg_fence();
      const uint32_t a = smem_base + s * S::STAGE_BYTES + wg * 8192, b = smem_base + s * S::STAGE_BYTES + S::A_BYTES;
#pragma unroll
      for (int k = 0; k < 4; ++k)     // 16 pixel rows per MMA = 2048 B down both tiles
#pragma unroll
        for (int nb = 0; nb < NB; ++nb) wgmma_n64<1, 1>(acc[nb], desc_mnmajor_sw128(a + k * 2048, 8192), desc_mnmajor_sw128(b + nb * 8192 + k * 2048, 8192));
      wg_commit();
      wg_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(bar_empty + 8 * prev);
      prev = s;
      if (++s == STAGES) { s = 0; ph ^= 1; }
    }
    wg_wait<0>();
    // fragment rows o, columns 8j + 2(l%4): each group of four lanes writes one full 32-byte sector of a partial row (zeros for an empty split)
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int o = o0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i;
      float* orow = p.out + (size_t)split * p.split_stride + (size_t)o * p.taps * p.C + col0;
#pragma unroll
      for (int nb = 0; nb < NB; ++nb)
#pragma unroll
        for (int j = 0; j < 8; ++j)
          *reinterpret_cast<float2*>(orow + nb * 64 + j * 8 + 2 * (lane & 3)) = make_float2(acc[nb][4 * j + 2 * i], acc[nb][4 * j + 2 * i + 1]);
    }
  }
}

// two consumer warpgroups x 64 channels x at most 128 fp32 accumulator columns (64 registers per thread)
static int wgrad_bnw(const ConvGeom& g) { if (g.C % 64) return 0; const long cols = (long)g.KH * g.KW * g.C; return cols % 128 == 0 ? 128 : 64; }
// CTA target of the split-K weight gradients: two thirds of a wave.  The weight-gradient kernels run on the side stream beside the
// input-gradient chain, which keeps the remaining SMs; fewer CTAs also cut the fp32 partials the deferred reduce reads.
static int wgrad_target() {
  static int env = -1; if (env < 0) { const char* e = getenv("B2G_WGRAD_CTAS"); env = e ? atoi(e) : 0; }
  return env >= 1 ? env : (2 * device_sm_count()) / 3;
}
// choose the split count so that the whole grid is at most wgrad_target() CTAs
static int wgrad_splits_for(const ConvGeom& g, int o_tile) {
  const int bnw = wgrad_bnw(g); if (!bnw) return 1;
  long tiles = (long)(g.O / o_tile) * (g.KH * g.KW * g.C / bnw), kbt = (long)g.N * g.OH * g.OW / 64;
  long sp = wgrad_target() / tiles, cap = kbt / 8; if (cap < 1) cap = 1; if (sp > cap) sp = cap; if (sp < 1) sp = 1; return (int)sp;
}
static int tc_wgrad_splits(const ConvGeom& g) { return wgrad_splits_for(g, 128); }
bool tc_wgrad_supported(const ConvGeom& g) {
  int a, b, c;
  return g.O % 128 == 0 && wgrad_bnw(g) != 0 && g.SH >= 1 && g.SH <= 2 && g.SW == g.SH && ((long)g.N * g.OH * g.OW) % 64 == 0 &&
         pick_row_tile(g.N, g.OH, g.OW, 64, &a, &b, &c) && c * g.SW <= 256 && b * g.SH <= 256;
}
size_t k_tc_wgrad_scratch_floats(const ConvGeom& g) {
  if (!tc_wgrad_supported(g)) return 0;
  return (size_t)wgrad_splits_for(g, 128) * g.O * g.KH * g.KW * g.C;
}

template <int BNW, int STAGES>
static int launch_wgrad(const CUtensorMap& tmDy, const CUtensorMap& tmX, const TcWgradParams& p, dim3 grid, cudaStream_t s, const char* name) {
  using S = TcWgradSmem<BNW, STAGES>;
  TC_SET_SMEM_ONCE((tc_wgrad_kernel<BNW, STAGES>), S::TOTAL);
  launch_pdl(tc_wgrad_kernel<BNW, STAGES>, dim3(grid), dim3(TC_THREADS), (size_t)(S::TOTAL), s, tmDy, tmX, p);
  LAUNCHED(); g_tc_last_kernel = name;
  return cudaPeekAtLastError() == cudaSuccess ? 0 : -3;
}

// the split-K partials land in `scratch`; their fixed-order sum into dw is either launched here or, with `defer`, queued for the caller's
// one k_reduce_multi launch at the end of the backward pass (scratch must then stay untouched until that launch)
static void reduce_or_defer(ReduceList* defer, const float* src, float* dst, size_t n, int splits, size_t stride, int accumulate, cudaStream_t s) {
  if (defer && !accumulate && defer->count < ReduceList::MAX_JOBS) { reduce_list_push(defer, src, dst, (int64_t)n, splits, (int64_t)stride); return; }
  k_reduce_splits(src, dst, n, splits, stride, accumulate, s);
}

int k_tc_wgrad(const ConvGeom& g, const __nv_bfloat16* x, const __nv_bfloat16* dy, float* dw, float* scratch, size_t scratch_floats, int accumulate, cudaStream_t s, ReduceList* defer) {
  TcWgradParams p{};
  if (!pick_row_tile(g.N, g.OH, g.OW, 64, &p.Nt, &p.Ht, &p.Wt)) return -1;
  const int BNW = wgrad_bnw(g); const size_t n = (size_t)g.O * g.KH * g.KW * g.C;
  int splits = tc_wgrad_splits(g);
  if ((size_t)splits * n > scratch_floats) return -5;
  p.tiles_y = g.OH / p.Ht; p.KW = g.KW; p.SH = g.SH; p.SW = g.SW; p.PH = g.PH; p.PW = g.PW; p.taps = g.KH * g.KW; p.C = g.C;
  p.kb_total = (int)((long)g.N * g.OH * g.OW / 64); p.kb_per_split = (p.kb_total + splits - 1) / splits;
  p.out = scratch; p.split_stride = n;
  CUtensorMap tmDy, tmX;
  { cuuint64_t dims[2] = {(cuuint64_t)g.O, (cuuint64_t)g.N * g.OH * g.OW}; cuuint64_t strides[1] = {(cuuint64_t)g.O * 2};
    cuuint32_t box[2] = {64, 64}; cuuint32_t es[2] = {1, 1};
    if (make_map_bf16(&tmDy, dy, 2, dims, strides, box, es)) return -1; }
  { cuuint64_t dims[4] = {(cuuint64_t)g.C, (cuuint64_t)g.W, (cuuint64_t)g.H, (cuuint64_t)g.N};
    cuuint64_t strides[3] = {(cuuint64_t)g.C * 2, (cuuint64_t)g.W * g.C * 2, (cuuint64_t)g.H * g.W * g.C * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)(p.Wt * g.SW), (cuuint32_t)(p.Ht * g.SH), (cuuint32_t)p.Nt}; cuuint32_t es[4] = {1, (cuuint32_t)g.SW, (cuuint32_t)g.SH, 1};
    if (make_map_bf16(&tmX, x, 4, dims, strides, box, es)) return -1; }
  dim3 grid((unsigned)splits, (unsigned)(p.taps * g.C / BNW), (unsigned)(g.O / 128));
  const int rc = BNW == 64 ? launch_wgrad<64, 4>(tmDy, tmX, p, grid, s, "tc_wgrad_kernel<64,4>") : launch_wgrad<128, 4>(tmDy, tmX, p, grid, s, "tc_wgrad_kernel<128,4>");
  if (rc) return rc;
  reduce_or_defer(defer, scratch, dw, n, splits, n, accumulate, s);
  return 0;
}

}  // namespace b2g
