// kernels.h -- launch wrappers of every CUDA kernel in libb200gan.so (sm_90a only).
// Host-callable, stream-ordered, no allocation.  "prec" selects the activation storage type
// (PREC_F32 = DL4J-parity mode, PREC_BF16 = tensor-core mode); statistics, parameters, gradients and
// updater state are always fp32.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

namespace b2g {

enum Prec { PREC_F32 = 0, PREC_BF16 = 1 };
enum Act { ACT_IDENTITY = 0, ACT_TANH = 1, ACT_SIGMOID = 2, ACT_RELU = 3, ACT_LRELU = 4 };

inline size_t prec_size(int prec) { return prec == PREC_F32 ? 4 : 2; }

// Convolution geometry, NHWC.  A dense layer is the 1x1 conv on a 1x1 image; a deconvolution is the
// transposed problem (its forward is this geometry's dgrad, its input-gradient this geometry's fprop).
struct ConvGeom {
  int N, H, W, C;        // conv input
  int OH, OW, O;         // conv output
  int KH, KW, SH, SW, PH, PW;
};

extern uint64_t g_launch_count;   // every kernel launch of this library bumps it (bench evidence)
// multiprocessor count of the current device (queried once per device): the one source every grid-sizing rule of the library uses
int device_sm_count();

// ---- layout ------------------------------------------------------------------------------------
void k_nchw_f32_to_nhwc(int prec, const float* src, void* dst, int N, int C, int HW, cudaStream_t s);
void k_nhwc_to_nchw_f32(int prec, const void* src, float* dst, int N, int C, int HW, cudaStream_t s);
void k_permute(int prec, const void* src, void* dst, int N, int C, int HW, int to_nhwc, cudaStream_t s);
void k_cast_f32_to_bf16(const float* src, __nv_bfloat16* dst, size_t n, cudaStream_t s);

// ---- batch norm --------------------------------------------------------------------------------
// Train-mode statistics per (group, channel): mean, invstd = 1/sqrt(var_biased+eps); optional DL4J running-stat
// pseudo-gradients g_mean += w*(1-decay)*(run_mean-mean) (w = 1/groups so groups average).
void k_bn_stats(int prec, const void* x, int rows_per_group, int C, int groups, float* scratch,
                float* mean, float* invstd, float eps,
                const float* run_mean, const float* run_var, float* g_mean, float* g_var, float decay, cudaStream_t s);
size_t k_bn_scratch_floats(int C, int groups);
// inference mode: mean <- run_mean, invstd <- rsqrt(run_var+eps) for every group
// scale[c] = gamma*rsqrt(var+eps), shift[c] = beta - mean*scale (+ conv_bias*scale): inference-mode BN as a GEMM epilogue
void k_bn_fold(const float* run_mean, const float* run_var, const float* gamma, const float* beta, const float* conv_bias, int C, float eps, float* scale, float* shift, cudaStream_t s);
void k_bn_prep_infer(const float* run_mean, const float* run_var, int C, int groups, float eps, float* mean, float* invstd, cudaStream_t s);
// y = act(gamma*(x-mean)*invstd+beta)
void k_bn_apply(int prec, const void* x, void* y, int rows_per_group, int C, int groups, const float* mean, const float* invstd,
                const float* gamma, const float* beta, int act, float alpha, cudaStream_t s);
// backward of y=act(bn(x)): reduce then apply.  dgamma/dbeta are ACCUMULATED over groups into g_gamma/g_beta (+=).
void k_bn_bwd(int prec, const void* x, const void* eps_out, void* eps_in, int rows_per_group, int C, int groups,
              const float* mean, const float* invstd, const float* gamma, const float* beta, int act, float alpha,
              float* scratch, float* g_gamma, float* g_beta, int want_param_grads, cudaStream_t s);

// Fused path (bf16, C % 8 == 0): the batch statistics live in 128-bit fixed-point accumulators acc[groups][2][2][C] (statistic, hi | lo,
// channel; common.cuh sacc_add) that the producing tensor-core GEMM fills from its epilogue (kernels_tc.cu EPI_STATS / EPI_BNBWD) or, where the
// producer has no such epilogue, the *_stats_acc kernels below; the apply kernels derive mean / invstd (and the backward coefficients) from
// them on the fly -- no partial buffers, no finalise launches.  The caller zeroes acc (one memset per pass).
bool k_bn_vec_ok(int prec, int C);
size_t k_bn_acc_elems(int C, int groups);                  // 64-bit words per accumulator set
void k_bn_stats_acc(const void* x, int rows_per_group, int C, int groups, unsigned long long* acc, cudaStream_t s);
// y = act(x*scale+shift) with shift = beta - mean*scale; block 0 also leaves coef[groups][4][C] = {scale = gamma*invstd, beta, mean, invstd} for the
// backward pass and (g_mean != null) the DL4J running-stat pseudo-gradients averaged over groups
void k_bn_apply_acc(const void* x, void* y, int rows_per_group, int C, int groups, const unsigned long long* acc, const float* gamma, const float* beta,
                    int act, float alpha, float eps, float* coef, const float* run_mean, const float* run_var, float* g_mean, float* g_var, float decay, cudaStream_t s, int replicas = 1);
// sum dy', sum dy'*xhat -> acc with dy' = eps_out * act'(z), z from kernels_ew.cu bn_pre_act: (x - mean)*scale + beta for tanh / sigmoid,
// the forward's x*scale+shift for relu / leaky relu   (producers without the EPI_BNBWD epilogue)
void k_bn_bwd_stats_acc(const void* x, const void* eps_out, int rows_per_group, int C, int groups, const float* coef, int act, float alpha, unsigned long long* acc, cudaStream_t s);
// eps_in = scale * (dy' - mean(dy') - xhat*mean(dy'*xhat)).  premul = 0: eps_out is the raw epsilon and acc = (sum dy', sum dy'*xhat) from
// k_bn_bwd_stats_acc; premul = 1: eps_out already holds dy' and acc = (sum dy', sum dy'*z) from the EPI_BNBWD epilogue, converted here in
// double: sum dy'*xhat = invstd * (sum dy'*z - mean * sum dy').  Block 0 adds dgamma / dbeta (summed over groups).
void k_bn_bwd_apply_acc(const void* x, const void* eps_out, void* eps_in, int rows_per_group, int C, int groups, const float* coef, int act, float alpha, int premul,
                        const unsigned long long* acc, float* g_gamma, float* g_beta, int want_param_grads, cudaStream_t s, int replicas = 1);
// replicas > 1 (sync_bn): acc holds the all-reduced sums of `replicas` ranks, each contributing rows_per_group rows per group

// ---- activations / pooling / upsampling -----------------------------------------------------------
void k_act_fwd(int prec, const void* x, void* y, size_t n, int act, float alpha, cudaStream_t s);
// eps_in = eps_out * f'(.) evaluated from the layer OUTPUT a (tanh: 1-a^2, sigmoid: a(1-a), relu/lrelu: sign of a)
void k_act_bwd_from_output(int prec, const void* a, const void* eps_out, void* eps_in, size_t n, int act, float alpha, cudaStream_t s);
void k_maxpool_fwd(int prec, const void* x, void* y, uint8_t* argmax, int N, int H, int W, int C, int OH, int OW, int KH, int KW, int SH, int SW, cudaStream_t s);
void k_maxpool_bwd(int prec, const void* eps_out, const uint8_t* argmax, void* eps_in, int N, int H, int W, int C, int OH, int OW, int KH, int KW, int SH, int SW, cudaStream_t s);
void k_upsample_fwd(int prec, const void* x, void* y, int N, int H, int W, int C, int f, cudaStream_t s);
void k_upsample_bwd(int prec, const void* eps_out, void* eps_in, int N, int H, int W, int C, int f, cudaStream_t s);

// ---- dropout (DL4J DropoutLayer, inverted dropout; mask definition in include/b200gan.h) ----------------------------------------
// Forward over the n elements of one pass (NHWC, element index e): y = x * (1/p) where kept, 0 where dropped, and the keep bits into
// mask[e >> 5] bit (e & 31).  The random word of element e is Philox4x32-10(ctr = {e >> 2, lo32(P), hi32(P), tag}, key = {lo32(seed), hi32(seed)})[e & 3],
// P = *pass read on the device.  bump_pass: the last block to finish advances *pass by one (ticket counter *ticket, reset by that block).
// tag = layer | rank << 16; keep where the word < threshold = floor(p * 2^32), or everywhere when keep_all (p >= 1); scale = 1.0f / p
struct DropoutArgs { uint64_t seed; uint32_t tag; uint32_t threshold; float scale; int keep_all; };
void k_dropout_fwd(int prec, const void* x, void* y, uint32_t* mask, size_t n, const DropoutArgs& a, unsigned long long* pass, unsigned* ticket, int bump_pass, cudaStream_t s);
// Backward: eps_in = eps_out * (1/p) where the forward kept the element, 0 elsewhere (eps_in may equal eps_out)
void k_dropout_bwd(int prec, const void* eps_out, void* eps_in, const uint32_t* mask, size_t n, float scale, cudaStream_t s);

// ---- loss ----------------------------------------------------------------------------------------------
// LossBinaryXENT on logits z[rows] with labels y[rows]: dz = dL/dz (sum form, not /mb), loss_sums[g] = sum of losses per group.
void k_xent(int prec, const void* z, const float* y, void* dz, float* loss_sums, int rows_per_group, int groups, float clip_eps, cudaStream_t s);
void k_sigmoid_out(int prec, const void* z, void* p, size_t n, cudaStream_t s);
// LossMCXENT + softmax over K classes: dz = softmax(z) - y, loss_sums[0] = -sum y log clip(p, 1e-10); p_out optional (probabilities)
void k_softmax_xent(int prec, const void* z, const float* y, void* dz, void* p_out, float* loss_sums, int rows, int K, cudaStream_t s);

// ---- reductions ------------------------------------------------------------------------------------
// out[c] (+)= sum_rows x[row][c]
void k_colsum(int prec, const void* x, int rows, int C, float* scratch, float* out, int accumulate, cudaStream_t s);
size_t k_colsum_scratch_floats(int C);
// out[0] = sum_i coef[i] * x[i]^2 over the listed segments (l2 score)
void k_sumsq_segments(const float* p, const int64_t* seg_off, const int64_t* seg_len, const float* seg_coef, int nseg, double* out, cudaStream_t s);
// dst[i] = sum_s src[s*stride + i]
void k_reduce_splits(const float* src, float* dst, size_t n, int splits, size_t stride, int accumulate, cudaStream_t s);
// the same for a whole list of (src, dst) pairs in ONE launch: the split-K partials of every weight gradient of a backward pass
struct ReduceJob { const float* src; float* dst; int64_t n, stride; int splits, blocks; };
struct ReduceList { static const int MAX_JOBS = 24; ReduceJob jobs[MAX_JOBS]; int count; };
void reduce_list_push(ReduceList* rl, const float* src, float* dst, int64_t n, int splits, int64_t stride);
void k_reduce_multi(const ReduceList& rl, cudaStream_t s);

// ---- updater (BaseMultiLayerUpdater + UpdaterBlock + params.subi, one pass) -----------------------------
struct UpdSeg {            // one parameter tensor
  int64_t off, len;
  int kind;                // 0 sgd, 1 rmsprop, 2 adam, 3 noop
  float lr, b1, b2, eps;   // rmsprop: b1 = rmsDecay
  float l2;                // post-updater, not lr-scaled (pre-beta4)
  float clip;              // elementwise clip threshold, 0 = off
  int div_mb;              // 0 for BN mean/var pseudo-gradients
  // bf16 shadow of a conv/deconv/dense weight: shadow[off_bf..] same layout [A][taps][B]; off_ps >= 0: also the packed [16][9][ps_O] operand of
  // the pixel-shuffle transposed conv (kernels_tc.cu k_pack_deconv_ps), every weight element has exactly one slot there
  int64_t off_bf, off_ps;
  int ps_O, ps_C;
};
// The last block to finish bumps *step_dev (Adam's t) and resets *ticket: no separate counter kernel.
// gn_mult (may be null): one fp32 multiplier per segment (k_gradnorm), applied to g right after the minibatch division.
void k_updater(float* params, const float* grads, float* st0, float* st1, const UpdSeg* segs_dev, const int32_t* chunk_seg_dev,
               const int64_t* chunk_off_dev, int nchunks, float inv_mb, float inv_world, int* step_dev /* t = *step_dev + 1 */, unsigned* ticket,
               __nv_bfloat16* shadow, const float* gn_mult, cudaStream_t s);
static const int UPD_CHUNK = 4096;

// ---- L2 gradient normalization (DL4J GradientNormalization.{Renormalize,Clip}L2Per{Layer,ParamType}; kernels_gradnorm.cu) ---------
// A norm group is a run of updater segments: one layer's segments, or one segment.  Its chunks are [chunk_begin, chunk_end) of the updater's
// chunk map, its segments [seg_begin, seg_end).
struct GnGroup { int32_t chunk_begin, chunk_end, seg_begin, seg_end; };
// One block per updater chunk: partial[c] = sum over the chunk of (double)(g * gscale)^2 (gscale = inv_mb, or inv_world for the BatchNorm
// running-stat pseudo-gradients, as in the updater).  The last block to finish (ticket counter *ticket, reset by that block) folds the
// partials of each group in chunk order, norm = sqrt(sum), and writes mult[s] for every segment s of the group, rounded to fp32 once:
//   clip = 0 (renormalize): 1 / norm, or 1 / 1e-5 when norm == 0;   clip = 1: threshold / norm when norm > threshold, else 1.
// The result does not depend on the order in which blocks run.
void k_gradnorm(const float* grads, const UpdSeg* segs_dev, const int32_t* chunk_seg_dev, const int64_t* chunk_off_dev, int nchunks,
                const GnGroup* groups_dev, int ngroups, int clip, float threshold, float inv_mb, float inv_world, double* partial, unsigned* ticket,
                float* mult, cudaStream_t s);
void k_fill_f32(float* p, float v, size_t n, cudaStream_t s);
void k_scale_f32(float* p, float v, size_t n, cudaStream_t s);
// Gradient all-reduce over NVLink peer memory (one process per GPU, buffers exchanged as CUDA IPC handles): ONE kernel per GPU does
// entry barrier -> reduce-scatter (this GPU sums its 1/world slice from every peer, fixed rank order) -> all-gather (writes the sum into
// every peer's buffer) -> exit barrier.  grads[r] / flags[r] are rank r's buffers as mapped into this process (r == rank: the local ones);
// flags = 16 words per GPU (entry[8] | exit[8], indexed by the signalling rank), state = {epoch, finished-block counter} (local).
struct P2pArgs { float* grads[8]; unsigned* flags[8]; int rank, world; size_t n; unsigned* state; };
void k_p2p_allreduce(const P2pArgs& a, cudaStream_t s);

// ---- GEMM-shaped kernels, SIMT (fp32 FMA) -----------------------------------------------------------------
// fprop:  out[m][o] = act(sum_k A[m][k] w[o][k] + bias[o]),  m=(n,oy,ox), k=(r,s,c);  w layout [O][KH][KW][C]
// optional per-output-channel `scale`: out = act(acc * scale[c] + bias[c])  (inference-mode BatchNorm folded into the epilogue)
void k_simt_fprop(int prec, int wprec, const ConvGeom& g, const void* x, const void* w, const float* bias, void* out, int act, float alpha, cudaStream_t s, const float* scale = nullptr);
// dgrad:  dx[m][c] = act(sum_k dy[..][o] w[o][r][s][c] + bias[c]),  m=(n,iy,ix)   (also the deconvolution forward)
void k_simt_dgrad(int prec, int wprec, const ConvGeom& g, const void* dy, const void* w, const float* bias, void* dx, int act, float alpha, cudaStream_t s, const float* scale = nullptr);
// wgrad:  dw[o][r][s][c] = sum_pixels dy[pix][o] x[pix(r,s)][c]   (fp32 out, split-K scratch of k_simt_wgrad_scratch floats)
void k_simt_wgrad(int prec, const ConvGeom& g, const void* x, const void* dy, float* dw, float* scratch, size_t scratch_floats, int accumulate, cudaStream_t s);
size_t k_simt_wgrad_scratch_floats(const ConvGeom& g);

// ---- skinny layers (kernels_edge.cu): <=4 image channels on one side, or <=4 output units ------------------
bool edge_deconv_small_c_supported(const ConvGeom& g);   // dgrad form, g.C <= 4
bool edge_conv_small_cin_supported(const ConvGeom& g);   // fprop form, g.C <= 4
bool edge_wgrad_small_cin_supported(const ConvGeom& g);
bool dense_small_o_supported(const ConvGeom& g);         // 1x1 geometry, g.O <= 4
void k_edge_deconv_small_c(int prec, int wprec, const ConvGeom& g, const void* dy, const void* w, const float* bias, void* dx, int act, float alpha, cudaStream_t s);
void k_edge_conv_small_cin(int prec, int wprec, const ConvGeom& g, const void* x, const void* w, const float* bias, void* out, int act, float alpha, cudaStream_t s);
void k_edge_wgrad_small_cin(int prec, const ConvGeom& g, const void* x, const void* dy, float* dw, float* scratch, int accumulate, cudaStream_t s);
size_t k_edge_wgrad_scratch_floats(const ConvGeom& g);
void k_dense_small_o_fwd(int prec, int wprec, const ConvGeom& g, const void* x, const void* w, const float* bias, void* out, int act, float alpha, cudaStream_t s);
void k_dense_small_o_dgrad(int prec, int wprec, const ConvGeom& g, const void* dy, const void* w, void* dx, cudaStream_t s);
void k_dense_small_o_wgrad(int prec, const ConvGeom& g, const void* x, const void* dy, float* dw, float* scratch, int accumulate, cudaStream_t s);
size_t k_dense_small_o_wgrad_scratch_floats(const ConvGeom& g);
bool dense_small_k_supported(const ConvGeom& g);         // 1x1 geometry, reduction g.O <= 128, g.C % 256 == 0 (DCGAN G-first: z -> 4x4 map)
void k_dense_small_k_dgrad(int prec, int wprec, const ConvGeom& g, const void* dy, const void* w, const float* bias, void* dx, int act, float alpha, cudaStream_t s);
void k_dense_small_k_wgrad(int prec, const ConvGeom& g, const void* x, const void* dy, float* dw, cudaStream_t s);

// ---- GEMM-shaped kernels, wgmma tensor cores (bf16 in, fp32 accumulate in registers) -------------------------
bool tc_fprop_supported(const ConvGeom& g);
bool tc_dgrad_supported(const ConvGeom& g);
bool tc_wgrad_supported(const ConvGeom& g);
int  tc_init();   // resolves cuTensorMapEncodeTiled; 0 on success
extern const char* g_tc_last_kernel;     // which tensor-core kernel the most recent k_tc_* call dispatched (parity tests assert it)
// Schedule overrides of tc_conv_kernel, set only by the kernel-level test hook around its launches (0 = production choice):
// g_tc_test_bn forces the 64- or 128-column tile, g_tc_test_max_ctas caps the persistent grid at min(work items, max_ctas)
extern int g_tc_test_bn, g_tc_test_max_ctas;
// epilogue of the fprop / dgrad kernels (kernels_tc.cu): what happens between the fp32 accumulator and the bf16 store
enum { EPI_PLAIN = 0, EPI_STATS = 1, EPI_BNBWD = 2, EPI_ACTBWD = 3 };
struct TcEpi {
  int mode;                    // EPI_*
  const float* scale;          // EPI_PLAIN / EPI_STATS: out = act(acc*scale[c] + bias[c]) (inference-mode BatchNorm folded in), may be null
  unsigned long long* acc;     // EPI_STATS: sum / sum-of-squares of the outputs; EPI_BNBWD: sum dy', sum dy'*z   [groups][2][2][OC]
  int imgs_per_group;          // statistics group = image index / imgs_per_group
  const __nv_bfloat16* aux;    // EPI_BNBWD / EPI_ACTBWD: the forward OUTPUT of the (BatchNorm +) activation whose derivative multiplies the result
  const __nv_bfloat16* aux2;   // EPI_BNBWD: the BatchNorm layer's input z
  int act; float alpha;        // EPI_BNBWD / EPI_ACTBWD: that activation
};
// w: the bf16 weight copy [O][taps][C].  w_mn = 1 (1x1 geometry): w is [C][O], the dense layer's own weight as its input-gradient operand.
int k_tc_fprop(const ConvGeom& g, const __nv_bfloat16* x, const __nv_bfloat16* w, const float* bias, __nv_bfloat16* out, int act, float alpha, cudaStream_t s, const TcEpi* epi = nullptr, int w_mn = 0);
// conv input gradient / transposed-conv forward (4x4 s2 p1, sub-pixel phases); w is the SAME straight copy [O][16][C] (MN-major weight tiles)
int k_tc_dgrad(const ConvGeom& g, const __nv_bfloat16* dy, const __nv_bfloat16* w, const float* bias, __nv_bfloat16* dx, int act, float alpha, cudaStream_t s, const TcEpi* epi = nullptr);
int k_tc_wgrad(const ConvGeom& g, const __nv_bfloat16* x, const __nv_bfloat16* dy, float* dw, float* scratch, size_t scratch_floats, int accumulate, cudaStream_t s, ReduceList* defer = nullptr);
size_t k_tc_wgrad_scratch_floats(const ConvGeom& g);
// transposed conv 4x4 s2 p1 onto <= 4 image channels as one 3x3 tensor-core conv over the 2x2 output blocks (weights packed by k_pack_deconv_ps)
bool tc_deconv_ps_shape(const ConvGeom& g);          // geometry only (allocation time)
bool tc_deconv_ps_supported(const ConvGeom& g);      // + the batch tiles into 128-pixel rows
size_t k_tc_deconv_ps_weight_elems(const ConvGeom& g);
void k_pack_deconv_ps(const float* w, __nv_bfloat16* wps, int O, int C, cudaStream_t s);
// conv 4x4 s2 p1 from <= 4 image channels (fprop form) and its weight gradient: im2col rows built in shared memory by the CTA, wgmma MMAs
bool tc_edge_conv_supported(const ConvGeom& g);
bool tc_edge_wgrad_supported(const ConvGeom& g);
size_t k_tc_edge_wgrad_scratch_floats(const ConvGeom& g);
int k_tc_edge_conv(const ConvGeom& g, const __nv_bfloat16* x, const __nv_bfloat16* w, const float* bias, __nv_bfloat16* out, int act, float alpha, cudaStream_t s);
// db (optional, g.C < 4): also the column sums of dy (= the conv bias gradient) from a ones column of the im2col tile; returns 1 if db was written, 0 if not, < 0 on error
int k_tc_edge_wgrad(const ConvGeom& g, const __nv_bfloat16* x, const __nv_bfloat16* dy, float* dw, float* db, float* scratch, size_t scratch_floats, int accumulate, cudaStream_t s, ReduceList* defer = nullptr);
int k_tc_deconv_ps(const ConvGeom& g, const __nv_bfloat16* dy, const __nv_bfloat16* wps, const float* bias, __nv_bfloat16* dx, int act, float alpha, cudaStream_t s, const TcEpi* epi = nullptr);

}  // namespace b2g
