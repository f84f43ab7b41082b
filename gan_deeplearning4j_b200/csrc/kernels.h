// kernels.h -- launch wrappers of every CUDA kernel in libb200gan.so (sm_90a only).
// Host-callable, stream-ordered, no allocation.  "prec" selects the activation storage type
// (PREC_F32 = DL4J-parity mode, PREC_BF16 = tensor-core mode); statistics, parameters, gradients and
// updater state are always fp32.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <math.h>
#include <stdint.h>

namespace b2g {

enum Prec { PREC_F32 = 0, PREC_BF16 = 1 };
enum Act { ACT_IDENTITY = 0, ACT_TANH = 1, ACT_SIGMOID = 2, ACT_RELU = 3, ACT_LRELU = 4,
           // kernels_act.cu only: the GEMM epilogues, BatchNorm, loss and act_* kernels take codes 0-4 and treat any other code as identity
           ACT_ELU = 5, ACT_SELU = 6, ACT_SOFTPLUS = 7, ACT_SOFTSIGN = 8, ACT_HARDTANH = 9, ACT_HARDSIGMOID = 10, ACT_RELU6 = 11, ACT_SWISH = 12,
           ACT_CUBE = 13, ACT_RATIONALTANH = 14, ACT_RECTIFIEDTANH = 15, ACT_THRESHOLDEDRELU = 16, ACT_EXT_FIRST = ACT_ELU, ACT_EXT_LAST = ACT_THRESHOLDEDRELU };
enum Loss { LOSS_MSE = 2, LOSS_L1 = 3, LOSS_L2 = 4, LOSS_MAE = 5, LOSS_HINGE = 6, LOSS_SQUARED_HINGE = 7, LOSS_WASSERSTEIN = 8 };   // b2g_loss

inline size_t prec_size(int prec) { return prec == PREC_F32 ? 4 : 2; }

// Convolution geometry, NHWC.  A dense layer is the 1x1 conv on a 1x1 image; a deconvolution is the
// transposed problem (its forward is this geometry's dgrad, its input-gradient this geometry's fprop).
struct ConvGeom {
  int N, H, W, C;        // conv input
  int OH, OW, O;         // conv output
  int KH, KW, SH, SW, PH, PW;
};

extern uint64_t g_launch_count;   // every kernel launch of this library bumps it (bench evidence)
// which kernel the most recent call of a reduction / loss / activation / pooling wrapper below dispatched (kernel-level tests assert it;
// k_colsum names its first stage)
extern const char* g_ew_last_kernel;
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
// b2g_activation codes 5-16 (kernels_act.cu; formulas in include/b200gan.h), one instantiation per kind: a = f(z); eps = eps * f'(z) in place.
// alpha = ELU's alpha / ThresholdedReLU's theta.  A code outside 5-16 launches nothing.
bool act_ext_kind(int act);
void k_act_ext_fwd(int prec, int act, float alpha, const void* z, void* a, size_t n, cudaStream_t s);
void k_act_ext_bwd(int prec, int act, float alpha, const void* z, void* eps, size_t n, cudaStream_t s);
void k_maxpool_fwd(int prec, const void* x, void* y, uint8_t* argmax, int N, int H, int W, int C, int OH, int OW, int KH, int KW, int SH, int SW, cudaStream_t s);
void k_maxpool_bwd(int prec, const void* eps_out, const uint8_t* argmax, void* eps_in, int N, int H, int W, int C, int OH, int OW, int KH, int KW, int SH, int SW, cudaStream_t s);
void k_upsample_fwd(int prec, const void* x, void* y, int N, int H, int W, int C, int f, cudaStream_t s);
void k_upsample_bwd(int prec, const void* eps_out, void* eps_in, int N, int H, int W, int C, int f, cudaStream_t s);

// ---- average / sum / p-norm pooling (kernels_pool.cu; formulas and summation order at b2g_pooling in include/b200gan.h) ----------------
// One instantiation per kind, precision and path (16-byte vectors when C is a multiple of the vector width and the tensors are aligned, else
// per element).  pn = PNORM's p (a whole number >= 1; ignored by the other kinds).
enum Pool { POOL_MAX = 0, POOL_AVG = 1, POOL_SUM = 2, POOL_PNORM = 3 };   // b2g_pooling
// SubsamplingLayer AVG / SUM / PNORM, Truncate geometry with zero padding; MAX launches nothing (B2G_LAYER_MAXPOOL's kernels).  The backward
// is the gather form; y = the forward's output (PNORM reads it and x).
void k_pool2d_fwd(int prec, int kind, int pn, const void* x, void* y, int N, int H, int W, int C, int OH, int OW, int KH, int KW, int SH, int SW, int PH, int PW,
                  cudaStream_t s);
void k_pool2d_bwd(int prec, int kind, int pn, const void* eps_out, const void* x, const void* y, void* eps_in, int N, int H, int W, int C, int OH, int OW, int KH,
                  int KW, int SH, int SW, int PH, int PW, cudaStream_t s);
// GlobalPoolingLayer: x [N][HW][C] -> y [N][C], MAX also idx [N][C] (the pixel of the first maximum).  Where N x channel chunks gives too few
// blocks the pixel range is split over k_global_pool_splits blocks (a function of the shape and of the vector path); their fp32 partials go to
// part / part_idx ([N][splits][C]; k_global_pool_partial_elems for every batch up to max_rows) and the last block to finish folds them (ticket
// word, 0 between launches).  One launch.
int k_global_pool_splits(int prec, int N, int HW, int C, int vec);
size_t k_global_pool_partial_elems(int prec, int max_rows, int HW, int C);
void k_global_pool_fwd(int prec, int kind, int pn, const void* x, void* y, int32_t* idx, int N, int HW, int C, float* part, int32_t* part_idx, unsigned* ticket,
                       cudaStream_t s);
void k_global_pool_bwd(int prec, int kind, int pn, const void* eps_out, const void* x, const void* y, const int32_t* idx, void* eps_in, int N, int HW, int C,
                       cudaStream_t s);
extern int g_pool_last_splits;   // the split count of the most recent k_global_pool_fwd (kernel-level tests assert it)

// ---- dropout (DL4J DropoutLayer, inverted dropout; mask definition in include/b200gan.h) ----------------------------------------
// Forward over the n elements of one pass (NHWC, element index e): y = x * (1/p) where kept, 0 where dropped, and the keep bits into
// mask[e >> 5] bit (e & 31).  The random word of element e is Philox4x32-10(ctr = {e >> 2, lo32(P), hi32(P), tag}, key = {lo32(seed), hi32(seed)})[e & 3],
// P = *pass read on the device.  bump_pass: the last block to finish advances *pass by one (ticket counter *ticket, reset by that block).
// tag = layer | rank << 16; keep where the word < threshold = floor(p * 2^32), or everywhere when keep_all (p >= 1); scale = 1.0f / p
struct DropoutArgs { uint64_t seed; uint32_t tag; uint32_t threshold; float scale; int keep_all; };
void k_dropout_fwd(int prec, const void* x, void* y, uint32_t* mask, size_t n, const DropoutArgs& a, unsigned long long* pass, unsigned* ticket, int bump_pass, cudaStream_t s);
// Backward: eps_in = eps_out * (1/p) where the forward kept the element, 0 elsewhere (eps_in may equal eps_out)
void k_dropout_bwd(int prec, const void* eps_out, void* eps_in, const uint32_t* mask, size_t n, float scale, cudaStream_t s);
// The other IDropout kinds (b2g_dropout_kind; definitions in include/b200gan.h), drawn from the same Philox stream and pass counter, and
// Dropout(p) with a schedule.  value: the layer's constant value; the rest is derived from a value by noise_derive.  scale: GAUSSIAN_DROPOUT /
// GAUSSIAN_NOISE sigma, ALPHA_DROPOUT a, DROPOUT / SPATIAL_DROPOUT 1/p; shift: ALPHA_DROPOUT b; fill: ALPHA_DROPOUT a' = -lambda alpha.
// hw, C: SPATIAL_DROPOUT's map (pixels per row, channels); its keep bit of (row, c) is mask bit j = row * C + c.
enum DropKind { DROP_BERNOULLI = 0, DROP_GAUSSIAN_DROPOUT = 1, DROP_GAUSSIAN_NOISE = 2, DROP_ALPHA = 3, DROP_SPATIAL = 4 };
struct NoiseArgs { uint64_t seed; uint32_t tag; uint32_t threshold; float value, scale, shift, fill; int keep_all; int hw, C; };
// A scheduled value outside its kind's range is clamped into it: p to [2^-32, 1], rate to [0, 1 - 2^-24], sigma to >= 0
__host__ __device__ inline float noise_clamp(int kind, float v) {
  if (kind == DROP_GAUSSIAN_DROPOUT) return fminf(fmaxf(v, 0.f), 0x1.fffffep-1f);
  if (kind == DROP_GAUSSIAN_NOISE) return fmaxf(v, 0.f);
  return fminf(fmaxf(v, 0x1p-32f), 1.f);
}
// The kernels' constants of value v, each computed in double and rounded to fp32 once (include/b200gan.h b2g_dropout_kind)
__host__ __device__ inline void noise_derive(int kind, float v, NoiseArgs& a) {
  if (kind == DROP_GAUSSIAN_DROPOUT) { a.scale = (float)sqrt((double)v / (1.0 - (double)v)); return; }
  if (kind == DROP_GAUSSIAN_NOISE) { a.scale = v; return; }
  a.keep_all = v >= 1.f ? 1 : 0; a.threshold = a.keep_all ? 0u : (uint32_t)floor((double)v * 4294967296.0);
  if (kind == DROP_ALPHA) {        // SELU's alpha and lambda
    const double ap = -1.0507009873554805 * 1.6732632423543772, p = v, A = 1.0 / sqrt(p + ap * ap * p * (1.0 - p));
    a.scale = (float)A; a.shift = (float)(-A * (1.0 - p) * ap); a.fill = (float)ap;
  } else a.scale = 1.0f / v;
}
// What a forward drew with, for its backward: the pass counter P (GAUSSIAN_DROPOUT draws m again) and the value (scheduled layers)
struct NoiseRec { unsigned long long P; float v; };
// A scheduled layer (sched != null): every block takes the value from the schedule at the iteration *step (before the update's increment) or
// the epoch *epoch, clamps it and derives the constants from it; the forward records the value in rec, the backward reads it from there.
struct UpdSched;
struct NoiseSched { const UpdSched* sched; const int* step; const int64_t* epoch; };
// Forward of a DropoutLayer other than unscheduled Dropout(p).  mask: DROPOUT / ALPHA one bit per element, SPATIAL one per (row, channel).
void k_noise_fwd(int prec, int kind, const void* x, void* y, uint32_t* mask, NoiseRec* rec, size_t n, const NoiseArgs& a, const NoiseSched& q,
                 unsigned long long* pass, unsigned* ticket, int bump_pass, cudaStream_t s);
// Its backward (eps_in may equal eps_out); GAUSSIAN_NOISE is the identity and launches nothing.
void k_noise_bwd(int prec, int kind, const void* eps_out, void* eps_in, const uint32_t* mask, const NoiseRec* rec, size_t n, const NoiseArgs& a,
                 const NoiseSched& q, cudaStream_t s);
// *out = the clamped value the next forward of a layer of this kind uses (one thread, one launch)
void k_noise_value(int kind, float value, const NoiseSched& q, float* out, cudaStream_t s);


// ---- loss ----------------------------------------------------------------------------------------------
// LossBinaryXENT on logits z[rows] with labels y[rows]: dz = dL/dz (sum form, not /mb), loss_sums[g] = sum of losses per group.
void k_xent(int prec, const void* z, const float* y, void* dz, float* loss_sums, int rows_per_group, int groups, float clip_eps, cudaStream_t s);
void k_sigmoid_out(int prec, const void* z, void* p, size_t n, cudaStream_t s);
// LossMCXENT + softmax over K classes: dz = softmax(z) - y, loss_sums[0] = -sum y log clip(p, 1e-10); p_out optional (probabilities)
void k_softmax_xent(int prec, const void* z, const float* y, void* dz, void* p_out, float* loss_sums, int rows, int K, cudaStream_t s);
// LossMSE / L1 / L2 / MAE / Hinge / SquaredHinge / Wasserstein (b2g_loss 2-8) on a = act(z), z and y [groups][rows][n_out]: dz = dL/da * act'(a)
// (sum form, not /mb), loss_sums[g] = the group's summed per-example scores.  One launch; the sums are bit-reproducible: partial
// [groups * k_loss_blocks(rows * n_out, groups)] doubles and a ticket word (0 between launches) hold the per-block sums the last block folds.
int k_loss_blocks(size_t n_per_group, int groups);
void k_loss(int prec, int loss, int act, float alpha, const void* z, const float* y, void* dz, float* loss_sums, int rows_per_group, int n_out, int groups,
            double* partial, unsigned* ticket, cudaStream_t s);
// CnnLossLayer (kernels_cnnloss.cu; summation orders stated there): sigmoid XENT over groups x n_per_group elements, and softmax MCXENT over
// the C channels of groups x rows_per_group NHWC pixels (y = null: the inference call, p_out only).  dz in the sum form, loss_sums[g] = group
// g's summed scores.  partial: [groups * k_loss_blocks(n_per_group, groups)] (XENT) / [groups * k_cnn_softmax_blocks(rows_per_group, groups)]
// (MCXENT) doubles, at most 1024; ticket: 0 between launches.
void k_cnn_xent(int prec, const void* z, const float* y, void* dz, float* loss_sums, size_t n_per_group, int groups, float clip_eps, double* partial,
                unsigned* ticket, cudaStream_t s);
int k_cnn_softmax_blocks(int rows_per_group, int groups);
void k_cnn_softmax_xent(int prec, const void* z, const float* y, void* dz, void* p_out, float* loss_sums, int rows_per_group, int C, int groups,
                        double* partial, unsigned* ticket, cudaStream_t s);
// Per-output weights and label mask of a loss (b2g_net_set_loss_weights / the masked fit; semantics at b2g_loss).  w: [C] or null; m: the
// mask, [rows][mw] in the rows of the labels (examples, or NHWC pixels of a CnnLossLayer) with mw = 1 or C, or null; C: the columns (nOut,
// or the channels of a CnnLossLayer).  A wrapper given null (or a LossWM with neither) launches its unweighted instantiation.
struct LossWM { const float* w; const float* m; int mw; int C; };
// The weighted / masked instantiations of the five loss kernels: the same launch, slicing and summation order as the wrappers above.
void k_xent_wm(int prec, const void* z, const float* y, void* dz, float* loss_sums, int rows_per_group, int groups, float clip_eps, const LossWM& wm, cudaStream_t s);
void k_softmax_xent_wm(int prec, const void* z, const float* y, void* dz, float* loss_sums, int rows, int K, const LossWM& wm, cudaStream_t s);
void k_loss_wm(int prec, int loss, int act, float alpha, const void* z, const float* y, void* dz, float* loss_sums, int rows_per_group, int n_out, int groups,
               double* partial, unsigned* ticket, const LossWM& wm, cudaStream_t s);
void k_cnn_xent_wm(int prec, const void* z, const float* y, void* dz, float* loss_sums, size_t n_per_group, int groups, float clip_eps, double* partial,
                   unsigned* ticket, const LossWM& wm, cudaStream_t s);
void k_cnn_softmax_xent_wm(int prec, const void* z, const float* y, void* dz, float* loss_sums, int rows_per_group, int C, int groups,
                           double* partial, unsigned* ticket, const LossWM& wm, cudaStream_t s);

// ---- skip-connection vertices (kernels_graph.cu; semantics at b2g_elementwise_op in include/b200gan.h) ----------------------------
// One launch each.  a, b: the vertex's inputs in its input order.  The fp32 accumulator acc of a skip source is written (accumulate = 0, the
// first contributor of a backward pass) or added to (1).
enum VertexOp { VERTEX_ADD = 0, VERTEX_SUBTRACT = 1, VERTEX_PRODUCT = 2, VERTEX_AVERAGE = 3, VERTEX_MAX = 4 };   // b2g_elementwise_op
void k_vertex_ew_fwd(int prec, int op, const void* a, const void* b, void* y, size_t n, cudaStream_t s);
// eps (w.r.t. the vertex output) becomes the spine's share in place; the skip's share goes to acc.  order 0: inputs (spine, skip), 1: (skip, spine)
void k_vertex_ew_bwd(int prec, int op, int order, void* eps, const void* spine, const void* skip, float* acc, int accumulate, size_t n, cudaStream_t s);
// y [P][Ca + Cb] = concat(a [P][Ca], b [P][Cb]) per pixel (NHWC channel concat; [N][F] vectors with P = N)
void k_merge_fwd(int prec, const void* a, const void* b, void* y, size_t P, int Ca, int Cb, cudaStream_t s);
// eps [P][Ca + Cb] -> the spine's slice into dst (T), the skip's into acc (fp32).  spine_first: the spine is the first input
void k_merge_bwd(int prec, const void* eps, void* dst, float* acc, size_t P, int Ca, int Cb, int spine_first, int accumulate, cudaStream_t s);
// eps = eps + acc in fp32, rounded once to T (the skip gradient joining the spine at its source)
void k_skip_add(int prec, void* eps, const float* acc, size_t n, cudaStream_t s);

// ---- PReLULayer (kernels_prelu.cu; semantics and summation order at B2G_LAYER_PRELU in include/b200gan.h) ---------------------------
// A [rows][H][W][C] map (a feed-forward input: H = W = 1, C = F).  The slopes alpha are in DL4J's order [C][H][W] with every axis whose bit is
// set in `shared` (1 = C, 2 = H, 4 = W) of extent 1: K = prelu_slopes slopes, each shared by S = H*W*C / K positions of a row.
struct PreluGeom { int H, W, C, shared; };
__host__ __device__ inline size_t prelu_slopes(const PreluGeom& g) {
  return (size_t)((g.shared & 1) ? 1 : g.C) * ((g.shared & 2) ? 1 : g.H) * ((g.shared & 4) ? 1 : g.W);
}
// The backward's row groups for `rows` rows (a function of the shape only): *groups groups of *rows_per_group consecutive rows, the last ragged
void prelu_row_groups(int rows, const PreluGeom& g, int* groups, int* rows_per_group);
// fp32 partial sums the backward of a pass of up to max_rows rows writes
size_t k_prelu_part_floats(int max_rows, const PreluGeom& g);
// y = x < 0 ? alpha*x : x (one launch)
void k_prelu_fwd(int prec, const void* x, void* y, const float* alpha, int rows, const PreluGeom& g, cudaStream_t s);
// One launch: eps = x < 0 ? alpha*eps : eps in place (write_dx); part (may be null): part[(grp*S + s)*K + k] = the fp32 sum, over the rows of
// row group grp in ascending order, of x*eps (x < 0) at the position s of slope k
void k_prelu_bwd(int prec, const void* x, void* eps, const float* alpha, float* part, int write_dx, int rows, const PreluGeom& g, cudaStream_t s);
// Queues dalpha[k] = sum over t < groups*S of part[t*K + k] as one job of a reduce list (k_reduce_multi sums it)
struct ReduceList;
void prelu_queue_reduce(ReduceList* rl, const float* part, float* dalpha, int rows, const PreluGeom& g);

// ---- reductions ------------------------------------------------------------------------------------
// out[c] (+)= sum_rows x[row][c]
void k_colsum(int prec, const void* x, int rows, int C, float* scratch, float* out, int accumulate, cudaStream_t s);
size_t k_colsum_scratch_floats(int C);
// out[0] = sum_i coef[i] * x[i]^2 over the listed segments (l2 score); segments with coef 0 are skipped
void k_sumsq_segments(const float* p, const int64_t* seg_off, const int64_t* seg_len, const float* seg_coef, int nseg, double* out, cudaStream_t s);
// out[0] = sum_i coef[i] * |x[i]| over the listed segments (l1 score), in the order of k_sumsq_segments; segments with coef 0 are skipped
void k_sumabs_segments(const float* p, const int64_t* seg_off, const int64_t* seg_len, const float* seg_coef, int nseg, double* out, cudaStream_t s);
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
  int kind;                // b2g_updater: 0 sgd, 1 rmsprop, 2 adam, 3 noop, 4 nesterovs, 5 adagrad, 6 adamax, 7 nadam, 8 amsgrad, 9 adadelta
  float lr, b1, b2, eps;   // rmsprop: b1 = rmsDecay; nesterovs: b1 = momentum; adadelta: b1 = rho (lr unused)
  float l2;                // post-updater, not lr-scaled (pre-beta4): u = fmaf(l2, p, u)
  float l1;                // then u += l1 * sign(p), sign(+-0) = 0; W takes the layer's l1 / l2, b its l1Bias / l2Bias
  float clip;              // elementwise clip threshold, 0 = off
  int div_mb;              // 0 for BN mean/var pseudo-gradients
  // bf16 shadow of a conv/deconv/dense weight: shadow[off_bf..] same layout [A][taps][B]; off_ps >= 0: also the packed [16][9][ps_O] operand of
  // the pixel-shuffle transposed conv (kernels_tc.cu k_pack_deconv_ps), every weight element has exactly one slot there
  int64_t off_bf, off_ps;
  int ps_O, ps_C;
};
// Writes the bf16 value pb of parameter element i (an index into the flattened vector, inside sg) to its slot(s) of the bf16 weight operands:
// the straight copy, and the packed pixel-shuffle operand where sg has one.  Shared by the updater and the weight constraints.
__device__ __forceinline__ void upd_shadow(const UpdSeg& sg, __nv_bfloat16* __restrict__ shadow, int64_t i, __nv_bfloat16 pb) {
  shadow[sg.off_bf + (i - sg.off)] = pb;
  if (sg.off_ps >= 0) {       // [O][4][4][C] element -> its one slot of the packed [(py,px,c4)][(dyr,dxc)][O] pixel-shuffle operand (kernels_tc.cu pack_deconv_ps_kernel)
    const int e = (int)(i - sg.off), c = e % sg.ps_C, tap = (e / sg.ps_C) % 16, o = e / (sg.ps_C * 16), r = tap >> 2, sx = tap & 3;
    const int py = (r == 0 || r == 2) ? 1 : 0, dyr = r == 3 ? -1 : r == 0 ? 1 : 0, px = (sx == 0 || sx == 2) ? 1 : 0, dxc = sx == 3 ? -1 : sx == 0 ? 1 : 0;
    shadow[sg.off_ps + ((int64_t)((py * 8 + px * 4 + c) * 9 + (dyr + 1) * 3 + (dxc + 1))) * sg.ps_O + o] = pb;
  }
}
// Learning-rate schedule of one segment (b2g_lr_schedule; kind 0 = the segment's constant lr).  keys / vals: the MAP schedule's entries in
// the net's device memory.  Kept beside UpdSeg, not in it, so that the unscheduled updater reads the segment table it always read.
struct UpdSched {
  int kind, type;          // b2g_schedule_kind, b2g_schedule_type
  int n_map;
  double initial, gamma, power, step, decay;
  const int32_t* keys; const double* vals;
};
// The last block to finish bumps *step_dev (Adam's t) and resets *ticket: no separate counter kernel.
// gn_mult (may be null): one fp32 multiplier per segment (k_gradnorm), applied to g right after the minibatch division.
// sched (may be null): one UpdSched per segment; each block then takes its segment's lr from the schedule at iteration *step_dev (before the
// increment) or at epoch *epoch_dev, both read from device memory.
// ext: some segment has a kind >= 4 (then the extended instantiations run; every other net launches the kernels it always launched).  st2: the
// third state slot (AMSGrad's v-hat), may be null when no segment is AMSGrad.
void k_updater(float* params, const float* grads, float* st0, float* st1, float* st2, const UpdSeg* segs_dev, const int32_t* chunk_seg_dev,
               const int64_t* chunk_off_dev, int nchunks, float inv_mb, float inv_world, int* step_dev /* t = *step_dev + 1 */, unsigned* ticket,
               __nv_bfloat16* shadow, const float* gn_mult, const UpdSched* sched, const int64_t* epoch_dev, bool ext, cudaStream_t s);
// *out = the fp32 learning rate the updater kernel would use for segment seg at the current *step_dev / *epoch_dev (one thread, one launch)
void k_sched_lr(const UpdSeg* segs_dev, const UpdSched* sched, int seg, const int* step_dev, const int64_t* epoch_dev, float* out, cudaStream_t s);
static const int UPD_CHUNK = 4096;
// The learning rate of a segment at iteration `it` (the counter before this update's increment) / epoch `ep`: DL4J's ISchedule.valueAt in
// double, rounded to fp32 once (include/b200gan.h, b2g_lr_schedule); kind 0 = the constant lr.  Also the scheduled DropoutLayer value.
__device__ inline float sched_lr(const UpdSched& sc, float lr, int it, long long ep) {
  if (sc.kind == 0) return lr;
  const long long ii = sc.type == 1 ? ep : (long long)it;
  const double i = (double)ii;
  double v;
  if (sc.kind == 1) v = sc.initial * pow(sc.gamma, i);
  else if (sc.kind == 2) v = sc.initial / pow(1.0 + sc.gamma * i, sc.power);
  else if (sc.kind == 3) v = sc.initial / (1.0 + exp(-sc.gamma * (i - sc.step)));
  else if (sc.kind == 4) v = sc.initial * pow(sc.decay, floor(i / sc.step));
  else {          // MAP: the largest key <= i (keys strictly increase, keys[0] <= 0 <= i)
    int lo = 0, hi = sc.n_map - 1;
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if ((long long)sc.keys[mid] <= ii) lo = mid; else hi = mid - 1; }
    v = sc.vals[lo];
  }
  return (float)v;
}

// ---- weight noise (DL4J DropConnect / WeightNoise; definitions at b2g_weight_noise in include/b200gan.h) ------------------------------
// One job = one noisy tensor: n fp32 master elements src[0, n) drawn with indices j = j0 + i and counter word 3 = layer | rank << 16.  Output:
// dst_f32[i] (FP32 nets' W, every b), or for BF16 W the bf16 value through upd_shadow(sg, dst_bf16, i, .) (sg.off = 0: the straight copy at
// sg.off_bf, and the packed pixel-shuffle slot at sg.off_ps >= 0).  Blocks [blk_begin, blk_begin + blocks) of the launch serve the job,
// WN_CHUNK elements each (4 per thread, one Philox call).  sched (DROPCONNECT, may be null): thread 0 of each block evaluates p.
enum { WN_DROPCONNECT = 1, WN_WEIGHTNOISE = 2 };   // b2g_weight_noise_kind
enum { WN_NORMAL = 0, WN_UNIFORM = 1 };            // b2g_distribution_kind
static const int WN_CHUNK = 1024;
struct WnJob {
  const float* src; int64_t n, j0;
  float* dst_f32; __nv_bfloat16* dst_bf16; UpdSeg sg;
  int layer, kind, dist, additive;
  float p, a, b;                 // DROPCONNECT p; WEIGHTNOISE NORMAL (mean, std) / UNIFORM (lower, upper)
  const UpdSched* sched;
  int blk_begin, blocks;
};
// jobs: device table of njobs jobs, nblocks blocks in all.  P = *pass read on the device; bump_pass: the last block advances *pass (ticket as
// k_dropout_fwd).  step / epoch: the counters scheduled jobs read.
void k_weight_noise(const WnJob* jobs, int njobs, int nblocks, uint64_t seed, int rank, const int* step, const int64_t* epoch, unsigned long long* pass,
                    unsigned* ticket, int bump_pass, cudaStream_t s);

// ---- weight initialization (DL4J WeightInit / Distribution / biasInit; definitions at b2g_weight_init in include/b200gan.h; kernels_init.cu) ----
// What a scheme draws, resolved on the host: a b2g_distribution_kind (not ORTHOGONAL) with its fp32 parameters, or WI_IDENTITY.
enum { WI_NORMAL = 0, WI_UNIFORM = 1, WI_TRUNCATED_NORMAL = 2, WI_LOG_NORMAL = 3, WI_BINOMIAL = 4, WI_CONSTANT = 5, WI_IDENTITY = 6 };
struct WiDraw {
  int kind;
  float a, b;                    // NORMAL / TRUNCATED_NORMAL / LOG_NORMAL (mean, std); UNIFORM (lower, upper); CONSTANT a
  int trials; uint64_t thr;      // BINOMIAL: nTrials and floor(p 2^32) (up to 2^32)
};
// W (the fp32 master of A*taps*B elements in the internal [A][taps][B] order) drawn element by element at its DL4J view index j =
// (a*B + b)*taps + t, with counter word 3 = layer | 0x80000000; bias[0, n_bias) = bias_init (bias may be null).  One launch.
void k_weight_init(float* w, int A, int taps, int B, const WiDraw& d, float* bias, int n_bias, float bias_init, uint64_t seed, int layer, cudaStream_t s);

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
// ---- weight constraints (DL4J LayerConstraint: MaxNorm, MinMaxNorm, UnitNorm, NonNegative; kernels_constraint.cu) ----------------------
// One job = one constraint on one parameter tensor.  The tensor (internal layout, an UpdSeg for its place and bf16 operands; off_bf < 0: none)
// is viewed as [K0][R0][K1][R1][K2]: a group is one (k0, k1, k2), its elements (r0, r1) in that order, j = r0*R1 + r1 < R.  K2 > 1 exactly
// when the tensor's innermost axis is kept (the groups are strided: a deconv W per output unit, a conv W over {0}, a dense W over {1}).
//   CON_ONEPASS  (K2 == 1, R <= CON_CHUNK): one block per group; reads the group once into registers, scales, writes.
//   CON_TWOPASS  the rest: a norm launch of per-chunk double partials whose last block folds them into one multiplier per group, then a scale
//                launch over the tensor.  K2 == 1: one block per (group, chunk of CON_CHUNK j's);  K2 > 1: one block per (k0, k1, tile of 32
//                k2, chunk of CON_SCHUNK j's), lane l of each warp reading group k2 = 32 tile + l (consecutive addresses).
//   CON_ELEMWISE NonNegative: one block per CON_CHUNK elements.
// blk_begin / blocks: the job's blocks in its one-pass or norm launch; blk2_begin / blocks2: in its scale launch; partials at
// partial[part_begin + g*chunks + c], multipliers at mult[mult_begin + g].
enum { CON_ONEPASS = 0, CON_TWOPASS = 1, CON_ELEMWISE = 2 };
static const int CON_CHUNK = 4096, CON_SCHUNK = 256;
struct ConJob {
  UpdSeg sg;
  int kind, path;           // b2g_constraint_kind, CON_*
  double max_norm, min_norm, rate;
  int K0, R0, K1, R1, K2, groups, R;
  int blk_begin, blocks, blk2_begin, blocks2, chunks;
  int64_t part_begin, mult_begin;
};
// jobs[j0, j1) of one round, all of them of CON_ONEPASS / CON_ELEMWISE paths, in ONE launch of `blocks` blocks
void k_constraint_onepass(float* params, __nv_bfloat16* shadow, const ConJob* jobs, int j0, int j1, int blocks, cudaStream_t s);
// jobs[j0, j1) of one round, all CON_TWOPASS: the norm launch (norm_blocks) then the scale launch (scale_blocks)
void k_constraint_twopass(float* params, __nv_bfloat16* shadow, const ConJob* jobs, int j0, int j1, int norm_blocks, int scale_blocks, double* partial,
                          unsigned* ticket, float* mult, cudaStream_t s);
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
// which SIMT / skinny-layer / dense kernel the most recent k_simt_* / k_edge_* / k_dense_* call below dispatched, and the number of split-K
// partial sums it reduced (wgrad_splits, edge_wgrad_ctas, dense_wgrad_splits; 1 where the kernel has no split).  Kernel-level tests assert both.
extern const char* g_gemm_last_kernel;
extern int g_gemm_last_splits;

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

// ---- few-output conv, BF16 nets (kernels_head.cu): k x k conv (KH*KW > 1, KH, KW <= 7, stride 1-2, 0 <= pad < kernel) from C % 8 == 0
// channels onto O <= 4 on a map wider than one pixel (the PatchGAN head).  w: the bf16 weight copy [O][taps][C].  Forward and input gradient
// take bias / activation (codes 0-4); the weight gradient writes fp32 partials [splits][O][taps][C] into part (k_head_wgrad_scratch_floats for
// the production split count; force_splits > 0 forces a count, splits past the last pixel are empty) and queues their sum into defer, or
// sums them at once when defer is null.  Returns -1 when part is too small.
bool head_conv_supported(const ConvGeom& g);
size_t k_head_wgrad_scratch_floats(const ConvGeom& g);
void k_head_fwd(const ConvGeom& g, const __nv_bfloat16* x, const __nv_bfloat16* w, const float* bias, __nv_bfloat16* out, int act, float alpha, cudaStream_t s);
void k_head_dgrad(const ConvGeom& g, const __nv_bfloat16* dy, const __nv_bfloat16* w, const float* bias, __nv_bfloat16* dx, int act, float alpha, cudaStream_t s);
int k_head_wgrad(const ConvGeom& g, const __nv_bfloat16* x, const __nv_bfloat16* dy, float* dw, float* part, size_t part_floats, int force_splits, cudaStream_t s,
                 ReduceList* defer);

// ---- GEMM-shaped kernels, wgmma tensor cores (bf16 in, fp32 accumulate in registers) -------------------------
bool tc_fprop_supported(const ConvGeom& g);
bool tc_dgrad_supported(const ConvGeom& g);
bool tc_wgrad_supported(const ConvGeom& g);
int  tc_init();   // resolves cuTensorMapEncodeTiled; 0 on success
extern const char* g_tc_last_kernel;     // which tensor-core kernel the most recent k_tc_* call dispatched (parity tests assert it)
// Schedule overrides of tc_conv_kernel, set only by the kernel-level test hook around its launches (0 = production choice):
// g_tc_test_bn forces the 64- or 128-column tile, g_tc_test_max_ctas caps the persistent grid at min(work items, max_ctas)
extern int g_tc_test_bn, g_tc_test_max_ctas;
// g_tc_test_per_tap keeps 4x4 s2 p1 fprop / dgrad on the per-tap activation loads; g_tc_last_slab: the most recent fprop / dgrad launch
// loaded its activations as 2x2-tap slabs (kernels_tc.cu slab_tile)
extern int g_tc_test_per_tap;
extern bool g_tc_last_slab;
// g_tc_test_splits forces the split count of the weight gradients: tc_wgrad_kernel's grid.x (any value >= 1; splits past the last K-block are
// empty) and tc_edge_wgrad_kernel's CTA target (tiles_per_cta = ceil(tiles / splits)); g_tc_test_max_ctas is tc_edge_conv_kernel's CTA target
// the same way.  g_tc_last_splits: the split count the most recent k_tc_wgrad / k_tc_edge_wgrad launched
extern int g_tc_test_splits, g_tc_last_splits;
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
