// engine.cu -- host side of libb200gan.so: the chain-graph executor (ComputationGraph.init / output /
// computeGradientAndScore / fit), the fused adversarial step, the NCCL gradient all-reduce, and the
// C-ABI declared in include/b200gan.h.
//
// What it replaces in the reference (J = Java/src/main/java/org/deeplearning4j/dl4jGANComputerVision.java):
//   ComputationGraph.init()            J:166,222,311   -> b2g_net_create   (one arena: params | grads | updater state | activations)
//   ComputationGraph.output()          J:170,420       -> b2g_net_output
//   SparkComputationGraph.fit()        J:426,471       -> b2g_net_fit / b2g_gan_step
//   Layer.getParam/setParam            J:429-510       -> b2g_net_get_param / b2g_net_set_param (aliasing inside b2g_gan)
//   ParameterAveragingTrainingMaster   J:325-333       -> b2g_ctx_comm_init + ncclAllReduce of the gradient vector
// Arithmetic contract: oracle/dl4j_oracle.py (DL4J 1.0.0-beta3 semantics).
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/b200gan.h"
#include "kernels.h"

using namespace b2g;

// ------------------------------------------------------------------ errors ---------------------------
static thread_local char g_err[1024] = "";
static int32_t fail(int32_t code, const char* fmt, ...) {
  va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof(g_err), fmt, ap); va_end(ap); return code;
}
#define CU(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return fail(B2G_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); } while (0)
#define B2(call) do { int32_t r_ = (call); if (r_ != 0) return r_; } while (0)
#define CHECK_KERNELS() CU(cudaGetLastError())

// ------------------------------------------------------------------ NCCL (dlopen, no link-time dep) ----
struct NcclId { char internal[128]; };
typedef int (*fn_ncclGetUniqueId)(NcclId*);
typedef int (*fn_ncclCommInitRank)(void**, int, NcclId, int);
typedef int (*fn_ncclAllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t);
typedef int (*fn_ncclAllGather)(const void*, void*, size_t, int, void*, cudaStream_t);
typedef int (*fn_ncclCommDestroy)(void*);
typedef const char* (*fn_ncclGetErrorString)(int);
static struct { void* h; fn_ncclGetUniqueId uid; fn_ncclCommInitRank init; fn_ncclAllReduce ar; fn_ncclAllGather ag; fn_ncclCommDestroy destroy; fn_ncclGetErrorString errstr; } g_nccl = {};
static int32_t nccl_load() {
  if (g_nccl.h) return 0;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  for (const char* n : names) { g_nccl.h = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (g_nccl.h) break; }
  if (!g_nccl.h) return fail(B2G_ERR_NCCL, "dlopen(libnccl.so.2) failed: %s", dlerror());
  g_nccl.uid = (fn_ncclGetUniqueId)dlsym(g_nccl.h, "ncclGetUniqueId");
  g_nccl.init = (fn_ncclCommInitRank)dlsym(g_nccl.h, "ncclCommInitRank");
  g_nccl.ar = (fn_ncclAllReduce)dlsym(g_nccl.h, "ncclAllReduce");
  g_nccl.ag = (fn_ncclAllGather)dlsym(g_nccl.h, "ncclAllGather");
  g_nccl.destroy = (fn_ncclCommDestroy)dlsym(g_nccl.h, "ncclCommDestroy");
  g_nccl.errstr = (fn_ncclGetErrorString)dlsym(g_nccl.h, "ncclGetErrorString");
  if (!g_nccl.uid || !g_nccl.init || !g_nccl.ar || !g_nccl.destroy) return fail(B2G_ERR_NCCL, "libnccl is missing symbols");
  return 0;
}
#define NC(call) do { int e_ = (call); if (e_ != 0) return fail(B2G_ERR_NCCL, "%s -> %s", #call, g_nccl.errstr ? g_nccl.errstr(e_) : "nccl error"); } while (0)

// ------------------------------------------------------------------ context --------------------------
struct b2g_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaStream_t side = nullptr;          // weight-gradient kernels run here, concurrently with the input-gradient chain
  cudaStream_t side2 = nullptr;         // the generator's train-mode forward of the G step runs here, under the D step
  cudaEvent_t ev_a = nullptr, ev_b = nullptr;
  cudaStream_t comm_stream = nullptr;   // bucketed gradient all-reduce: the tail bucket travels here while backward continues
  cudaEvent_t ev_c0 = nullptr, ev_c1 = nullptr, ev_c2 = nullptr;
  cudaDeviceProp prop;
  void* comm = nullptr; int world = 1, rank = 0;
  // gradient all-reduce over peer memory (b2g_net_enable_p2p_allreduce): this GPU's flag words, its {epoch, counter} and every rank's flags as mapped here
  unsigned* p2p_flags = nullptr; unsigned* p2p_state = nullptr; unsigned* p2p_peer_flags[8] = {}; bool p2p_flags_mapped = false;
  bool tc_ok = false;
  cudaEvent_t t0 = nullptr, t1 = nullptr; void* flush_buf = nullptr; size_t flush_bytes = 0;
};

struct LayerRT {
  b2g_layer_desc d;
  int ih = 1, iw = 1, ic = 1, oh = 1, ow = 1, oc = 1;         // per-example NHWC dims
  size_t in_elems = 0, out_elems = 0;
  ConvGeom geom{};                                             // conv-equivalent geometry (N filled per call)
  int64_t off_W = -1, n_W = 0, off_b = -1, off_gamma = -1, off_beta = -1, off_mean = -1, off_var = -1;
  b2g_regularization reg{};                                    // l1, l2 (W), l1_bias, l2_bias (b) of a GEMM layer (b2g_net_set_regularization)
  int64_t off_W_bf = -1;                                       // bf16 operand copy [A][taps][B] (written by the updater itself); serves fprop, dgrad (MN-major tiles) and wgrad
  int64_t off_Wps_bf = -1;                                     // packed [16][9][O] weights of the tensor-core pixel-shuffle transposed conv (<= 4 image channels)
  int wA = 0, wTaps = 0, wB = 0;                               // internal weight layout [A][taps][B]
  void* out = nullptr; bool out_alias = false;
  void* probs = nullptr;                                       // OUTPUT / LOSS: the output activation of the logits (sigmoid, softmax or loss_act)
  int loss_act = ACT_IDENTITY; float loss_alpha = 0.f;         // OUTPUT / LOSS with loss codes 2-8: the activation the loss applies to z
  // b2g_activation codes 5-16 (kernels_act.cu): the layer's kind and alpha, moved out of d.act (which then reads identity, so no kernel that takes
  // codes 0-4 ever sees them); ext_z: a GEMM layer's pre-activation z, from which both f and f' are computed
  int ext_act = 0; float ext_alpha = 0.f; void* ext_z = nullptr;
  uint8_t* argmax = nullptr;
  // SUBSAMPLING / GLOBAL_POOLING (kernels_pool.cu): the b2g_pooling kind (from d.act) and PNORM's p (from act_alpha); a global MAX layer's
  // pixel index per (example, channel), and the split partials and ticket word of its forward
  int pool = 0, pnorm = 0;
  int32_t* pool_idx = nullptr; float* pool_part = nullptr; int32_t* pool_part_idx = nullptr; unsigned* pool_ticket = nullptr;
  float* bn_mean = nullptr; float* bn_invstd = nullptr; float* bn_fold = nullptr;   // bn_fold: [scale | shift] for the inference-mode epilogue fold
  float* bn_coef = nullptr;                                    // fused path: [groups][4][C] = scale, beta, mean, invstd of the latest train-mode forward
  unsigned long long *acc_fwd = nullptr, *acc_bwd = nullptr;   // fused path: 128-bit statistics accumulators (forward: sum x, sum x^2; backward: sum dy', sum dy'*xhat)
  bool fwd_fused = false; int fwd_groups = 1;                  // the latest train-mode forward of this BatchNorm took the accumulator path (so must its backward)
  bool stats_by_producer = false, bwd_premul = false;          // set per pass: the producing GEMM's epilogue has already filled acc_fwd / (acc_bwd and eps = dy')
  int fused_act = ACT_IDENTITY; float fused_alpha = 0.f;       // BN followed by an ActivationLayer
  bool act_fused_into_prev = false;
  float* wg_part = nullptr; size_t wg_part_floats = 0;         // split-K partials of this layer's tensor-core weight gradient (reduced by ONE k_reduce_multi per pass)
  // DropoutLayer: its own output buffer (never its input: the layer below differentiates from its own pre-dropout output) and the 1-bit
  // keep mask of the latest train-mode forward; `out` is drop_buf after a masked forward and the input itself after a pass-through one
  void* drop_buf = nullptr; uint32_t* drop_mask = nullptr; bool drop_live = false;
  // the other kinds (b2g_dropout_kind in d.act): the mask is per element (ALPHA), per (row, channel) (SPATIAL) or absent (Gaussian kinds);
  // drop_rec: the P and value of the latest forward (GAUSSIAN_DROPOUT's backward draws m again from them; a scheduled backward takes the
  // forward's value).  drop_sched: b2g_net_set_dropout_schedule gave the layer a schedule, held on the device in drop_sched_dev (MAP entries
  // in drop_map); such a layer is stochastic whatever its value
  NoiseRec* drop_rec = nullptr; UpdSched* drop_sched_dev = nullptr; bool drop_sched = false; void* drop_map = nullptr;
  // ELEMENTWISE / MERGE (include/b200gan.h): the skip source j (d.pre_h), the input order (d.pre_w), and whether this vertex is the first
  // consumer of j the backward visits (it writes j's accumulator; the later ones add).  A skip source: its consumer count and fp32 accumulator.
  int vsrc = -1, vorder = 0; bool vfirst = false;
  int n_skip = 0; float* skip_acc = nullptr;
  // PRELU (kernels_prelu.cu): the map and shared-axes mask; the slope gradient's row-group partials (non-frozen layers)
  PreluGeom pg{}; float* prelu_part = nullptr;
  // a stochastic DropoutLayer: train mode draws from the pass counter.  FrozenLayer: test mode, identity; p = 1, rate = 0, stddev = 0: identity
  bool drop_active() const {
    if (d.type != B2G_LAYER_DROPOUT || d.frozen) return false;
    if (drop_sched) return true;
    return d.act == B2G_DROPOUT_GAUSSIAN_DROPOUT || d.act == B2G_DROPOUT_GAUSSIAN_NOISE ? d.act_alpha > 0.f : d.act_alpha < 1.f;
  }
  bool has_gemm() const { return d.type == B2G_LAYER_CONV2D || d.type == B2G_LAYER_DECONV2D || d.type == B2G_LAYER_DENSE || d.type == B2G_LAYER_OUTPUT; }
  // a layer whose W takes l1 / l2 (b2g_regularization): the GEMM layers and PReLU's slopes
  bool has_reg() const { return has_gemm() || d.type == B2G_LAYER_PRELU; }
  // Weight noise (b2g_net_set_weight_noise; wn.p_schedule is never kept): the layer's DropConnect schedule on the device (MAP entries in
  // wn_map).  Its noisy operands, allocated when the layer first gets noise: wn_w = W' (fp32 in FP32 nets; in BF16 nets the bf16 straight
  // copy, and the packed pixel-shuffle copy from element wn_ps on), wn_b = b' (fp32).  wn_live: the latest forward was a train-mode pass that
  // drew, so the pass's GEMMs read the noisy operands; wn_drawn: some train-mode pass has drawn them
  b2g_weight_noise wn{}; bool wn_sched = false; UpdSched* wn_sched_dev = nullptr; void* wn_map = nullptr;
  void* wn_w = nullptr; int64_t wn_ps = -1; float* wn_b = nullptr; bool wn_live = false, wn_drawn = false;
  // a layer whose train-mode passes draw: FrozenLayer never, constant DropConnect(1) is the identity
  bool wn_active() const {
    if (wn.kind == B2G_WEIGHT_NOISE_NONE || d.frozen) return false;
    return wn.kind != B2G_WEIGHT_NOISE_DROPCONNECT || wn_sched || wn.p < 1.f;
  }
};

struct b2g_net {
  b2g_ctx* ctx = nullptr;
  b2g_net_config cfg{};
  std::vector<LayerRT> L;
  int prec = PREC_F32;
  int64_t n_params = 0;
  float *params = nullptr, *grads = nullptr, *st0 = nullptr, *st1 = nullptr;
  float* st2 = nullptr;                // third updater state slot (AMSGrad's v-hat): only nets with an AMSGrad segment have it
  bool upd_ext = false;                // some segment has a kind >= 4: the updater runs its extended instantiations
  __nv_bfloat16* shadow = nullptr; int64_t n_shadow = 0;
  std::vector<UpdSeg> segs; UpdSeg* segs_dev = nullptr; int32_t* chunk_seg_dev = nullptr; int64_t* chunk_off_dev = nullptr; int nchunks = 0;
  // Regularization score: one entry per W and b of every non-frozen GEMM layer, in segment order (reg_seg: the entry's segment), with the
  // fp32 coefficients of its l2 term (0.5 * l2) and l1 term on the host and the device; n_l2 / n_l1: entries with a non-zero coefficient
  std::vector<int> reg_seg; std::vector<float> reg_l2c, reg_l1c;
  int64_t *reg_off_dev = nullptr, *reg_len_dev = nullptr; float *reg_l2c_dev = nullptr, *reg_l1c_dev = nullptr; int n_l2 = 0, n_l1 = 0;
  int* step_dev = nullptr;
  int max_rows = 0;                    // cfg.max_batch
  size_t in_elems = 0;
  void* input = nullptr;               // T NHWC [max_rows][in_elems]
  float* stage_f32 = nullptr; size_t stage_floats = 0;   // host<->device fp32 staging (inputs, outputs, params)
  float* labels_dev = nullptr;         // [max_rows]
  float* mask_dev = nullptr;           // the masked fit's label mask: [max_rows][output size] at most
  float* loss_w = nullptr; bool loss_w_on = false;   // the loss's per-output weights (b2g_net_set_loss_weights): [loss columns]
  void *epsA = nullptr, *epsB = nullptr, *epsC = nullptr; size_t eps_elems = 0;
  float* scratch2 = nullptr;           // split-K / colsum partials of the side stream
  std::vector<cudaEvent_t> ev_fork, ev_done; cudaEvent_t ev_join = nullptr;
  unsigned long long* bn_acc = nullptr; size_t bn_acc_bytes = 0;  // every BatchNorm layer's accumulators, zeroed by one memset per train-mode forward
  unsigned* upd_ticket = nullptr;                                  // block-completion counter of the updater kernel (the last block bumps step_dev)
  unsigned long long* drop_pass = nullptr;                         // dropout pass counter P (device): read by every dropout kernel of a train-mode pass
  unsigned* drop_ticket = nullptr;                                 // block-completion counter of the pass's last dropout kernel (its last block bumps P)
  // Updater settings generation: bumped by every gradient-normalization or learning-rate-schedule change (a captured GAN step holds the
  // launches and kernel instantiations those settings select, so it is re-captured when the generation differs)
  uint64_t settings_gen = 0;
  // L2 gradient normalization (b2g_net_set_gradient_normalization): mode and threshold; norm groups per layer and per segment; the norm
  // kernel's per-chunk partial sums, block-completion counter and per-segment multipliers
  int gn_mode = B2G_GN_NONE; float gn_threshold = 1.0f;
  GnGroup *gn_layer_groups = nullptr, *gn_param_groups = nullptr; int gn_n_layer_groups = 0, gn_n_param_groups = 0;
  double* gn_partial = nullptr; unsigned* gn_ticket = nullptr; float* gn_mult = nullptr;
  // Learning-rate schedules (b2g_net_set_lr_schedule): per layer on the host (MAP entries included), per segment on the device with the
  // MAP entries in sched_map (reallocated when the entries outgrow it); sched_on = some segment has one (selects the scheduled updater);
  // the epoch word EPOCH schedules read; a one-float result slot of b2g_net_get_learning_rate
  struct LayerSched { UpdSched sc{}; std::vector<int32_t> keys; std::vector<double> vals; };
  std::vector<LayerSched> layer_sched; std::vector<int> seg_layer;
  UpdSched* sched_dev = nullptr; bool sched_on = false; void* sched_map = nullptr; size_t sched_map_bytes = 0;
  int64_t* epoch_dev = nullptr; float* lr_out = nullptr;
  // Weight constraints (b2g_net_set_constraints): each constrained tensor's layer, parameter and list; the plan, rebuilt by every set: round r
  // is the r-th constraint of every tensor, its one-pass / element-wise jobs [j0, j1) in one launch and its two-pass jobs [t0, t1) in a norm
  // and a scale launch; the jobs' device table, the two-pass partials and multipliers (cudaMalloc'd per plan) and the norm kernel's ticket
  struct ConTensor { int layer; char param[8]; std::vector<b2g_constraint> list; };
  struct ConRound { int j0, j1, onepass_blocks, t0, t1, norm_blocks, scale_blocks; };
  std::vector<ConTensor> con; std::vector<ConRound> con_rounds;
  ConJob* con_jobs = nullptr; double* con_partial = nullptr; float* con_mult = nullptr; unsigned* con_ticket = nullptr;
  // Weight noise: the job table of every drawing layer's noisy tensors (device, room for two per layer) and its block count; empty: no launch
  WnJob* wn_jobs = nullptr; int wn_njobs = 0, wn_blocks = 0;
  ReduceList pending{};                                           // split-K partial sums queued by this backward pass
  uint64_t simt_gemm_calls = 0;                                    // BF16 nets: GEMM-shaped ops that ran on the SIMT kernels (skinny / unsupported shapes) -- reported, never silent
  float* scratch = nullptr; size_t scratch_floats = 0;
  float* loss_dev = nullptr;           // [8]
  double* loss_partial = nullptr; unsigned* loss_ticket = nullptr;   // k_loss's per-block sums and its ticket
  double* reg_dev = nullptr;          // [2]: the score's L2 and L1 sums
  void* input_grad = nullptr;          // where the last backward left d(loss)/d(input), or null
  int last_rows = 0;
  cudaStream_t fwd_stream = nullptr;   // when set, net_forward launches here instead of ctx->stream
  bool grad_allreduce = true;          // false: parameter-averaging mode (b2g_net_average_parameters)
  bool sync_bn = false;                // cross-replica BatchNorm statistics: the 64-bit statistic accumulators are all-reduced (SURVEY.md 8e)
  bool ar_bf16 = false;                // gradient all-reduce payload in bf16 (half the bytes; default fp32 for parity)
  bool p2p = false; float* p2p_peer_grads[8] = {};      // every rank's gradient vector as mapped into this process (CUDA IPC)
  __nv_bfloat16* ar_buf = nullptr;
  int ar_split_layer = -1; int64_t ar_split_off = 0;   // gradients of layers >= ar_split_layer (= grads[ar_split_off, n_params)) are all-reduced while backward continues
  bool ar_tail_sent = false;
  std::vector<void*> allocs;
};

template <typename P>
static int32_t dalloc(b2g_net* n, P** p, size_t bytes) {
  void* q = nullptr; if (bytes == 0) bytes = 16;
  cudaError_t e = cudaMalloc(&q, bytes);
  if (e != cudaSuccess) return fail(B2G_ERR_OOM, "cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
  n->allocs.push_back(q); *p = (P*)q; return 0;
}

// ------------------------------------------------------------------ host RNG for Xavier init -----------
static inline uint64_t splitmix(uint64_t& s) { uint64_t z = (s += 0x9E3779B97F4A7C15ull); z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull; z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; return z ^ (z >> 31); }
static inline double urand(uint64_t& s) { return ((splitmix(s) >> 11) + 0.5) * (1.0 / 9007199254740992.0); }
static inline float nrand(uint64_t& s) { double u1 = urand(s), u2 = urand(s); return (float)(sqrt(-2.0 * log(u1)) * cos(6.283185307179586 * u2)); }

// ------------------------------------------------------------------ layout helpers (host) ---------------
// DL4J conv W [A][B][taps] ('c' order [nOut,nIn,kH,kW] / deconv [nIn,nOut,kH,kW]) <-> internal [A][taps][B]
static void w_dl4j_to_internal(const float* src, float* dst, int A, int B, int taps) {
  for (int a = 0; a < A; ++a) for (int b = 0; b < B; ++b) for (int t = 0; t < taps; ++t) dst[((size_t)a * taps + t) * B + b] = src[((size_t)a * B + b) * taps + t];
}
static void w_internal_to_dl4j(const float* src, float* dst, int A, int B, int taps) {
  for (int a = 0; a < A; ++a) for (int b = 0; b < B; ++b) for (int t = 0; t < taps; ++t) dst[((size_t)a * B + b) * taps + t] = src[((size_t)a * taps + t) * B + b];
}

// ------------------------------------------------------------------ net construction --------------------
// OUTPUT / LOSS layers: checks the loss code and keeps the activation a loss of codes 2-8 applies (b2g_loss); an OUTPUT layer's GEMM then runs
// without an activation, as for XENT and MCXENT, whose activations are implied.
static int32_t take_loss(LayerRT& l) {
  b2g_layer_desc& d = l.d;
  if (d.loss < B2G_LOSS_XENT || d.loss > B2G_LOSS_WASSERSTEIN) return fail(B2G_ERR_ARG, "layer %s: unknown loss %d", d.name, d.loss);
  if (d.loss >= B2G_LOSS_MSE) {
    if (d.act < B2G_ACT_IDENTITY || d.act > B2G_ACT_THRESHOLDEDRELU) return fail(B2G_ERR_ARG, "layer %s: unknown activation %d", d.name, d.act);
    l.loss_act = d.act; l.loss_alpha = d.act_alpha;      // identity for codes 5-16 (take_act cleared d.act): net_loss applies ext_act
  }
  if (d.type == B2G_LAYER_OUTPUT) d.act = B2G_ACT_IDENTITY;
  return 0;
}
// Layers whose activation is b2g_layer_desc.act: checks the code, and moves a code of 5-16 into ext_act / ext_alpha (d.act becomes identity).
static int32_t take_act(LayerRT& l) {
  b2g_layer_desc& d = l.d;
  const bool lossy = d.type == B2G_LAYER_OUTPUT || d.type == B2G_LAYER_LOSS || d.type == B2G_LAYER_CNN_LOSS;
  const bool has_act = d.type == B2G_LAYER_CONV2D || d.type == B2G_LAYER_DECONV2D || d.type == B2G_LAYER_DENSE || d.type == B2G_LAYER_ACTIVATION ||
                       (lossy && d.loss >= B2G_LOSS_MSE && d.loss <= B2G_LOSS_WASSERSTEIN);
  if (!has_act) return 0;
  if (d.act < B2G_ACT_IDENTITY || d.act > B2G_ACT_THRESHOLDEDRELU) return fail(B2G_ERR_ARG, "layer %s: unknown activation %d", d.name, d.act);
  if (!act_ext_kind(d.act)) return 0;
  if (!std::isfinite(d.act_alpha)) return fail(B2G_ERR_ARG, "layer %s: activation %d needs a finite act_alpha, not %g", d.name, d.act, (double)d.act_alpha);
  l.ext_act = d.act; l.ext_alpha = d.act_alpha; d.act = B2G_ACT_IDENTITY;
  return 0;
}
// SUBSAMPLING / GLOBAL_POOLING: the pooling kind is carried in act, PNORM's p in act_alpha (b2g_pooling)
static int32_t take_pool(LayerRT& l) {
  const b2g_layer_desc& d = l.d;
  const int lo = d.type == B2G_LAYER_SUBSAMPLING ? B2G_POOL_AVG : B2G_POOL_MAX;
  if (d.act < lo || d.act > B2G_POOL_PNORM)
    return fail(B2G_ERR_ARG, "layer %s: pooling kind %d not accepted here (%s)", d.name, d.act, d.type == B2G_LAYER_SUBSAMPLING ? "AVG, SUM or PNORM; MAX is B2G_LAYER_MAXPOOL" : "MAX, AVG, SUM or PNORM");
  l.pool = d.act;
  if (d.act == B2G_POOL_PNORM) {
    const float p = d.act_alpha;
    if (!std::isfinite(p) || p < 1.f || p > 1024.f || p != floorf(p)) return fail(B2G_ERR_ARG, "layer %s: p-norm p = %g is not a whole number >= 1", d.name, (double)p);
    l.pnorm = (int)p;
  }
  return 0;
}
static int32_t net_build(b2g_net* n, const b2g_layer_desc* layers, int32_t nl) {
  const b2g_net_config& c = n->cfg;
  int h = c.in_h, w = c.in_w, ch = c.in_c;
  n->in_elems = (size_t)h * w * ch;
  int64_t off = 0, off_bf = 0;
  for (int i = 0; i < nl; ++i) {
    LayerRT l; l.d = layers[i]; l.d.name[B2G_NAME_LEN - 1] = 0;
    l.ih = h; l.iw = w; l.ic = ch; l.in_elems = (size_t)h * w * ch;
    b2g_layer_desc& d = l.d;
    if (d.has_bias < 0) d.has_bias = 1;
    B2(take_act(l));
    switch (d.type) {
      case B2G_LAYER_CONV2D: {
        if (d.n_in == 0) d.n_in = ch; if (d.n_in != ch) return fail(B2G_ERR_SHAPE, "layer %s: nIn %d != incoming channels %d", d.name, d.n_in, ch);
        if (d.s_h < 1) d.s_h = 1; if (d.s_w < 1) d.s_w = 1;
        l.oh = (h - d.k_h + 2 * d.p_h) / d.s_h + 1; l.ow = (w - d.k_w + 2 * d.p_w) / d.s_w + 1; l.oc = d.n_out;   // ConvolutionMode.Truncate
        if (l.oh < 1 || l.ow < 1) return fail(B2G_ERR_SHAPE, "layer %s: kernel larger than input", d.name);
        l.geom = ConvGeom{0, h, w, ch, l.oh, l.ow, d.n_out, d.k_h, d.k_w, d.s_h, d.s_w, d.p_h, d.p_w};
        // a "valid" conv whose window is the whole input (DCGAN D-last) is a dense layer over the NHWC-flattened input
        if (l.oh == 1 && l.ow == 1 && d.k_h == h && d.k_w == w && d.p_h == 0 && d.p_w == 0) l.geom = ConvGeom{0, 1, 1, h * w * ch, 1, 1, d.n_out, 1, 1, 1, 1, 0, 0};
        l.wA = d.n_out; l.wTaps = d.k_h * d.k_w; l.wB = d.n_in;
        if (d.has_bias) { l.off_b = off; off += d.n_out; }                 // ConvolutionParamInitializer: [b | W]
        l.off_W = off; l.n_W = (int64_t)l.wA * l.wTaps * l.wB; off += l.n_W;
      } break;
      case B2G_LAYER_DECONV2D: {
        if (d.n_in == 0) d.n_in = ch; if (d.n_in != ch) return fail(B2G_ERR_SHAPE, "layer %s: nIn %d != incoming channels %d", d.name, d.n_in, ch);
        if (d.s_h < 1) d.s_h = 1; if (d.s_w < 1) d.s_w = 1;
        l.oh = d.s_h * (h - 1) + d.k_h - 2 * d.p_h; l.ow = d.s_w * (w - 1) + d.k_w - 2 * d.p_w; l.oc = d.n_out;
        // conv-equivalent: conv input = deconv output, conv output = deconv input
        l.geom = ConvGeom{0, l.oh, l.ow, d.n_out, h, w, d.n_in, d.k_h, d.k_w, d.s_h, d.s_w, d.p_h, d.p_w};
        // a transposed conv of a 1x1 map (DCGAN G-first: z -> 4x4) is the 1x1 problem with taps*nOut output channels: out[n][tap][c] = sum_o z[n][o] W[o][tap][c]
        if (h == 1 && w == 1 && d.s_h == 1 && d.s_w == 1 && d.p_h == 0 && d.p_w == 0 && !d.has_bias && d.act == B2G_ACT_IDENTITY)
          l.geom = ConvGeom{0, 1, 1, d.k_h * d.k_w * d.n_out, 1, 1, d.n_in, 1, 1, 1, 1, 0, 0};
        l.wA = d.n_in; l.wTaps = d.k_h * d.k_w; l.wB = d.n_out;
        if (d.has_bias) { l.off_b = off; off += d.n_out; }
        l.off_W = off; l.n_W = (int64_t)l.wA * l.wTaps * l.wB; off += l.n_W;
      } break;
      case B2G_LAYER_DENSE: case B2G_LAYER_OUTPUT: {
        if (h != 1 || w != 1) return fail(B2G_ERR_SHAPE, "layer %s: dense layer needs a feed-forward input (insert CNN_TO_FF)", d.name);
        if (d.n_in == 0) d.n_in = ch; if (d.n_in != ch) return fail(B2G_ERR_SHAPE, "layer %s: nIn %d != incoming features %d", d.name, d.n_in, ch);
        l.oh = l.ow = 1; l.oc = d.n_out;
        l.geom = ConvGeom{0, 1, 1, ch, 1, 1, d.n_out, 1, 1, 1, 1, 0, 0};
        l.wA = d.n_out; l.wTaps = 1; l.wB = d.n_in;                        // 'f'-order [nIn,nOut] == row-major [nOut][nIn]
        l.off_W = off; l.n_W = (int64_t)d.n_in * d.n_out; off += l.n_W;    // DefaultParamInitializer: [W | b]
        if (d.has_bias) { l.off_b = off; off += d.n_out; }
        if (d.type == B2G_LAYER_OUTPUT) {
          B2(take_loss(l));      // the GEMM's epilogue stays identity: the loss applies the activation
          if (d.loss == B2G_LOSS_XENT && d.n_out != 1) return fail(B2G_ERR_UNSUPPORTED, "layer %s: XENT output supports nOut=1 (use MCXENT for nOut>1)", d.name);
        }
      } break;
      case B2G_LAYER_BATCHNORM: {
        d.n_in = d.n_out = ch; l.oh = h; l.ow = w; l.oc = ch;
        if (d.bn_decay <= 0.f) d.bn_decay = 0.9f; if (d.bn_eps <= 0.f) d.bn_eps = 1e-5f;
        l.off_gamma = off; l.off_beta = off + ch; l.off_mean = off + 2 * ch; l.off_var = off + 3 * ch; off += 4 * (int64_t)ch;
      } break;
      case B2G_LAYER_ACTIVATION: l.oh = h; l.ow = w; l.oc = ch; break;
      case B2G_LAYER_MAXPOOL:
        if (d.s_h < 1) d.s_h = 1; if (d.s_w < 1) d.s_w = 1;
        l.oh = (h - d.k_h) / d.s_h + 1; l.ow = (w - d.k_w) / d.s_w + 1; l.oc = ch;
        if (d.k_h * d.k_w > 255) return fail(B2G_ERR_UNSUPPORTED, "layer %s: pooling window too large", d.name);
        break;
      case B2G_LAYER_UPSAMPLE2D: if (d.k_h < 1) d.k_h = 2; l.oh = h * d.k_h; l.ow = w * d.k_h; l.oc = ch; break;
      case B2G_LAYER_SUBSAMPLING:    // SubsamplingLayer AVG / SUM / PNORM, Truncate geometry with zero padding
        B2(take_pool(l));
        if (d.k_h < 1 || d.k_w < 1 || d.s_h < 1 || d.s_w < 1) return fail(B2G_ERR_SHAPE, "layer %s: kernel %dx%d / stride %dx%d below 1", d.name, d.k_h, d.k_w, d.s_h, d.s_w);
        if (d.p_h < 0 || d.p_w < 0 || d.p_h >= d.k_h || d.p_w >= d.k_w) return fail(B2G_ERR_SHAPE, "layer %s: padding %dx%d outside [0, kernel)", d.name, d.p_h, d.p_w);
        l.oh = (h + 2 * d.p_h - d.k_h) / d.s_h + 1; l.ow = (w + 2 * d.p_w - d.k_w) / d.s_w + 1; l.oc = ch;
        if (h + 2 * d.p_h < d.k_h || w + 2 * d.p_w < d.k_w || l.oh < 1 || l.ow < 1) return fail(B2G_ERR_SHAPE, "layer %s: empty pooling output", d.name);
        break;
      case B2G_LAYER_GLOBAL_POOLING: // GlobalPoolingLayer: [H][W][C] -> [1][1][C], the feed-forward layout
        B2(take_pool(l));
        l.oh = l.ow = 1; l.oc = ch; break;
      case B2G_LAYER_LOSS:
        l.oh = h; l.ow = w; l.oc = ch; B2(take_loss(l));
        if (d.loss == B2G_LOSS_MCXENT) return fail(B2G_ERR_UNSUPPORTED, "layer %s: MCXENT is supported on OutputLayer only", d.name);
        if (d.loss == B2G_LOSS_XENT && (size_t)h * w * ch != 1) return fail(B2G_ERR_UNSUPPORTED, "layer %s: XENT loss needs one logit per example", d.name);
        if ((h != 1 || w != 1) && (size_t)h * w * ch != 1) return fail(B2G_ERR_UNSUPPORTED, "layer %s: a loss on a %dx%d map is not supported (feed-forward input or one element per example)", d.name, h, w);
        break;
      case B2G_LAYER_CNN_LOSS:       // CnnLossLayer: the rows are the N*H*W pixels, the columns the C channels (NHWC: the buffer as it is)
        l.oh = h; l.ow = w; l.oc = ch; B2(take_loss(l)); break;
      case B2G_LAYER_FF_TO_CNN:
        if ((size_t)d.pre_h * d.pre_w * d.pre_c != l.in_elems) return fail(B2G_ERR_SHAPE, "layer %s: FeedForwardToCnn(%d,%d,%d) != %zu features", d.name, d.pre_h, d.pre_w, d.pre_c, l.in_elems);
        l.oh = d.pre_h; l.ow = d.pre_w; l.oc = d.pre_c; break;
      case B2G_LAYER_CNN_TO_FF: l.oh = l.ow = 1; l.oc = h * w * ch; break;
      case B2G_LAYER_DROPOUT: {      // DropoutLayer.Builder(IDropout): the b2g_dropout_kind in act, its value (p, rate, stddev) in act_alpha; no parameters
        const float v = d.act_alpha;
        switch (d.act) {
          case B2G_DROPOUT: case B2G_DROPOUT_ALPHA: case B2G_DROPOUT_SPATIAL:
            if (!(v > 0.f && v <= 1.f)) return fail(B2G_ERR_ARG, "layer %s: dropout retain probability %g outside (0, 1]", d.name, (double)v);
            break;
          case B2G_DROPOUT_GAUSSIAN_DROPOUT: if (!(v >= 0.f && v < 1.f)) return fail(B2G_ERR_ARG, "layer %s: GaussianDropout rate %g outside [0, 1)", d.name, (double)v); break;
          case B2G_DROPOUT_GAUSSIAN_NOISE: if (!(v >= 0.f && std::isfinite(v))) return fail(B2G_ERR_ARG, "layer %s: GaussianNoise stddev %g not finite and >= 0", d.name, (double)v); break;
          default: return fail(B2G_ERR_ARG, "layer %s: unknown dropout kind %d", d.name, d.act);
        }
        if (d.act == B2G_DROPOUT_SPATIAL && h == 1 && w == 1) return fail(B2G_ERR_SHAPE, "layer %s: SpatialDropout needs a convolutional [H, W, C] input, not a feed-forward one", d.name);
        l.oh = h; l.ow = w; l.oc = ch;
        if ((uint64_t)c.max_batch * h * w * ch > (1ull << 34))     // checked before anything is allocated
          return fail(B2G_ERR_UNSUPPORTED, "layer %s: a dropout pass of %llu elements exceeds the 2^34 the mask counter addresses", d.name, (unsigned long long)c.max_batch * h * w * ch);
      } break;
      case B2G_LAYER_ELEMENTWISE: case B2G_LAYER_MERGE: {      // the spine (entry i-1) and a skip source j = pre_h, in the order pre_w
        const int j = d.pre_h;
        if (j < 0 || j >= i) return fail(B2G_ERR_ARG, "layer %s: skip source %d outside [0, %d)", d.name, j, i);
        if (d.pre_w != 0 && d.pre_w != 1) return fail(B2G_ERR_ARG, "layer %s: input order %d (0 = spine first, 1 = skip first)", d.name, d.pre_w);
        if (d.type == B2G_LAYER_ELEMENTWISE && (d.act < B2G_EW_OP_ADD || d.act > B2G_EW_OP_MAX)) return fail(B2G_ERR_ARG, "layer %s: unknown element-wise op %d", d.name, d.act);
        const LayerRT& src = n->L[j];
        if (src.d.type == B2G_LAYER_LOSS || src.d.type == B2G_LAYER_CNN_LOSS || src.d.type == B2G_LAYER_OUTPUT)
          return fail(B2G_ERR_UNSUPPORTED, "layer %s: skip source %s is a loss-bearing layer", d.name, src.d.name);
        if (src.oh != h || src.ow != w || (d.type == B2G_LAYER_ELEMENTWISE && src.oc != ch))
          return fail(B2G_ERR_SHAPE, "layer %s: inputs [%d,%d,%d] (spine) and [%d,%d,%d] (%s) do not match", d.name, ch, h, w, src.oc, src.oh, src.ow, src.d.name);
        l.vsrc = j; l.vorder = d.pre_w;
        l.oh = h; l.ow = w; l.oc = d.type == B2G_LAYER_MERGE ? ch + src.oc : ch;
      } break;
      case B2G_LAYER_PRELU: {        // PReLULayer: the shared-axes mask in act, inputShape (0 = not given) in pre_c, pre_h, pre_w
        // a 1x1 map is a feed-forward input [F] (axis 1 only) unless inputShape says [C, 1, 1]
        const bool ff = h == 1 && w == 1 && !(d.pre_h == 1 && d.pre_w == 1);
        if (d.act < 0 || (d.act >> (ff ? 1 : 3)) != 0) return fail(B2G_ERR_ARG, "layer %s: shared axes mask 0x%x outside the input's %d dimension(s)", d.name, d.act, ff ? 1 : 3);
        if ((d.pre_c || d.pre_h || d.pre_w) && (d.pre_c != ch || (ff ? (d.pre_h || d.pre_w) : (d.pre_h != h || d.pre_w != w))))
          return fail(B2G_ERR_SHAPE, "layer %s: inputShape [%d,%d,%d] != the inferred input [%d,%d,%d] (a feed-forward input is [%d])", d.name, d.pre_c, d.pre_h, d.pre_w, ch, h, w, ch);
        l.oh = h; l.ow = w; l.oc = ch;
        l.pg = PreluGeom{h, w, ch, d.act};
        l.wA = 1; l.wTaps = 1; l.n_W = (int64_t)prelu_slopes(l.pg); l.wB = (int)l.n_W;
        l.off_W = off; off += l.n_W;           // "W" in DL4J's [C][H][W] order with the shared axes of extent 1
      } break;
      default: return fail(B2G_ERR_ARG, "layer %d: unknown type %d", i, d.type);
    }
    l.out_elems = (size_t)l.oh * l.ow * l.oc;
    if (l.has_gemm() && n->prec == PREC_BF16) { l.off_W_bf = off_bf; off_bf += l.n_W; off_bf = (off_bf + 63) / 64 * 64;
      if (n->ctx->tc_ok && tc_deconv_ps_shape(l.geom)) { l.off_Wps_bf = off_bf; off_bf += (int64_t)k_tc_deconv_ps_weight_elems(l.geom); off_bf = (off_bf + 63) / 64 * 64; } }
    h = l.oh; w = l.ow; ch = l.oc;
    n->L.push_back(l);
  }
  // skip sources: consumer counts, and the first consumer in backward order (the highest index) of each
  for (int i = (int)n->L.size() - 1; i >= 0; --i) {
    LayerRT& l = n->L[i];
    if (l.vsrc >= 0) { l.vfirst = n->L[l.vsrc].n_skip == 0; ++n->L[l.vsrc].n_skip; }
  }
  // fuse BatchNormalization + ActivationLayer (north_star's BN+ReLU / BN+LeakyReLU); an ActivationLayer of codes 5-16 runs its own kernels.
  // Not where the BatchNorm is a skip source: its vertex reads the BatchNorm's own output and hands it an epsilon w.r.t. that output.
  for (size_t i = 0; i + 1 < n->L.size(); ++i)
    if (n->L[i].d.type == B2G_LAYER_BATCHNORM && !n->L[i].n_skip && n->L[i + 1].d.type == B2G_LAYER_ACTIVATION && !n->L[i + 1].ext_act) {
      n->L[i].fused_act = n->L[i + 1].d.act; n->L[i].fused_alpha = n->L[i + 1].d.act_alpha; n->L[i + 1].act_fused_into_prev = true;
    }
  int last = n->L.back().d.type;
  (void)last;
  n->n_params = off; n->n_shadow = off_bf;
  return 0;
}

static int32_t net_alloc(b2g_net* n) {
  const int R = n->cfg.max_batch; n->max_rows = R;
  const size_t ts = prec_size(n->prec);
  const int G = std::max(1, n->cfg.bn_groups);
  B2(dalloc(n, &n->params, sizeof(float) * n->n_params)); B2(dalloc(n, &n->grads, sizeof(float) * n->n_params));
  B2(dalloc(n, &n->st0, sizeof(float) * n->n_params)); B2(dalloc(n, &n->st1, sizeof(float) * n->n_params));
  if (n->n_shadow) B2(dalloc(n, &n->shadow, sizeof(__nv_bfloat16) * n->n_shadow));
  B2(dalloc(n, &n->upd_ticket, sizeof(unsigned))); CU(cudaMemsetAsync(n->upd_ticket, 0, sizeof(unsigned), n->ctx->stream));
  B2(dalloc(n, &n->drop_pass, sizeof(unsigned long long))); CU(cudaMemsetAsync(n->drop_pass, 0, sizeof(unsigned long long), n->ctx->stream));
  B2(dalloc(n, &n->drop_ticket, sizeof(unsigned))); CU(cudaMemsetAsync(n->drop_ticket, 0, sizeof(unsigned), n->ctx->stream));
  B2(dalloc(n, &n->step_dev, sizeof(int))); B2(dalloc(n, &n->loss_dev, sizeof(float) * 8)); B2(dalloc(n, &n->reg_dev, 2 * sizeof(double)));
  B2(dalloc(n, &n->labels_dev, sizeof(float) * R * std::max<size_t>(1, n->L.back().out_elems)));
  B2(dalloc(n, &n->mask_dev, sizeof(float) * R * std::max<size_t>(1, n->L.back().out_elems)));
  B2(dalloc(n, &n->loss_w, sizeof(float) * std::max<size_t>(1, n->L.back().out_elems)));
  {  // k_loss's per-block sums for one group of max_batch rows (fit) or two of max_batch / 2 (the GAN step's D pass)
    const size_t per = n->L.back().out_elems;
    // CnnLossLayer: every slicing of kernels_cnnloss.cu and loss_kernel stays within LOSS_MAX_GRID = 1024 blocks
    const int cnn = n->L.back().d.type == B2G_LAYER_CNN_LOSS ? 1024 : 0;
    B2(dalloc(n, &n->loss_partial, sizeof(double) * std::max(cnn, std::max(k_loss_blocks((size_t)R * per, 1), 2 * k_loss_blocks((size_t)(R / 2) * per, 2)))));
  }
  B2(dalloc(n, &n->loss_ticket, sizeof(unsigned))); CU(cudaMemsetAsync(n->loss_ticket, 0, sizeof(unsigned), n->ctx->stream));
  B2(dalloc(n, (char**)&n->input, ts * R * n->in_elems));
  size_t max_act = n->in_elems, scratch = 1 << 16, max_w = 0, bn_acc_words = 0;
  for (auto& l : n->L) {
    max_act = std::max(max_act, std::max(l.in_elems, l.out_elems));
    bool alias = l.act_fused_into_prev || l.d.type == B2G_LAYER_LOSS || l.d.type == B2G_LAYER_CNN_LOSS ||
                 (l.d.type == B2G_LAYER_FF_TO_CNN && (l.oc == 1 || l.oh * l.ow == 1)) ||
                 (l.d.type == B2G_LAYER_CNN_TO_FF && (l.ic == 1 || l.ih * l.iw == 1));
    l.out_alias = alias;
    if (!alias) B2(dalloc(n, (char**)&l.out, ts * R * l.out_elems));
    if (l.d.type == B2G_LAYER_DROPOUT) {
      l.drop_buf = l.out;
      const size_t bits = l.d.act == B2G_DROPOUT_SPATIAL ? (size_t)R * l.oc : l.d.act == B2G_DROPOUT || l.d.act == B2G_DROPOUT_ALPHA ? (size_t)R * l.out_elems : 0;
      if (bits) B2(dalloc(n, &l.drop_mask, sizeof(uint32_t) * ((bits + 31) / 32)));
      B2(dalloc(n, &l.drop_rec, sizeof(NoiseRec))); CU(cudaMemsetAsync(l.drop_rec, 0, sizeof(NoiseRec), n->ctx->stream));
      B2(dalloc(n, &l.drop_sched_dev, sizeof(UpdSched))); CU(cudaMemsetAsync(l.drop_sched_dev, 0, sizeof(UpdSched), n->ctx->stream));
    }
    if (l.d.type == B2G_LAYER_OUTPUT || l.d.type == B2G_LAYER_LOSS || l.d.type == B2G_LAYER_CNN_LOSS) B2(dalloc(n, (char**)&l.probs, ts * R * l.out_elems));
    if (l.ext_act && l.has_gemm() && l.d.type != B2G_LAYER_OUTPUT) B2(dalloc(n, (char**)&l.ext_z, ts * R * l.out_elems));
    if (l.d.type == B2G_LAYER_MAXPOOL) B2(dalloc(n, &l.argmax, (size_t)R * l.out_elems));
    if (l.n_skip) B2(dalloc(n, &l.skip_acc, sizeof(float) * R * l.out_elems));
    if (l.d.type == B2G_LAYER_PRELU && !l.d.frozen) B2(dalloc(n, &l.prelu_part, sizeof(float) * k_prelu_part_floats(R, l.pg)));
    if (l.d.type == B2G_LAYER_GLOBAL_POOLING) {
      if (l.pool == B2G_POOL_MAX) B2(dalloc(n, &l.pool_idx, sizeof(int32_t) * R * l.oc));
      const size_t part = k_global_pool_partial_elems(n->prec, R, l.ih * l.iw, l.ic);
      if (part) {
        B2(dalloc(n, &l.pool_part, sizeof(float) * part));
        if (l.pool == B2G_POOL_MAX) B2(dalloc(n, &l.pool_part_idx, sizeof(int32_t) * part));
      }
      B2(dalloc(n, &l.pool_ticket, sizeof(unsigned))); CU(cudaMemsetAsync(l.pool_ticket, 0, sizeof(unsigned), n->ctx->stream));
    }
    if (l.d.type == B2G_LAYER_BATCHNORM) { B2(dalloc(n, &l.bn_fold, sizeof(float) * 2 * l.oc)); B2(dalloc(n, &l.bn_mean, sizeof(float) * G * l.oc)); B2(dalloc(n, &l.bn_invstd, sizeof(float) * G * l.oc)); scratch = std::max(scratch, k_bn_scratch_floats(l.oc, G));
      if (k_bn_vec_ok(n->prec, l.oc)) { B2(dalloc(n, &l.bn_coef, sizeof(float) * 4 * G * l.oc)); bn_acc_words += 2 * k_bn_acc_elems(l.oc, G); } }
    if (l.has_gemm()) {
      ConvGeom g = l.geom; g.N = R;
      scratch = std::max(scratch, std::max(k_simt_wgrad_scratch_floats(g), k_tc_wgrad_scratch_floats(g)));
      scratch = std::max(scratch, std::max(k_edge_wgrad_scratch_floats(g), k_dense_small_o_wgrad_scratch_floats(g)));
      scratch = std::max(scratch, k_tc_edge_wgrad_scratch_floats(g));
      scratch = std::max(scratch, k_colsum_scratch_floats(std::max(l.oc, l.ic)));
      max_w = std::max(max_w, (size_t)l.n_W);
      // split-K partials of the tensor-core weight gradients stay in a per-layer region until the pass's single k_reduce_multi launch
      if (n->prec == PREC_BF16 && n->ctx->tc_ok && !l.d.frozen) {
        l.wg_part_floats = std::max(std::max(k_tc_wgrad_scratch_floats(g), k_tc_edge_wgrad_scratch_floats(g)), k_head_wgrad_scratch_floats(g));
        if (l.wg_part_floats) B2(dalloc(n, &l.wg_part, sizeof(float) * l.wg_part_floats));
      }
    }
  }
  if (bn_acc_words) {
    n->bn_acc_bytes = sizeof(unsigned long long) * bn_acc_words; B2(dalloc(n, &n->bn_acc, n->bn_acc_bytes));
    unsigned long long* q = n->bn_acc;
    for (auto& l : n->L) if (l.bn_coef) { const size_t w = k_bn_acc_elems(l.oc, G); l.acc_fwd = q; l.acc_bwd = q + w; q += 2 * w; }
  }
  n->eps_elems = (size_t)R * max_act;
  B2(dalloc(n, (char**)&n->epsA, ts * n->eps_elems)); B2(dalloc(n, (char**)&n->epsB, ts * n->eps_elems)); B2(dalloc(n, (char**)&n->epsC, ts * n->eps_elems));
  n->scratch_floats = scratch; B2(dalloc(n, &n->scratch, sizeof(float) * scratch)); B2(dalloc(n, &n->scratch2, sizeof(float) * scratch));
  {  // bucket boundary for the overlapped gradient all-reduce: maximise min(share of parameters already final, share of backward work still ahead)
    double tot_p = (double)std::max<int64_t>(1, n->n_params), tot_w = 0; std::vector<double> work(n->L.size(), 0.0);
    for (size_t i = 0; i < n->L.size(); ++i) { const auto& l = n->L[i]; if (l.has_gemm()) work[i] = (double)l.geom.OH * l.geom.OW * l.geom.O * l.geom.KH * l.geom.KW * l.geom.C; tot_w += work[i]; }
    double best = 0.0, ahead = 0.0;
    for (size_t i = 1; i < n->L.size(); ++i) {
      ahead += work[i - 1];
      const auto& l = n->L[i]; int64_t off = -1;
      if (l.has_gemm()) off = l.off_b >= 0 ? std::min(l.off_b, l.off_W) : l.off_W; else if (l.d.type == B2G_LAYER_BATCHNORM) off = l.off_gamma;
      if (off < 0 || tot_w <= 0) continue;
      const double score = std::min((tot_p - (double)off) / tot_p, ahead / tot_w);
      if (score > best) { best = score; n->ar_split_layer = (int)i; n->ar_split_off = off; }
    }
    if (best < 0.1) n->ar_split_layer = -1;
  }
  n->ev_fork.resize(n->L.size()); n->ev_done.resize(n->L.size());
  for (size_t i = 0; i < n->L.size(); ++i) { CU(cudaEventCreateWithFlags(&n->ev_fork[i], cudaEventDisableTiming)); CU(cudaEventCreateWithFlags(&n->ev_done[i], cudaEventDisableTiming)); }
  CU(cudaEventCreateWithFlags(&n->ev_join, cudaEventDisableTiming));
  n->stage_floats = std::max((size_t)R * max_act, std::max((size_t)n->n_params, max_w)); B2(dalloc(n, &n->stage_f32, sizeof(float) * n->stage_floats));
  return 0;
}

// b2g_updater values are the updater kernel's kinds (b2g_net_create has rejected any other value)
static int updater_kind(int u) { return u; }

static int32_t net_init_params_and_updater(b2g_net* n) {
  cudaStream_t s = n->ctx->stream;
  std::vector<float> hp(n->n_params, 0.f), h0(n->n_params, 0.f);
  uint64_t seed = n->cfg.seed ? n->cfg.seed : 666;
  std::vector<int64_t> rego, regl;
  std::vector<int> seg_layer;      // layer index of every segment (the norm groups of the PerLayer modes)
  for (auto& l : n->L) {
    const b2g_layer_desc& d = l.d;
    auto add_seg = [&](int64_t off, int64_t len, bool weight, bool noop) {
      if (d.frozen) return;      // FrozenLayer: no update, no l2 decay, no l2 score (calcL2() == 0)
      UpdSeg sg{}; sg.off = off; sg.len = len; sg.kind = noop ? 3 : updater_kind(d.updater);
      sg.lr = d.lr; sg.b1 = d.beta1; sg.b2 = d.beta2; sg.eps = d.eps; sg.l2 = weight ? d.l2 : 0.f; sg.l1 = 0.f; sg.clip = n->cfg.grad_clip; sg.div_mb = noop ? 0 : 1;
      sg.off_bf = (weight && l.off_W_bf >= 0) ? l.off_W_bf : -1; sg.off_ps = (weight && l.off_Wps_bf >= 0) ? l.off_Wps_bf : -1; sg.ps_O = l.geom.O; sg.ps_C = l.geom.C; n->segs.push_back(sg); seg_layer.push_back((int)(&l - n->L.data()));
      if (!noop && (sg.kind == 1 || sg.kind == 5)) for (int64_t i = 0; i < len; ++i) h0[off + i] = d.eps;     // RmsProp cache / AdaGrad history initialised to epsilon
      if (l.has_reg()) { n->reg_seg.push_back((int)n->segs.size() - 1); rego.push_back(off); regl.push_back(len); n->reg_l2c.push_back(0.5f * sg.l2); n->reg_l1c.push_back(0.f); }
    };
    if (l.has_gemm()) {
      l.reg.l2 = d.l2;
      // WeightInit.XAVIER (J:127): N(0, 2/(fanIn+fanOut)); conv fanIn = nIn*kH*kW, fanOut = nOut*kH*kW/(sH*sW)
      double fi = (double)d.n_in * l.wTaps, fo = (double)d.n_out * l.wTaps / ((d.type == B2G_LAYER_CONV2D || d.type == B2G_LAYER_DECONV2D) ? (double)(d.s_h * d.s_w) : 1.0);
      float sd = (float)sqrt(2.0 / (fi + fo));
      for (int64_t i = 0; i < l.n_W; ++i) hp[l.off_W + i] = sd * nrand(seed);
      if (l.off_b >= 0 && l.off_b < l.off_W) add_seg(l.off_b, d.n_out, false, false);
      add_seg(l.off_W, l.n_W, true, false);
      if (l.off_b >= 0 && l.off_b > l.off_W) add_seg(l.off_b, d.n_out, false, false);
    } else if (d.type == B2G_LAYER_BATCHNORM) {
      for (int c = 0; c < l.oc; ++c) { hp[l.off_gamma + c] = 1.f; hp[l.off_var + c] = 1.f; }
      add_seg(l.off_gamma, l.oc, false, false); add_seg(l.off_beta, l.oc, false, false);
      add_seg(l.off_mean, l.oc, false, true); add_seg(l.off_var, l.oc, false, true);
    } else if (d.type == B2G_LAYER_PRELU) {      // alpha starts at 0 (hp): a new PReLU is a ReLU
      l.reg.l2 = d.l2;
      add_seg(l.off_W, l.n_W, true, false);
    }
  }
  CU(cudaMemcpyAsync(n->params, hp.data(), sizeof(float) * n->n_params, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(n->st0, h0.data(), sizeof(float) * n->n_params, cudaMemcpyHostToDevice, s));
  CU(cudaMemsetAsync(n->st1, 0, sizeof(float) * n->n_params, s)); CU(cudaMemsetAsync(n->grads, 0, sizeof(float) * n->n_params, s));
  bool amsgrad = false;
  for (const UpdSeg& sg : n->segs) { n->upd_ext = n->upd_ext || sg.kind >= 4; amsgrad = amsgrad || sg.kind == 8; }
  if (amsgrad) { B2(dalloc(n, &n->st2, sizeof(float) * n->n_params)); CU(cudaMemsetAsync(n->st2, 0, sizeof(float) * n->n_params, s)); }
  CU(cudaMemsetAsync(n->step_dev, 0, sizeof(int), s));
  std::vector<int32_t> cs; std::vector<int64_t> co;
  for (size_t i = 0; i < n->segs.size(); ++i) for (int64_t o = n->segs[i].off; o < n->segs[i].off + n->segs[i].len; o += UPD_CHUNK) { cs.push_back((int32_t)i); co.push_back(o); }
  n->nchunks = (int)cs.size();
  B2(dalloc(n, &n->segs_dev, sizeof(UpdSeg) * std::max<size_t>(1, n->segs.size()))); B2(dalloc(n, &n->chunk_seg_dev, sizeof(int32_t) * std::max(1, n->nchunks))); B2(dalloc(n, &n->chunk_off_dev, sizeof(int64_t) * std::max(1, n->nchunks)));
  CU(cudaMemcpyAsync(n->segs_dev, n->segs.data(), sizeof(UpdSeg) * n->segs.size(), cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(n->chunk_seg_dev, cs.data(), sizeof(int32_t) * cs.size(), cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(n->chunk_off_dev, co.data(), sizeof(int64_t) * co.size(), cudaMemcpyHostToDevice, s));
  {  // L2 gradient normalization: norm groups over the chunk map (chunks follow segment order, segments follow layer order), partial sums, multipliers
    const int ns = (int)n->segs.size();
    std::vector<int32_t> seg_c0(ns + 1, n->nchunks);
    for (int c = n->nchunks - 1; c >= 0; --c) seg_c0[cs[c]] = c;
    std::vector<GnGroup> per_layer, per_param;
    for (int i = 0; i < ns; ++i) {
      per_param.push_back(GnGroup{seg_c0[i], seg_c0[i + 1], i, i + 1});
      if (i > 0 && seg_layer[i] == seg_layer[i - 1]) { per_layer.back().chunk_end = seg_c0[i + 1]; per_layer.back().seg_end = i + 1; }
      else per_layer.push_back(GnGroup{seg_c0[i], seg_c0[i + 1], i, i + 1});
    }
    n->gn_n_layer_groups = (int)per_layer.size(); n->gn_n_param_groups = (int)per_param.size();
    B2(dalloc(n, &n->gn_layer_groups, sizeof(GnGroup) * std::max<size_t>(1, per_layer.size()))); B2(dalloc(n, &n->gn_param_groups, sizeof(GnGroup) * std::max<size_t>(1, per_param.size())));
    B2(dalloc(n, &n->gn_partial, sizeof(double) * std::max(1, n->nchunks))); B2(dalloc(n, &n->gn_mult, sizeof(float) * std::max(1, ns)));
    B2(dalloc(n, &n->gn_ticket, sizeof(unsigned))); CU(cudaMemsetAsync(n->gn_ticket, 0, sizeof(unsigned), s));
    CU(cudaMemcpyAsync(n->gn_layer_groups, per_layer.data(), sizeof(GnGroup) * per_layer.size(), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(n->gn_param_groups, per_param.data(), sizeof(GnGroup) * per_param.size(), cudaMemcpyHostToDevice, s));
  }
  {  // learning-rate schedules: none yet (every segment kind 0), epoch 0
    n->seg_layer = seg_layer; n->layer_sched.assign(n->L.size(), b2g_net::LayerSched{});
    B2(dalloc(n, &n->sched_dev, sizeof(UpdSched) * std::max<size_t>(1, n->segs.size()))); CU(cudaMemsetAsync(n->sched_dev, 0, sizeof(UpdSched) * std::max<size_t>(1, n->segs.size()), s));
    B2(dalloc(n, &n->epoch_dev, sizeof(int64_t))); CU(cudaMemsetAsync(n->epoch_dev, 0, sizeof(int64_t), s));
    B2(dalloc(n, &n->lr_out, sizeof(float)));
  }
  {  // regularization score table: every W and b of a non-frozen GEMM layer, so that b2g_net_set_regularization only rewrites coefficients
    const size_t nr = std::max<size_t>(1, rego.size());
    B2(dalloc(n, &n->reg_off_dev, sizeof(int64_t) * nr)); B2(dalloc(n, &n->reg_len_dev, sizeof(int64_t) * nr));
    B2(dalloc(n, &n->reg_l2c_dev, sizeof(float) * nr)); B2(dalloc(n, &n->reg_l1c_dev, sizeof(float) * nr));
    if (!rego.empty()) {
      CU(cudaMemcpyAsync(n->reg_off_dev, rego.data(), sizeof(int64_t) * rego.size(), cudaMemcpyHostToDevice, s));
      CU(cudaMemcpyAsync(n->reg_len_dev, regl.data(), sizeof(int64_t) * regl.size(), cudaMemcpyHostToDevice, s));
      CU(cudaMemcpyAsync(n->reg_l2c_dev, n->reg_l2c.data(), sizeof(float) * rego.size(), cudaMemcpyHostToDevice, s));
      CU(cudaMemcpyAsync(n->reg_l1c_dev, n->reg_l1c.data(), sizeof(float) * rego.size(), cudaMemcpyHostToDevice, s));
    }
    n->n_l2 = (int)std::count_if(n->reg_l2c.begin(), n->reg_l2c.end(), [](float c) { return c != 0.f; }); n->n_l1 = 0;
  }
  CU(cudaStreamSynchronize(s));
  return 0;
}

// bf16 operand copy of every GEMM weight (plus the packed pixel-shuffle operand of the <= 4-channel transposed conv); no-op in FP32 mode.
// Only setParam / setParams / parameter averaging need it: after an updater pass both were written by the updater kernel itself.
static void net_refresh_shadow(b2g_net* n, int only_layer = -1) {
  if (n->prec != PREC_BF16) return;
  cudaStream_t st = n->ctx->stream;
  for (size_t i = 0; i < n->L.size(); ++i) { auto& l = n->L[i];
    if (!l.has_gemm() || (only_layer >= 0 && (int)i != only_layer)) continue;
    if (l.off_Wps_bf >= 0) k_pack_deconv_ps(n->params + l.off_W, n->shadow + l.off_Wps_bf, l.geom.O, l.geom.C, st);
    k_cast_f32_to_bf16(n->params + l.off_W, n->shadow + l.off_W_bf, (size_t)l.n_W, st);
  }
}

// ------------------------------------------------------------------ forward / backward -------------------
// sched_step / sched_epoch: the counters scheduled DropoutLayers read (null: the net's own)
struct FwdOpts { int rows; int groups; bool train; bool update_running; void* out_override; const int* sched_step = nullptr; const int64_t* sched_epoch = nullptr; };

// The weight operand of every GEMM route: the noisy W' while the layer's latest forward drew one (b2g_weight_noise), else the clean weights
static const void* w_ptr(const b2g_net* n, const LayerRT& l, int* wprec) {
  if (n->prec == PREC_BF16) { *wprec = PREC_BF16; return l.wn_live ? l.wn_w : n->shadow + l.off_W_bf; }
  *wprec = PREC_F32; return l.wn_live ? l.wn_w : n->params + l.off_W;
}

static inline bool tc_on(const b2g_net* n) { return n->prec == PREC_BF16 && n->ctx->tc_ok; }
static inline cudaStream_t fstream(const b2g_net* n) { return n->fwd_stream ? n->fwd_stream : n->ctx->stream; }
// A BF16 net whose GEMM-shaped op has no tensor-core kernel runs it on the SIMT kernels: counted (b2g_net_simt_gemm_calls, bench.py prints
// it per step) so that a shape falling off the tensor-core path is visible, never silent.  The by-design skinny layers (<= 4 units on one
// side, K = 100 G-first) are counted too.
static inline void note_simt(b2g_net* n) { if (n->prec == PREC_BF16) ++n->simt_gemm_calls; }

// sync_bn: the number of replicas whose statistics are pooled (1 = local statistics, what Spark workers do in the reference)
static inline int sync_bn_world(const b2g_net* n) { return (n->sync_bn && n->ctx->comm && n->ctx->world > 1) ? n->ctx->world : 1; }
// `scale` (inference-mode BatchNorm folded into the epilogue) must be honoured; `fuse` (EPI_STATS / EPI_BNBWD / EPI_ACTBWD) is opportunistic:
// *fused tells the caller whether the kernel that ran did it -- if not, the unfused elementwise kernels follow.
static int32_t gemm_fprop(b2g_net* n, const LayerRT& l, const ConvGeom& g, const void* x, const float* bias, void* out, int act, float alpha,
                          const float* scale = nullptr, const TcEpi* fuse = nullptr, bool* fused = nullptr) {
  cudaStream_t s = fstream(n); int wp; const void* w = w_ptr(n, l, &wp);
  if (fused) *fused = false;
  if (scale) {       // folded epilogue: tensor-core or SIMT GEMM kernels only
    if (tc_on(n) && tc_fprop_supported(g)) { TcEpi e{}; e.mode = EPI_PLAIN; e.scale = scale; return k_tc_fprop(g, (const __nv_bfloat16*)x, (const __nv_bfloat16*)w, bias, (__nv_bfloat16*)out, act, alpha, s, &e) == 0 ? 0 : fail(B2G_ERR_CUDA, "tensor-core fprop launch failed"); }
    note_simt(n); k_simt_fprop(n->prec, wp, g, x, w, bias, out, act, alpha, s, scale); return 0;
  }
  if (tc_on(n) && tc_edge_conv_supported(g) && k_tc_edge_conv(g, (const __nv_bfloat16*)x, (const __nv_bfloat16*)w, bias, (__nv_bfloat16*)out, act, alpha, s) == 0) return 0;
  if (edge_conv_small_cin_supported(g)) { note_simt(n); k_edge_conv_small_cin(n->prec, wp, g, x, w, bias, out, act, alpha, s); return 0; }
  if (dense_small_o_supported(g)) { note_simt(n); k_dense_small_o_fwd(n->prec, wp, g, x, w, bias, out, act, alpha, s); return 0; }
  if (tc_on(n) && tc_fprop_supported(g)) {
    if (fuse && k_tc_fprop(g, (const __nv_bfloat16*)x, (const __nv_bfloat16*)w, bias, (__nv_bfloat16*)out, act, alpha, s, fuse) == 0) { if (fused) *fused = true; return 0; }
    if (k_tc_fprop(g, (const __nv_bfloat16*)x, (const __nv_bfloat16*)w, bias, (__nv_bfloat16*)out, act, alpha, s) == 0) return 0;
    return fail(B2G_ERR_CUDA, "tensor-core fprop launch failed");
  }
  if (n->prec == PREC_BF16 && head_conv_supported(g)) { k_head_fwd(g, (const __nv_bfloat16*)x, (const __nv_bfloat16*)w, bias, (__nv_bfloat16*)out, act, alpha, s); return 0; }
  note_simt(n); k_simt_fprop(n->prec, wp, g, x, w, bias, out, act, alpha, s); return 0;
}
static int32_t gemm_dgrad(b2g_net* n, const LayerRT& l, const ConvGeom& g, const void* dy, const float* bias, void* dx, int act, float alpha,
                          const float* scale = nullptr, const TcEpi* fuse = nullptr, bool* fused = nullptr) {
  cudaStream_t s = fstream(n); int wp; const void* w = w_ptr(n, l, &wp);
  if (fused) *fused = false;
  if (scale) {
    if (tc_on(n) && tc_dgrad_supported(g) && !edge_deconv_small_c_supported(g)) { TcEpi e{}; e.mode = EPI_PLAIN; e.scale = scale; return k_tc_dgrad(g, (const __nv_bfloat16*)dy, (const __nv_bfloat16*)w, bias, (__nv_bfloat16*)dx, act, alpha, s, &e) == 0 ? 0 : fail(B2G_ERR_CUDA, "tensor-core dgrad launch failed"); }
    note_simt(n); k_simt_dgrad(n->prec, wp, g, dy, w, bias, dx, act, alpha, s, scale); return 0;
  }
  if (tc_on(n) && l.off_Wps_bf >= 0 && tc_deconv_ps_supported(g)) {
    const TcEpi* f = (fuse && fuse->mode == EPI_ACTBWD) ? fuse : nullptr;
    const __nv_bfloat16* wps = l.wn_live ? (const __nv_bfloat16*)l.wn_w + l.wn_ps : n->shadow + l.off_Wps_bf;
    if (k_tc_deconv_ps(g, (const __nv_bfloat16*)dy, wps, bias, (__nv_bfloat16*)dx, act, alpha, s, f) == 0) { if (fused) *fused = f != nullptr; return 0; }
    return fail(B2G_ERR_CUDA, "tensor-core pixel-shuffle deconv launch failed");
  }
  if (edge_deconv_small_c_supported(g)) { note_simt(n); k_edge_deconv_small_c(n->prec, wp, g, dy, w, bias, dx, act, alpha, s); return 0; }
  if (dense_small_o_supported(g) && !bias && act == ACT_IDENTITY) { note_simt(n); k_dense_small_o_dgrad(n->prec, wp, g, dy, w, dx, s); return 0; }
  if (dense_small_k_supported(g) && !(tc_on(n) && g.O % 64 == 0)) { note_simt(n); k_dense_small_k_dgrad(n->prec, wp, g, dy, w, bias, dx, act, alpha, s); return 0; }
  if (tc_on(n) && g.KH == 1 && g.KW == 1 && g.H == 1 && g.W == 1) {
    // dense layer: dx = dy . W is the fprop kernel reading the layer's own [nOut][nIn] weight as an MN-major operand (reduction over nOut)
    ConvGeom t = g; t.C = g.O; t.O = g.C;
    if (tc_fprop_supported(t)) {
      if (fuse && k_tc_fprop(t, (const __nv_bfloat16*)dy, (const __nv_bfloat16*)w, bias, (__nv_bfloat16*)dx, act, alpha, s, fuse, 1) == 0) { if (fused) *fused = true; return 0; }
      if (k_tc_fprop(t, (const __nv_bfloat16*)dy, (const __nv_bfloat16*)w, bias, (__nv_bfloat16*)dx, act, alpha, s, nullptr, 1) == 0) return 0;
      return fail(B2G_ERR_CUDA, "tensor-core dense dgrad launch failed");
    }
  }
  if (tc_on(n) && tc_dgrad_supported(g)) {
    if (fuse && k_tc_dgrad(g, (const __nv_bfloat16*)dy, (const __nv_bfloat16*)w, bias, (__nv_bfloat16*)dx, act, alpha, s, fuse) == 0) { if (fused) *fused = true; return 0; }
    if (k_tc_dgrad(g, (const __nv_bfloat16*)dy, (const __nv_bfloat16*)w, bias, (__nv_bfloat16*)dx, act, alpha, s) == 0) return 0;
    return fail(B2G_ERR_CUDA, "tensor-core dgrad launch failed");
  }
  if (n->prec == PREC_BF16 && head_conv_supported(g)) { k_head_dgrad(g, (const __nv_bfloat16*)dy, (const __nv_bfloat16*)w, bias, (__nv_bfloat16*)dx, act, alpha, s); return 0; }
  note_simt(n); k_simt_dgrad(n->prec, wp, g, dy, w, bias, dx, act, alpha, s); return 0;
}
static int32_t gemm_wgrad(b2g_net* n, LayerRT& l, const ConvGeom& g, const void* x, const void* dy, float* dw, cudaStream_t s, float* scratch, float* db = nullptr, bool* bias_done = nullptr) {
  if (tc_on(n) && tc_edge_wgrad_supported(g) && l.wg_part) { const int r = k_tc_edge_wgrad(g, (const __nv_bfloat16*)x, (const __nv_bfloat16*)dy, dw, db, l.wg_part, l.wg_part_floats, 0, s, &n->pending); if (r >= 0) { if (bias_done) *bias_done = r == 1; return 0; } }
  if (edge_wgrad_small_cin_supported(g)) { note_simt(n); k_edge_wgrad_small_cin(n->prec, g, x, dy, dw, scratch, 0, s); return 0; }
  if (dense_small_o_supported(g)) { note_simt(n); k_dense_small_o_wgrad(n->prec, g, x, dy, dw, scratch, 0, s); return 0; }
  if (dense_small_k_supported(g) && !(tc_on(n) && tc_wgrad_supported(g))) { note_simt(n); k_dense_small_k_wgrad(n->prec, g, x, dy, dw, s); return 0; }
  if (tc_on(n) && tc_wgrad_supported(g) && l.wg_part) {
    if (k_tc_wgrad(g, (const __nv_bfloat16*)x, (const __nv_bfloat16*)dy, dw, l.wg_part, l.wg_part_floats, 0, s, &n->pending) == 0) return 0;
    return fail(B2G_ERR_CUDA, "tensor-core wgrad launch failed");
  }
  if (n->prec == PREC_BF16 && head_conv_supported(g) && l.wg_part) {
    if (k_head_wgrad(g, (const __nv_bfloat16*)x, (const __nv_bfloat16*)dy, dw, l.wg_part, l.wg_part_floats, 0, s, &n->pending) == 0) return 0;
    return fail(B2G_ERR_CUDA, "few-output conv weight gradient: partials larger than the layer's region");
  }
  note_simt(n); k_simt_wgrad(n->prec, g, x, dy, dw, scratch, n->scratch_floats, 0, s); return 0;
}

// The mask inputs of a DropoutLayer (include/b200gan.h): key = the net's seed (0 -> 666, as for Xavier init), counter word 3 = chain index |
// rank << 16.  The rank is fixed per context, so a captured graph may hold it; P is read by the kernel.
static DropoutArgs make_dropout_args(uint64_t seed, int layer, int rank, float p) {
  DropoutArgs a{}; a.seed = seed ? seed : 666; a.tag = (uint32_t)layer | ((uint32_t)rank << 16);
  a.keep_all = p >= 1.f ? 1 : 0; a.threshold = a.keep_all ? 0u : (uint32_t)floor((double)p * 4294967296.0); a.scale = 1.0f / p;
  return a;
}
static DropoutArgs dropout_args(const b2g_net* n, int layer) { return make_dropout_args(n->cfg.seed, layer, n->ctx->rank, n->L[layer].d.act_alpha); }
// The same inputs for the other kinds, with the kernels' constants derived from the value v (b2g_dropout_kind): sigma, AlphaDropout's a, b
// and a', SpatialDropout's 1/p, and the Bernoulli threshold.  hw, C: the layer's map.
static NoiseArgs make_noise_args(uint64_t seed, int layer, int rank, int kind, float v, int hw, int C) {
  NoiseArgs a{}; a.seed = seed ? seed : 666; a.tag = (uint32_t)layer | ((uint32_t)rank << 16); a.hw = hw; a.C = C; a.value = v;
  noise_derive(kind, v, a);
  return a;
}
static NoiseArgs noise_args(const b2g_net* n, int layer) {
  const LayerRT& l = n->L[layer];
  return make_noise_args(n->cfg.seed, layer, n->ctx->rank, l.d.act, l.d.act_alpha, l.oh * l.ow, l.oc);
}
// The schedule inputs of a layer's kernels: its schedule (null when it has none) at the counters of the pass (the net's own, or in the GAN
// step's generator pass the generator's)
static NoiseSched noise_sched(const b2g_net* n, const LayerRT& l, const int* step, const int64_t* epoch) {
  return NoiseSched{l.drop_sched ? l.drop_sched_dev : nullptr, step ? step : n->step_dev, epoch ? epoch : n->epoch_dev};
}

// Runs layers [0, L) on `in` (T NHWC, rows examples). Returns pointer to the final activations.
static int32_t net_forward(b2g_net* n, const void* in, const FwdOpts& o, const void** result) {
  cudaStream_t s = fstream(n);
  if (o.rows > n->max_rows || o.rows < 1) return fail(B2G_ERR_SHAPE, "batch %d outside [1, max_batch=%d]", o.rows, n->max_rows);
  if (o.groups < 1 || o.rows % o.groups) return fail(B2G_ERR_SHAPE, "batch %d not divisible into %d groups", o.rows, o.groups);
  const int R = o.rows; const void* cur = in;
  n->last_rows = R;
  // every BatchNorm accumulator of the pass (forward statistics and the backward reductions that follow) starts from zero: one memset node
  if (o.train && n->bn_acc) CU(cudaMemsetAsync(n->bn_acc, 0, n->bn_acc_bytes, s));
  // every stochastic DropoutLayer of a train-mode pass draws with the same pass counter P; the last one's kernel advances P on the device
  int last_drop = -1;
  if (o.train) for (size_t i = 0; i < n->L.size(); ++i) if (n->L[i].drop_active()) last_drop = (int)i;
  // weight noise: one launch at the top of a train-mode pass draws every noisy tensor with the same P; it advances P itself only when no
  // DropoutLayer of the pass will
  for (auto& l : n->L) l.wn_live = o.train && l.wn_active();
  if (o.train && n->wn_njobs) {
    k_weight_noise(n->wn_jobs, n->wn_njobs, n->wn_blocks, n->cfg.seed ? n->cfg.seed : 666, n->ctx->rank, o.sched_step ? o.sched_step : n->step_dev,
                   o.sched_epoch ? o.sched_epoch : n->epoch_dev, n->drop_pass, n->drop_ticket, last_drop < 0 ? 1 : 0, s);
    for (auto& l : n->L) l.wn_drawn = l.wn_drawn || l.wn_live;
  }
  for (size_t i = 0; i < n->L.size(); ++i) {
    LayerRT& l = n->L[i]; const b2g_layer_desc& d = l.d;
    void* out = l.out;
    if (i + 1 == n->L.size() && o.out_override && !l.out_alias) out = o.out_override;
    const float* bias = l.off_b >= 0 ? (l.wn_live && l.wn.apply_to_bias ? l.wn_b : n->params + l.off_b) : nullptr;
    const bool gemm_then_bn = (d.type == B2G_LAYER_CONV2D || d.type == B2G_LAYER_DECONV2D || d.type == B2G_LAYER_DENSE) && i + 1 < n->L.size() && n->L[i + 1].d.type == B2G_LAYER_BATCHNORM;
    // a 1x1-input deconv is computed as the 1x1 problem with taps*C output channels: its columns are not the BatchNorm's channels
    const bool remapped = d.type == B2G_LAYER_DECONV2D && l.geom.KH == 1 && l.geom.C != l.oc;
    // inference-mode (or frozen) BatchNorm right after a linear conv / deconv / dense: fold it, and its activation, into that GEMM's epilogue
    // (not when the GEMM is a skip source: the fold never writes the GEMM's own output, which its vertex reads)
    if (gemm_then_bn && d.act == B2G_ACT_IDENTITY && !l.ext_act && (!o.train || n->L[i + 1].d.frozen) && !(i + 2 == n->L.size() && o.out_override) && !remapped &&
        !l.n_skip) {
      LayerRT& bn = n->L[i + 1];
      ConvGeom g = l.geom; g.N = R;
      k_bn_fold(n->params + bn.off_mean, n->params + bn.off_var, n->params + bn.off_gamma, n->params + bn.off_beta, bias, bn.oc, bn.d.bn_eps, bn.bn_fold, bn.bn_fold + bn.oc, s);
      if (d.type == B2G_LAYER_DECONV2D) B2(gemm_dgrad(n, l, g, cur, bn.bn_fold + bn.oc, bn.out, bn.fused_act, bn.fused_alpha, bn.bn_fold));
      else B2(gemm_fprop(n, l, g, cur, bn.bn_fold + bn.oc, bn.out, bn.fused_act, bn.fused_alpha, bn.bn_fold));
      cur = bn.out; ++i; continue;
    }
    // train-mode BatchNorm right after a GEMM: its batch statistics come out of the GEMM's epilogue (kernels_tc.cu EPI_STATS)
    TcEpi st{}; const TcEpi* fuse = nullptr; bool fused = false;
    // (not after an activation of codes 5-16: the BatchNorm's input is then a = f(z), not the GEMM's z)
    if (gemm_then_bn && o.train && !n->L[i + 1].d.frozen && n->L[i + 1].bn_coef && !remapped && tc_on(n) && !l.ext_act) {
      st.mode = EPI_STATS; st.acc = n->L[i + 1].acc_fwd; st.imgs_per_group = R / o.groups; fuse = &st;
    }
    // a GEMM layer with an activation of codes 5-16: the GEMM (identity epilogue) writes z into ext_z, then a = f(z)
    void* gout = l.ext_z ? l.ext_z : out;
    switch (d.type) {
      case B2G_LAYER_CONV2D: case B2G_LAYER_DENSE: case B2G_LAYER_OUTPUT: { ConvGeom g = l.geom; g.N = R; B2(gemm_fprop(n, l, g, cur, bias, gout, d.act, d.act_alpha, nullptr, fuse, &fused)); } break;
      case B2G_LAYER_DECONV2D: { ConvGeom g = l.geom; g.N = R; B2(gemm_dgrad(n, l, g, cur, bias, gout, d.act, d.act_alpha, nullptr, fuse, &fused)); } break;
      case B2G_LAYER_BATCHNORM: {
        int rows_pg = (R / o.groups) * l.oh * l.ow;
        const bool bn_train = o.train && !d.frozen;      // FrozenLayer always activates in test mode
        l.fwd_fused = false;
        if (bn_train && l.bn_coef) {
          if (!l.stats_by_producer) k_bn_stats_acc(cur, rows_pg, l.oc, o.groups, l.acc_fwd, s);
          const int reps = sync_bn_world(n);
          if (reps > 1) NC(g_nccl.ar(l.acc_fwd, l.acc_fwd, k_bn_acc_elems(l.oc, o.groups), /*ncclUint64*/ 5, /*ncclSum*/ 0, n->ctx->comm, s));      // integer sums: bit-identical on every rank
          k_bn_apply_acc(cur, out, rows_pg, l.oc, o.groups, l.acc_fwd, n->params + l.off_gamma, n->params + l.off_beta, l.fused_act, l.fused_alpha, d.bn_eps, l.bn_coef,
                         n->params + l.off_mean, n->params + l.off_var, o.update_running ? n->grads + l.off_mean : nullptr, o.update_running ? n->grads + l.off_var : nullptr, d.bn_decay, s, reps);
          l.fwd_fused = true; l.stats_by_producer = false; l.fwd_groups = o.groups;
          break;
        }
        if (bn_train) k_bn_stats(n->prec, cur, rows_pg, l.oc, o.groups, n->scratch, l.bn_mean, l.bn_invstd, d.bn_eps, n->params + l.off_mean, n->params + l.off_var,
                                o.update_running ? n->grads + l.off_mean : nullptr, o.update_running ? n->grads + l.off_var : nullptr, d.bn_decay, s);
        else k_bn_prep_infer(n->params + l.off_mean, n->params + l.off_var, l.oc, o.groups, d.bn_eps, l.bn_mean, l.bn_invstd, s);
        k_bn_apply(n->prec, cur, out, rows_pg, l.oc, o.groups, l.bn_mean, l.bn_invstd, n->params + l.off_gamma, n->params + l.off_beta, l.fused_act, l.fused_alpha, s);
      } break;
      case B2G_LAYER_ACTIVATION:
        if (l.act_fused_into_prev) out = (void*)cur;
        else if (l.ext_act) k_act_ext_fwd(n->prec, l.ext_act, l.ext_alpha, cur, out, (size_t)R * l.out_elems, s);
        else k_act_fwd(n->prec, cur, out, (size_t)R * l.out_elems, d.act, d.act_alpha, s);
        break;
      case B2G_LAYER_MAXPOOL: k_maxpool_fwd(n->prec, cur, out, l.argmax, R, l.ih, l.iw, l.ic, l.oh, l.ow, d.k_h, d.k_w, d.s_h, d.s_w, s); break;
      case B2G_LAYER_SUBSAMPLING: k_pool2d_fwd(n->prec, l.pool, l.pnorm, cur, out, R, l.ih, l.iw, l.ic, l.oh, l.ow, d.k_h, d.k_w, d.s_h, d.s_w, d.p_h, d.p_w, s); break;
      case B2G_LAYER_GLOBAL_POOLING: k_global_pool_fwd(n->prec, l.pool, l.pnorm, cur, out, l.pool_idx, R, l.ih * l.iw, l.ic, l.pool_part, l.pool_part_idx, l.pool_ticket, s); break;
      case B2G_LAYER_UPSAMPLE2D: k_upsample_fwd(n->prec, cur, out, R, l.ih, l.iw, l.ic, d.k_h, s); break;
      case B2G_LAYER_LOSS: case B2G_LAYER_CNN_LOSS: out = (void*)cur; break;
      case B2G_LAYER_FF_TO_CNN: if (l.out_alias) out = (void*)cur; else k_permute(n->prec, cur, out, R, l.oc, l.oh * l.ow, 1, s); break;
      case B2G_LAYER_CNN_TO_FF: if (l.out_alias) out = (void*)cur; else k_permute(n->prec, cur, out, R, l.ic, l.ih * l.iw, 0, s); break;
      case B2G_LAYER_DROPOUT:
        l.drop_live = o.train && l.drop_active();
        if (l.drop_live) {
          if (d.act == B2G_DROPOUT && !l.drop_sched) k_dropout_fwd(n->prec, cur, l.drop_buf, l.drop_mask, (size_t)R * l.out_elems, dropout_args(n, (int)i), n->drop_pass, n->drop_ticket, (int)i == last_drop, s);
          else k_noise_fwd(n->prec, d.act, cur, l.drop_buf, l.drop_mask, l.drop_rec, (size_t)R * l.out_elems, noise_args(n, (int)i),
                           noise_sched(n, l, o.sched_step, o.sched_epoch), n->drop_pass, n->drop_ticket, (int)i == last_drop, s);
          out = l.drop_buf;
        } else out = (void*)cur;       // inference, FrozenLayer, p = 1, rate = 0 or stddev = 0: the identity, no launch
        l.out = out;
        break;
      case B2G_LAYER_ELEMENTWISE: {
        const void* sk = n->L[l.vsrc].out;
        k_vertex_ew_fwd(n->prec, d.act, l.vorder ? sk : cur, l.vorder ? cur : sk, out, (size_t)R * l.out_elems, s);
      } break;
      case B2G_LAYER_MERGE: {
        const LayerRT& src = n->L[l.vsrc]; const size_t px = (size_t)R * l.oh * l.ow;
        if (l.vorder) k_merge_fwd(n->prec, src.out, cur, out, px, src.oc, l.ic, s);
        else k_merge_fwd(n->prec, cur, src.out, out, px, l.ic, src.oc, s);
      } break;
      case B2G_LAYER_PRELU: k_prelu_fwd(n->prec, cur, out, n->params + l.off_W, R, l.pg, s); break;     // the same function in both modes
    }
    if (l.ext_z) k_act_ext_fwd(n->prec, l.ext_act, l.ext_alpha, l.ext_z, out, (size_t)R * l.out_elems, s);
    if (fuse) n->L[i + 1].stats_by_producer = fused;
    if (l.out_alias) l.out = out;
    cur = out;
  }
  CHECK_KERNELS();
  if (result) *result = cur;
  return 0;
}

// B2G_AR_OVERLAP=1: two-bucket gradient all-reduce, the tail bucket (layers whose gradients are final first) travels on a comm stream while
// backward continues.
static bool ar_overlap_on(const b2g_net* n) {
  static int on = -1; if (on < 0) { const char* e = getenv("B2G_AR_OVERLAP"); on = (e && e[0] == '1') ? 1 : 0; }
  return on && n->ctx->comm && n->ctx->world > 1 && n->grad_allreduce && n->ar_split_layer > 0 && !n->sync_bn;
}
static void flush_pending_reduce(b2g_net* n, cudaStream_t s2) { if (n->pending.count) { k_reduce_multi(n->pending, s2); n->pending.count = 0; } }

// Back-propagates eps (T, w.r.t. the logits when the last layer is OUTPUT/LOSS: dz from k_xent) through the net.
// `eps` must live in n->epsA or be an external buffer; uses epsA/epsB/epsC in rotation.
// input_act: when the caller will multiply the input gradient by act'(a) of the layer that FED this net (the generator's tanh in the stacked
// gan graph, J:228-310), the first layer's dgrad epilogue can do it (EPI_ACTBWD): *input_act_done reports whether it did.
// top_act_done: the epsilon handed in has already been multiplied by the last layer's act' (the mirror image of the above).
static int32_t net_backward(b2g_net* n, const void* net_in, void* eps, int rows, int groups, bool want_wgrad, bool need_input_grad, bool allreduce_follows = false,
                            const TcEpi* input_act = nullptr, bool* input_act_done = nullptr, bool top_act_done = false) {
  cudaStream_t s = n->ctx->stream, s2 = n->ctx->side; const int R = rows;
  void* cur = eps;
  if (input_act_done) *input_act_done = false;
  n->pending.count = 0;
  // Three epsilon buffers in rotation.  Weight gradients are forked to the side stream (they only READ delta and the layer
  // input), so the input-gradient chain -- the critical path -- never waits for them; a buffer still being read by a
  // forked wgrad is not overwritten before that wgrad's event has fired.
  void* bufs[3] = {n->epsA, n->epsB, n->epsC}; cudaEvent_t reader[3] = {nullptr, nullptr, nullptr}; bool forked = false;
  auto other = [&](void* p) -> void* {
    int pick = -1;
    for (int k = 0; k < 3; ++k) if (bufs[k] != p && !reader[k]) { pick = k; break; }
    if (pick < 0) for (int k = 0; k < 3; ++k) if (bufs[k] != p) { pick = k; break; }
    if (reader[pick]) { cudaStreamWaitEvent(s, reader[pick], 0); reader[pick] = nullptr; }
    return bufs[pick];
  };
  auto fork_wgrad = [&](int li, const void* delta) {      // side stream starts once delta is final
    cudaEventRecord(n->ev_fork[li], s); cudaStreamWaitEvent(s2, n->ev_fork[li], 0); forked = true; (void)delta;
  };
  auto mark_reader = [&](int li, const void* delta) {
    cudaEventRecord(n->ev_done[li], s2);
    for (int k = 0; k < 3; ++k) if (bufs[k] == delta) reader[k] = n->ev_done[li];
  };
  std::vector<char> act_done(n->L.size(), 0);        // layer i's own activation derivative was applied by the dgrad epilogue of the layer above
  if (top_act_done) act_done.back() = 1;
  // what the dgrad of GEMM layer i can fold into its epilogue: the BatchNorm-backward reductions of the BatchNorm(+activation) below it, or the
  // activation derivative of the GEMM layer below it / of the layer that fed the net
  auto pick_fuse = [&](int i, TcEpi* e, int* target) -> bool {
    *target = -1;
    if (!tc_on(n)) return false;
    int k = i - 1; while (k >= 0 && n->L[k].act_fused_into_prev) --k;
    if (k < 0) { if (input_act) { *e = *input_act; *target = -2; return true; } return false; }
    // a skip source in [k, i) still waits for its vertices' share, added at the top of its own backward: nothing may be premultiplied before that
    for (int m = k; m < i; ++m) if (n->L[m].n_skip) return false;
    LayerRT& b = n->L[k];
    if (b.d.type == B2G_LAYER_BATCHNORM && b.fwd_fused && !b.d.frozen && b.fwd_groups == groups) {
      e->mode = EPI_BNBWD; e->acc = b.acc_bwd; e->imgs_per_group = R / groups; e->aux = (const __nv_bfloat16*)b.out; e->aux2 = (const __nv_bfloat16*)(k == 0 ? net_in : n->L[k - 1].out);
      e->act = b.fused_act; e->alpha = b.fused_alpha; *target = k; return true;
    }
    if (k == i - 1 && b.has_gemm() && b.d.act != B2G_ACT_IDENTITY && b.d.type != B2G_LAYER_OUTPUT) {
      e->mode = EPI_ACTBWD; e->aux = (const __nv_bfloat16*)b.out; e->act = b.d.act; e->alpha = b.d.act_alpha; *target = k; return true;
    }
    return false;
  };
  auto note_fused = [&](int target, const TcEpi& e, bool fused) {
    if (!fused || target == -1) return;
    if (target == -2) { if (input_act_done) *input_act_done = true; return; }
    if (e.mode == EPI_BNBWD) n->L[target].bwd_premul = true; else act_done[target] = 1;
  };
  for (int i = (int)n->L.size() - 1; i >= 0; --i) {
    LayerRT& l = n->L[i]; const b2g_layer_desc& d = l.d;
    const void* lin = i == 0 ? net_in : n->L[i - 1].out;
    // the epsilon w.r.t. this layer's input is needed only if a trainable layer sits below it (or the caller wants d/d input)
    bool need_in = need_input_grad;
    if (!need_in) for (int j = 0; j < i; ++j) if (!n->L[j].d.frozen && (n->L[j].has_reg() || n->L[j].d.type == B2G_LAYER_BATCHNORM)) need_in = true;
    const bool want_wgrad_l = want_wgrad && !d.frozen;
    // a skip source: its vertices' shares join the spine epsilon before anything of its own backward runs
    if (l.skip_acc) k_skip_add(n->prec, cur, l.skip_acc, (size_t)R * l.out_elems, s);
    switch (d.type) {
      case B2G_LAYER_LOSS: case B2G_LAYER_CNN_LOSS: break;
      case B2G_LAYER_ELEMENTWISE:      // the spine's share in place, the skip's into the source's accumulator; PRODUCT / MAX read both inputs
        if (need_in) k_vertex_ew_bwd(n->prec, d.act, l.vorder, cur, lin, n->L[l.vsrc].out, n->L[l.vsrc].skip_acc, l.vfirst ? 0 : 1, (size_t)R * l.out_elems, s);
        break;
      case B2G_LAYER_MERGE:
        if (need_in) {
          const LayerRT& src = n->L[l.vsrc]; void* nx = other(cur);
          k_merge_bwd(n->prec, cur, nx, src.skip_acc, (size_t)R * l.oh * l.ow, l.vorder ? src.oc : l.ic, l.vorder ? l.ic : src.oc, l.vorder == 0, l.vfirst ? 0 : 1, s);
          cur = nx;
        }
        break;
      case B2G_LAYER_CONV2D: case B2G_LAYER_DENSE: case B2G_LAYER_OUTPUT: {
        ConvGeom g = l.geom; g.N = R;
        if (d.act != B2G_ACT_IDENTITY && !act_done[i]) k_act_bwd_from_output(n->prec, l.out, cur, cur, (size_t)R * l.out_elems, d.act, d.act_alpha, s);
        if (l.ext_z) k_act_ext_bwd(n->prec, l.ext_act, l.ext_alpha, l.ext_z, cur, (size_t)R * l.out_elems, s);
        if (want_wgrad_l) {
          fork_wgrad(i, cur);
          bool bias_done = false;
          B2(gemm_wgrad(n, l, g, lin, cur, n->grads + l.off_W, s2, n->scratch2, l.off_b >= 0 ? n->grads + l.off_b : nullptr, &bias_done));
          if (l.off_b >= 0 && !bias_done) k_colsum(n->prec, cur, R * l.oh * l.ow, l.oc, n->scratch2, n->grads + l.off_b, 0, s2);
          mark_reader(i, cur);
        }
        if (need_in) { void* nx = other(cur); TcEpi e{}; int tgt; bool fused = false; const bool can = pick_fuse(i, &e, &tgt);
          B2(gemm_dgrad(n, l, g, cur, nullptr, nx, ACT_IDENTITY, 0.f, nullptr, can ? &e : nullptr, &fused)); note_fused(tgt, e, fused); cur = nx; }
      } break;
      case B2G_LAYER_DECONV2D: {
        ConvGeom g = l.geom; g.N = R;
        if (d.act != B2G_ACT_IDENTITY && !act_done[i]) k_act_bwd_from_output(n->prec, l.out, cur, cur, (size_t)R * l.out_elems, d.act, d.act_alpha, s);
        if (l.ext_z) k_act_ext_bwd(n->prec, l.ext_act, l.ext_alpha, l.ext_z, cur, (size_t)R * l.out_elems, s);
        if (want_wgrad_l) {
          fork_wgrad(i, cur);
          B2(gemm_wgrad(n, l, g, /*conv input = deconv out grad*/ cur, /*conv dy = deconv input*/ lin, n->grads + l.off_W, s2, n->scratch2));
          if (l.off_b >= 0) k_colsum(n->prec, cur, R * l.oh * l.ow, l.oc, n->scratch2, n->grads + l.off_b, 0, s2);
          mark_reader(i, cur);
        }
        if (need_in) { void* nx = other(cur); TcEpi e{}; int tgt; bool fused = false; const bool can = pick_fuse(i, &e, &tgt);
          B2(gemm_fprop(n, l, g, cur, nullptr, nx, ACT_IDENTITY, 0.f, nullptr, can ? &e : nullptr, &fused)); note_fused(tgt, e, fused); cur = nx; }
      } break;
      case B2G_LAYER_BATCHNORM: {
        // FrozenLayer BatchNorm ran in test mode (running statistics): it has no parameter gradients, and its input gradient would be the
        // affine-only dy * gamma * invstd, not the batch-statistics form below.  The reference never differentiates through its frozen
        // trunk (J:335-370: only the new head trains), so that case is refused rather than computed wrongly.
        if (d.frozen) { if (need_in) return fail(B2G_ERR_UNSUPPORTED, "layer %d: a gradient through a frozen BatchNorm (trainable layer or input gradient below it) is not implemented", i); break; }
        // an accumulator forward never writes bn_mean / bn_invstd: its backward is the accumulator path, over the forward's groups
        if (l.fwd_fused && l.fwd_groups != groups) return fail(B2G_ERR_ARG, "layer %d: BatchNorm backward in %d groups after a forward in %d", i, groups, l.fwd_groups);
        int rows_pg = (R / groups) * l.oh * l.ow; void* nx = need_in ? other(cur) : nullptr;
        if (l.fwd_fused) {
          if (!l.bwd_premul) k_bn_bwd_stats_acc(lin, cur, rows_pg, l.oc, groups, l.bn_coef, l.fused_act, l.fused_alpha, l.acc_bwd, s);
          const int reps = sync_bn_world(n);
          if (reps > 1) NC(g_nccl.ar(l.acc_bwd, l.acc_bwd, k_bn_acc_elems(l.oc, groups), /*ncclUint64*/ 5, /*ncclSum*/ 0, n->ctx->comm, s));
          k_bn_bwd_apply_acc(lin, cur, nx, rows_pg, l.oc, groups, l.bn_coef, l.fused_act, l.fused_alpha, l.bwd_premul ? 1 : 0, l.acc_bwd, n->grads + l.off_gamma, n->grads + l.off_beta, want_wgrad_l ? 1 : 0, s, reps);
          l.bwd_premul = false;
        } else
        k_bn_bwd(n->prec, lin, cur, nx, rows_pg, l.oc, groups, l.bn_mean, l.bn_invstd, n->params + l.off_gamma, n->params + l.off_beta, l.fused_act, l.fused_alpha,
                 n->scratch, n->grads + l.off_gamma, n->grads + l.off_beta, want_wgrad_l ? 1 : 0, s);
        if (need_in) cur = nx;
      } break;
      case B2G_LAYER_ACTIVATION:
        if (l.ext_act) k_act_ext_bwd(n->prec, l.ext_act, l.ext_alpha, lin, cur, (size_t)R * l.out_elems, s);      // z = the layer's input
        else if (!l.act_fused_into_prev) k_act_bwd_from_output(n->prec, l.out, cur, cur, (size_t)R * l.out_elems, d.act, d.act_alpha, s);
        break;
      case B2G_LAYER_MAXPOOL: if (need_in) { void* nx = other(cur); k_maxpool_bwd(n->prec, cur, l.argmax, nx, R, l.ih, l.iw, l.ic, l.oh, l.ow, d.k_h, d.k_w, d.s_h, d.s_w, s); cur = nx; } break;
      case B2G_LAYER_SUBSAMPLING:      // PNORM reads the layer's input x and its own output y
        if (need_in) { void* nx = other(cur); k_pool2d_bwd(n->prec, l.pool, l.pnorm, cur, lin, l.out, nx, R, l.ih, l.iw, l.ic, l.oh, l.ow, d.k_h, d.k_w, d.s_h, d.s_w, d.p_h, d.p_w, s); cur = nx; }
        break;
      case B2G_LAYER_GLOBAL_POOLING:
        if (need_in) { void* nx = other(cur); k_global_pool_bwd(n->prec, l.pool, l.pnorm, cur, lin, l.out, l.pool_idx, nx, R, l.ih * l.iw, l.ic, s); cur = nx; }
        break;
      case B2G_LAYER_UPSAMPLE2D: if (need_in) { void* nx = other(cur); k_upsample_bwd(n->prec, cur, nx, R, l.ih, l.iw, l.ic, d.k_h, s); cur = nx; } break;
      case B2G_LAYER_FF_TO_CNN: if (!l.out_alias && need_in) { void* nx = other(cur); k_permute(n->prec, cur, nx, R, l.oc, l.oh * l.ow, 0, s); cur = nx; } break;
      case B2G_LAYER_CNN_TO_FF: if (!l.out_alias && need_in) { void* nx = other(cur); k_permute(n->prec, cur, nx, R, l.ic, l.ih * l.iw, 1, s); cur = nx; } break;
      case B2G_LAYER_DROPOUT:       // the forward's mask (GAUSSIAN_DROPOUT: its P; GAUSSIAN_NOISE: the identity, no launch)
        if (need_in && l.drop_live) {
          if (d.act == B2G_DROPOUT && !l.drop_sched) k_dropout_bwd(n->prec, cur, cur, l.drop_mask, (size_t)R * l.out_elems, 1.0f / d.act_alpha, s);
          else k_noise_bwd(n->prec, d.act, cur, cur, l.drop_mask, l.drop_rec, (size_t)R * l.out_elems, noise_args(n, i), noise_sched(n, l, nullptr, nullptr), s);
        }
        break;
      case B2G_LAYER_PRELU:         // dx in place from the layer's input x; a trainable layer also leaves its slope partials for the reduce list
        if (need_in || want_wgrad_l) {
          k_prelu_bwd(n->prec, lin, cur, n->params + l.off_W, want_wgrad_l ? l.prelu_part : nullptr, need_in ? 1 : 0, R, l.pg, s);
          if (want_wgrad_l) {
            fork_wgrad(i, cur);             // the side stream, which runs the pass's reduce list, starts after the partials
            if (n->pending.count == ReduceList::MAX_JOBS) flush_pending_reduce(n, s2);
            prelu_queue_reduce(&n->pending, l.prelu_part, n->grads + l.off_W, R, l.pg);
          }
        }
        break;
    }
    if (i == n->ar_split_layer && want_wgrad && allreduce_follows && ar_overlap_on(n)) {
      // every gradient of layers >= i is queued (BN scale/shift on s, weights/biases on s2): all-reduce that tail on the comm stream now
      b2g_ctx* c = n->ctx;
      cudaEventRecord(c->ev_c0, s); cudaStreamWaitEvent(c->comm_stream, c->ev_c0, 0);
      if (forked) { flush_pending_reduce(n, s2); cudaEventRecord(c->ev_c1, s2); cudaStreamWaitEvent(c->comm_stream, c->ev_c1, 0); }
      NC(g_nccl.ar(n->grads + n->ar_split_off, n->grads + n->ar_split_off, (size_t)(n->n_params - n->ar_split_off), /*ncclFloat32*/ 7, /*ncclSum*/ 0, c->comm, c->comm_stream));
      n->ar_tail_sent = true;
    }
    if (!need_in) { cur = nullptr; break; }
  }
  n->input_grad = cur;
  if (forked) { flush_pending_reduce(n, s2); cudaEventRecord(n->ev_join, s2); cudaStreamWaitEvent(s, n->ev_join, 0); }   // join before all-reduce / updater
  CHECK_KERNELS();
  return 0;
}

static int32_t net_allreduce_grads(b2g_net* n) {
  b2g_ctx* c = n->ctx; if (!c->comm || c->world == 1 || !n->grad_allreduce) return 0;
  if (n->ar_tail_sent) {        // the tail bucket left during backward; the head follows on the same stream, the updater waits for both
    n->ar_tail_sent = false;
    cudaEventRecord(c->ev_c0, c->stream); cudaStreamWaitEvent(c->comm_stream, c->ev_c0, 0);
    NC(g_nccl.ar(n->grads, n->grads, (size_t)n->ar_split_off, /*ncclFloat32*/ 7, /*ncclSum*/ 0, c->comm, c->comm_stream));
    cudaEventRecord(c->ev_c2, c->comm_stream); cudaStreamWaitEvent(c->stream, c->ev_c2, 0);
    return 0;
  }
  if (n->ar_bf16 && n->ar_buf) {     // half the bytes on the wire: round to bf16, sum in bf16, widen (option; the default fp32 payload keeps DP bit-identical to one GPU)
    k_cast_f32_to_bf16(n->grads, n->ar_buf, (size_t)n->n_params, c->stream);
    NC(g_nccl.ar(n->ar_buf, n->ar_buf, (size_t)n->n_params, /*ncclBfloat16*/ 9, /*ncclSum*/ 0, c->comm, c->stream));
    k_nhwc_to_nchw_f32(PREC_BF16, n->ar_buf, n->grads, 1, 1, (int)n->n_params, c->stream);
    return 0;
  }
  if (n->p2p) {        // one kernel over NVLink peer memory instead of the NCCL ring
    P2pArgs a{}; for (int r = 0; r < c->world; ++r) { a.grads[r] = n->p2p_peer_grads[r]; a.flags[r] = c->p2p_peer_flags[r]; }
    a.rank = c->rank; a.world = c->world; a.n = (size_t)n->n_params; a.state = c->p2p_state;
    k_p2p_allreduce(a, c->stream); CHECK_KERNELS(); return 0;
  }
  NC(g_nccl.ar(n->grads, n->grads, (size_t)n->n_params, /*ncclFloat32*/ 7, /*ncclSum*/ 0, c->comm, c->stream));
  return 0;
}
// The constraint rounds of the net's plan, in order; a net without constraints launches nothing
static void net_launch_constraints(b2g_net* n, cudaStream_t s) {
  for (const auto& r : n->con_rounds) {
    k_constraint_onepass(n->params, n->shadow, n->con_jobs, r.j0, r.j1, r.onepass_blocks, s);
    k_constraint_twopass(n->params, n->shadow, n->con_jobs, r.t0, r.t1, r.norm_blocks, r.scale_blocks, n->con_partial, n->con_ticket, n->con_mult, s);
  }
}
static int32_t net_update(b2g_net* n, int mb_local) {
  cudaStream_t s = n->ctx->stream; int W = n->ctx->comm ? n->ctx->world : 1;
  // BN running-stat pseudo-gradients are exempt from the minibatch division; under DP they are averaged over ranks
  if (!n->grad_allreduce) W = 1;     // parameter-averaging mode: purely local update
  const float inv_mb = 1.0f / ((float)mb_local * W), inv_world = 1.0f / (float)W;
  // L2 gradient normalization: one kernel takes the norms of the (all-reduced) gradient after /mb and leaves one multiplier per segment
  const bool gn = n->gn_mode != B2G_GN_NONE;
  if (gn) {
    const bool per_layer = n->gn_mode == B2G_GN_RENORM_L2_LAYER || n->gn_mode == B2G_GN_CLIP_L2_LAYER;
    const bool clip = n->gn_mode == B2G_GN_CLIP_L2_LAYER || n->gn_mode == B2G_GN_CLIP_L2_PARAM;
    k_gradnorm(n->grads, n->segs_dev, n->chunk_seg_dev, n->chunk_off_dev, n->nchunks, per_layer ? n->gn_layer_groups : n->gn_param_groups,
               per_layer ? n->gn_n_layer_groups : n->gn_n_param_groups, clip ? 1 : 0, n->gn_threshold, inv_mb, inv_world, n->gn_partial, n->gn_ticket, n->gn_mult, s);
  }
  // one pass: /mb -> [x multiplier] -> clip -> updater [at the scheduled lr] -> +l2*W -> theta -= g, the bf16 operand copies (straight and
  // packed) and the iteration counter
  k_updater(n->params, n->grads, n->st0, n->st1, n->st2, n->segs_dev, n->chunk_seg_dev, n->chunk_off_dev, n->nchunks, inv_mb, inv_world, n->step_dev, n->upd_ticket,
            n->shadow, gn ? n->gn_mult : nullptr, n->sched_on ? n->sched_dev : nullptr, n->epoch_dev, n->upd_ext, s);
  net_launch_constraints(n, s);      // applyConstraints after the step (StochasticGradientDescent.optimize)
  CHECK_KERNELS();
  return 0;
}

// ------------------------------------------------------------------ C-ABI: context ----------------------
extern "C" int32_t b2g_version(void) { return B2G_VERSION; }
extern "C" const char* b2g_last_error(void) { return g_err; }

extern "C" int32_t b2g_ctx_create(int32_t device, b2g_ctx** out) {
  if (!out) return fail(B2G_ERR_ARG, "null out");
  int count = 0; cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) return fail(B2G_ERR_NO_DEVICE, "no CUDA device (%s); libb200gan has no CPU fallback", e == cudaSuccess ? "count=0" : cudaGetErrorString(e));
  if (device < 0 || device >= count) return fail(B2G_ERR_ARG, "device %d of %d", device, count);
  CU(cudaSetDevice(device));
  b2g_ctx* c = new b2g_ctx(); c->device = device;
  CU(cudaGetDeviceProperties(&c->prop, device));
  if (c->prop.major != 9) { int mj = c->prop.major, mn = c->prop.minor; delete c; return fail(B2G_ERR_NO_DEVICE, "device is sm_%d%d; this library is built for sm_90a (H100) only", mj, mn); }
  CU(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  CU(cudaStreamCreateWithFlags(&c->side, cudaStreamNonBlocking)); CU(cudaStreamCreateWithFlags(&c->side2, cudaStreamNonBlocking));
  CU(cudaEventCreateWithFlags(&c->ev_a, cudaEventDisableTiming)); CU(cudaEventCreateWithFlags(&c->ev_b, cudaEventDisableTiming));
  CU(cudaStreamCreateWithFlags(&c->comm_stream, cudaStreamNonBlocking));
  CU(cudaEventCreateWithFlags(&c->ev_c0, cudaEventDisableTiming)); CU(cudaEventCreateWithFlags(&c->ev_c1, cudaEventDisableTiming)); CU(cudaEventCreateWithFlags(&c->ev_c2, cudaEventDisableTiming));
  c->tc_ok = tc_init() == 0;
  *out = c; return 0;
}
extern "C" int32_t b2g_ctx_destroy(b2g_ctx* c) {
  if (!c) return 0; cudaSetDevice(c->device);
  if (c->p2p_flags_mapped) for (int r = 0; r < c->world; ++r) if (r != c->rank && c->p2p_peer_flags[r]) cudaIpcCloseMemHandle(c->p2p_peer_flags[r]);
  if (c->p2p_flags) cudaFree(c->p2p_flags); if (c->p2p_state) cudaFree(c->p2p_state);
  if (c->comm && g_nccl.destroy) g_nccl.destroy(c->comm);
  if (c->t0) { cudaEventDestroy(c->t0); cudaEventDestroy(c->t1); } if (c->flush_buf) cudaFree(c->flush_buf);
  if (c->side) cudaStreamDestroy(c->side); if (c->side2) cudaStreamDestroy(c->side2); if (c->ev_a) cudaEventDestroy(c->ev_a); if (c->ev_b) cudaEventDestroy(c->ev_b);
  if (c->comm_stream) cudaStreamDestroy(c->comm_stream); if (c->ev_c0) cudaEventDestroy(c->ev_c0); if (c->ev_c1) cudaEventDestroy(c->ev_c1); if (c->ev_c2) cudaEventDestroy(c->ev_c2);
  if (c->stream) cudaStreamDestroy(c->stream); delete c; return 0;
}
extern "C" int32_t b2g_timer_start(b2g_ctx* c) {
  if (!c) return fail(B2G_ERR_ARG, "null ctx"); CU(cudaSetDevice(c->device));
  if (!c->t0) { CU(cudaEventCreate(&c->t0)); CU(cudaEventCreate(&c->t1)); }
  CU(cudaEventRecord(c->t0, c->stream)); return 0;
}
extern "C" int32_t b2g_timer_stop_ms(b2g_ctx* c, float* ms) {
  if (!c || !ms || !c->t0) return fail(B2G_ERR_ARG, "timer not started"); CU(cudaSetDevice(c->device));
  CU(cudaEventRecord(c->t1, c->stream)); CU(cudaEventSynchronize(c->t1)); CU(cudaEventElapsedTime(ms, c->t0, c->t1)); return 0;
}
extern "C" int32_t b2g_flush_l2(b2g_ctx* c) {
  if (!c) return fail(B2G_ERR_ARG, "null ctx"); CU(cudaSetDevice(c->device));
  if (!c->flush_buf) { c->flush_bytes = (size_t)256 << 20; CU(cudaMalloc(&c->flush_buf, c->flush_bytes)); }
  CU(cudaMemsetAsync(c->flush_buf, 0, c->flush_bytes, c->stream)); return 0;
}
extern "C" int32_t b2g_sync(b2g_ctx* c) { if (!c) return fail(B2G_ERR_ARG, "null ctx"); CU(cudaSetDevice(c->device)); CU(cudaStreamSynchronize(c->stream)); return 0; }
extern "C" int32_t b2g_launch_count(b2g_ctx* c, uint64_t* out) { if (!c || !out) return fail(B2G_ERR_ARG, "null"); *out = g_launch_count; return 0; }
extern "C" int32_t b2g_device_info(b2g_ctx* c, int32_t* sm, int32_t* mj, int32_t* mn, uint64_t* mem) {
  if (!c) return fail(B2G_ERR_ARG, "null ctx");
  if (sm) *sm = c->prop.multiProcessorCount; if (mj) *mj = c->prop.major; if (mn) *mn = c->prop.minor; if (mem) *mem = c->prop.totalGlobalMem; return 0;
}

// ------------------------------------------------------------------ C-ABI: nets --------------------------
extern "C" int32_t b2g_net_create(b2g_ctx* ctx, const b2g_net_config* cfg, const b2g_layer_desc* layers, int32_t nl, b2g_net** out) {
  if (!ctx || !cfg || !layers || nl < 1 || !out) return fail(B2G_ERR_ARG, "b2g_net_create: null/empty argument");
  if (cfg->max_batch < 1 || cfg->in_h < 1 || cfg->in_w < 1 || cfg->in_c < 1) return fail(B2G_ERR_ARG, "b2g_net_create: bad input type / max_batch");
  if (cfg->precision != B2G_PREC_FP32 && cfg->precision != B2G_PREC_BF16) return fail(B2G_ERR_ARG, "b2g_net_create: precision %d", cfg->precision);
  for (int32_t i = 0; i < nl; ++i)
    if (layers[i].updater < B2G_UPD_SGD || layers[i].updater > B2G_UPD_ADADELTA) return fail(B2G_ERR_ARG, "b2g_net_create: layer %d: unknown updater %d", i, layers[i].updater);
  CU(cudaSetDevice(ctx->device));
  b2g_net* n = new b2g_net(); n->ctx = ctx; n->cfg = *cfg; n->prec = cfg->precision == B2G_PREC_BF16 ? PREC_BF16 : PREC_F32;
  if (n->cfg.bn_groups < 1) n->cfg.bn_groups = 1;
  int32_t r = net_build(n, layers, nl); if (!r) r = net_alloc(n); if (!r) r = net_init_params_and_updater(n);
  if (!r) { net_refresh_shadow(n); cudaError_t e = cudaStreamSynchronize(ctx->stream); if (e != cudaSuccess) r = fail(B2G_ERR_CUDA, "init: %s", cudaGetErrorString(e)); }
  if (r) { for (void* p : n->allocs) cudaFree(p); delete n; return r; }
  *out = n; return 0;
}
extern "C" int32_t b2g_net_destroy(b2g_net* n) {
  if (!n) return 0; cudaSetDevice(n->ctx->device); cudaStreamSynchronize(n->ctx->stream); cudaStreamSynchronize(n->ctx->side);
  for (auto e : n->ev_fork) if (e) cudaEventDestroy(e); for (auto e : n->ev_done) if (e) cudaEventDestroy(e); if (n->ev_join) cudaEventDestroy(n->ev_join);
  if (n->p2p) for (int r = 0; r < n->ctx->world; ++r) if (r != n->ctx->rank && n->p2p_peer_grads[r]) cudaIpcCloseMemHandle(n->p2p_peer_grads[r]);
  if (n->sched_map) cudaFree(n->sched_map);
  for (auto& l : n->L) { if (l.drop_map) cudaFree(l.drop_map); if (l.wn_map) cudaFree(l.wn_map); }
  cudaFree(n->con_jobs); cudaFree(n->con_partial); cudaFree(n->con_mult);
  for (void* p : n->allocs) cudaFree(p); delete n; return 0;
}
extern "C" int32_t b2g_net_num_params(b2g_net* n, int64_t* out) { if (!n || !out) return fail(B2G_ERR_ARG, "null"); *out = n->n_params; return 0; }
extern "C" int32_t b2g_net_output_size(b2g_net* n, int64_t* out) { if (!n || !out) return fail(B2G_ERR_ARG, "null"); *out = (int64_t)n->L.back().out_elems; return 0; }
extern "C" int32_t b2g_net_layer_output_size(b2g_net* n, int32_t layer, int64_t* out) {
  if (!n || !out || layer < 0 || layer >= (int)n->L.size()) return fail(B2G_ERR_ARG, "bad layer index"); *out = (int64_t)n->L[layer].out_elems; return 0;
}

struct ParamRef { int64_t off, len; bool conv_w; int A, B, taps; int layer; };
static int32_t find_param(b2g_net* n, const char* layer, const char* param, ParamRef* r) {
  for (size_t i = 0; i < n->L.size(); ++i) { LayerRT& l = n->L[i];
    if (strncmp(l.d.name, layer, B2G_NAME_LEN)) continue;
    r->conv_w = false; r->layer = (int)i;
    if (!strcmp(param, "W") && l.off_W >= 0) { r->off = l.off_W; r->len = l.n_W; r->conv_w = l.wTaps > 1; r->A = l.wA; r->B = l.wB; r->taps = l.wTaps; return 0; }
    if (!strcmp(param, "b") && l.off_b >= 0) { r->off = l.off_b; r->len = l.d.n_out; return 0; }
    if (l.d.type == B2G_LAYER_BATCHNORM) {
      if (!strcmp(param, "gamma")) { r->off = l.off_gamma; r->len = l.oc; return 0; }
      if (!strcmp(param, "beta")) { r->off = l.off_beta; r->len = l.oc; return 0; }
      if (!strcmp(param, "mean")) { r->off = l.off_mean; r->len = l.oc; return 0; }
      if (!strcmp(param, "var")) { r->off = l.off_var; r->len = l.oc; return 0; }
    }
    return fail(B2G_ERR_ARG, "layer %s has no parameter %s", layer, param);
  }
  return fail(B2G_ERR_ARG, "no layer named %s", layer);
}
extern "C" int32_t b2g_net_set_param(b2g_net* n, const char* layer, const char* param, const float* host, int64_t cnt) {
  if (!n || !layer || !param || !host) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device));
  ParamRef r; B2(find_param(n, layer, param, &r));
  if (cnt != r.len) return fail(B2G_ERR_SHAPE, "%s.%s has %lld elements, got %lld", layer, param, (long long)r.len, (long long)cnt);
  std::vector<float> tmp; const float* src = host;
  if (r.conv_w) { tmp.resize(r.len); w_dl4j_to_internal(host, tmp.data(), r.A, r.B, r.taps); src = tmp.data(); }
  CU(cudaMemcpyAsync(n->params + r.off, src, sizeof(float) * r.len, cudaMemcpyHostToDevice, n->ctx->stream));
  CU(cudaStreamSynchronize(n->ctx->stream));
  if (!strcmp(param, "W")) { net_refresh_shadow(n, r.layer); CU(cudaStreamSynchronize(n->ctx->stream)); }
  return 0;
}
static int32_t read_flat(b2g_net* n, const float* dev, float* host, int64_t cnt) {
  if (cnt != n->n_params) return fail(B2G_ERR_SHAPE, "net has %lld parameters, got %lld", (long long)n->n_params, (long long)cnt);
  std::vector<float> tmp(n->n_params);
  CU(cudaMemcpyAsync(tmp.data(), dev, sizeof(float) * n->n_params, cudaMemcpyDeviceToHost, n->ctx->stream)); CU(cudaStreamSynchronize(n->ctx->stream));
  memcpy(host, tmp.data(), sizeof(float) * n->n_params);
  for (auto& l : n->L) if (l.has_gemm() && l.wTaps > 1) w_internal_to_dl4j(tmp.data() + l.off_W, host + l.off_W, l.wA, l.wB, l.wTaps);
  return 0;
}
static int32_t write_flat(b2g_net* n, float* dev, const float* host, int64_t cnt) {
  if (cnt != n->n_params) return fail(B2G_ERR_SHAPE, "net has %lld parameters, got %lld", (long long)n->n_params, (long long)cnt);
  std::vector<float> tmp(host, host + n->n_params);
  for (auto& l : n->L) if (l.has_gemm() && l.wTaps > 1) w_dl4j_to_internal(host + l.off_W, tmp.data() + l.off_W, l.wA, l.wB, l.wTaps);
  CU(cudaMemcpyAsync(dev, tmp.data(), sizeof(float) * n->n_params, cudaMemcpyHostToDevice, n->ctx->stream)); CU(cudaStreamSynchronize(n->ctx->stream));
  return 0;
}
extern "C" int32_t b2g_net_get_param(b2g_net* n, const char* layer, const char* param, float* host, int64_t cnt) {
  if (!n || !layer || !param || !host) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device));
  ParamRef r; B2(find_param(n, layer, param, &r));
  if (cnt != r.len) return fail(B2G_ERR_SHAPE, "%s.%s has %lld elements, got %lld", layer, param, (long long)r.len, (long long)cnt);
  std::vector<float> tmp(r.len);
  CU(cudaMemcpyAsync(tmp.data(), n->params + r.off, sizeof(float) * r.len, cudaMemcpyDeviceToHost, n->ctx->stream)); CU(cudaStreamSynchronize(n->ctx->stream));
  if (r.conv_w) w_internal_to_dl4j(tmp.data(), host, r.A, r.B, r.taps); else memcpy(host, tmp.data(), sizeof(float) * r.len);
  return 0;
}
extern "C" int32_t b2g_net_get_params(b2g_net* n, float* host, int64_t cnt) { if (!n || !host) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device)); return read_flat(n, n->params, host, cnt); }
extern "C" int32_t b2g_net_set_params(b2g_net* n, const float* host, int64_t cnt) {
  if (!n || !host) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device)); B2(write_flat(n, n->params, host, cnt)); net_refresh_shadow(n); CU(cudaStreamSynchronize(n->ctx->stream)); return 0;
}
extern "C" int32_t b2g_net_get_gradients(b2g_net* n, float* host, int64_t cnt) { if (!n || !host) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device)); return read_flat(n, n->grads, host, cnt); }
// [state0 | state1], plus | state2 on nets with an AMSGrad segment
static int64_t updater_state_size(const b2g_net* n) { return (n->st2 ? 3 : 2) * n->n_params; }
extern "C" int32_t b2g_net_updater_state_size(b2g_net* n, int64_t* out) { if (!n || !out) return fail(B2G_ERR_ARG, "null"); *out = updater_state_size(n); return 0; }
extern "C" int32_t b2g_net_get_updater_state(b2g_net* n, float* host, int64_t cnt) {
  if (!n || !host) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device));
  if (cnt != updater_state_size(n)) return fail(B2G_ERR_SHAPE, "updater state has %lld elements", (long long)updater_state_size(n));
  B2(read_flat(n, n->st0, host, n->n_params)); B2(read_flat(n, n->st1, host + n->n_params, n->n_params));
  return n->st2 ? read_flat(n, n->st2, host + 2 * n->n_params, n->n_params) : 0;
}
extern "C" int32_t b2g_net_set_updater_state(b2g_net* n, const float* host, int64_t cnt) {
  if (!n || !host) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device));
  if (cnt != updater_state_size(n)) return fail(B2G_ERR_SHAPE, "updater state has %lld elements", (long long)updater_state_size(n));
  B2(write_flat(n, n->st0, host, n->n_params)); B2(write_flat(n, n->st1, host + n->n_params, n->n_params));
  return n->st2 ? write_flat(n, n->st2, host + 2 * n->n_params, n->n_params) : 0;
}

// host NCHW fp32 -> device input buffer (T NHWC)
static int32_t upload_input(b2g_net* n, const float* x, int rows, void* dst) {
  cudaStream_t s = n->ctx->stream; size_t cnt = (size_t)rows * n->in_elems;
  if (cnt > n->stage_floats) return fail(B2G_ERR_SHAPE, "input larger than staging");
  CU(cudaMemcpyAsync(n->stage_f32, x, sizeof(float) * cnt, cudaMemcpyHostToDevice, s));
  k_nchw_f32_to_nhwc(n->prec, n->stage_f32, dst, rows, n->cfg.in_c, n->cfg.in_h * n->cfg.in_w, s);
  return 0;
}
static int32_t download_act(b2g_net* n, const void* src, int rows, int C, int HW, float* host) {
  cudaStream_t s = n->ctx->stream; size_t cnt = (size_t)rows * C * HW;
  if (cnt > n->stage_floats) return fail(B2G_ERR_SHAPE, "activation larger than staging");
  k_nhwc_to_nchw_f32(n->prec, src, n->stage_f32, rows, C, HW, s);
  CU(cudaMemcpyAsync(host, n->stage_f32, sizeof(float) * cnt, cudaMemcpyDeviceToHost, s)); CU(cudaStreamSynchronize(s));
  return 0;
}

extern "C" int32_t b2g_net_output(b2g_net* n, const float* x, int32_t batch, int32_t train, float* out) {
  if (!n || !x || !out) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device));
  if (batch < 1 || batch > n->max_rows) return fail(B2G_ERR_SHAPE, "batch %d outside [1,%d]", batch, n->max_rows);
  B2(upload_input(n, x, batch, n->input));
  const void* res = nullptr; FwdOpts o{batch, 1, train != 0, false, nullptr};
  B2(net_forward(n, n->input, o, &res));
  LayerRT& l = n->L.back();
  if (l.d.type == B2G_LAYER_CNN_LOSS && l.d.loss == B2G_LOSS_MCXENT) {      // the per-pixel softmax
    k_cnn_softmax_xent(n->prec, res, nullptr, nullptr, l.probs, nullptr, batch * l.oh * l.ow, l.oc, 1, nullptr, nullptr, n->ctx->stream); res = l.probs;
  }
  else if (l.d.type == B2G_LAYER_CNN_LOSS && l.d.loss == B2G_LOSS_XENT) { k_sigmoid_out(n->prec, res, l.probs, (size_t)batch * l.out_elems, n->ctx->stream); res = l.probs; }
  else if (l.d.type == B2G_LAYER_CNN_LOSS) {      // a = act(z), as on a LOSS layer
    if (l.ext_act) { k_act_ext_fwd(n->prec, l.ext_act, l.ext_alpha, res, l.probs, (size_t)batch * l.out_elems, n->ctx->stream); res = l.probs; }
    else if (l.loss_act != ACT_IDENTITY) { k_act_fwd(n->prec, res, l.probs, (size_t)batch * l.out_elems, l.loss_act, l.loss_alpha, n->ctx->stream); res = l.probs; }
  }
  else if (l.d.type == B2G_LAYER_OUTPUT && l.d.loss == B2G_LOSS_MCXENT) { k_softmax_xent(n->prec, res, nullptr, nullptr, l.probs, nullptr, batch, l.oc, n->ctx->stream); res = l.probs; }
  else if ((l.d.type == B2G_LAYER_OUTPUT || l.d.type == B2G_LAYER_LOSS) && l.d.loss >= B2G_LOSS_MSE) {      // a = act(z); identity: the logits themselves
    if (l.ext_act) { k_act_ext_fwd(n->prec, l.ext_act, l.ext_alpha, res, l.probs, (size_t)batch * l.out_elems, n->ctx->stream); res = l.probs; }
    else if (l.loss_act != ACT_IDENTITY) { k_act_fwd(n->prec, res, l.probs, (size_t)batch * l.out_elems, l.loss_act, l.loss_alpha, n->ctx->stream); res = l.probs; }
  }
  else if (l.d.type == B2G_LAYER_OUTPUT || l.d.type == B2G_LAYER_LOSS) { k_sigmoid_out(n->prec, res, l.probs, (size_t)batch * l.out_elems, n->ctx->stream); res = l.probs; }
  return download_act(n, res, batch, l.oc, l.oh * l.ow, out);
}
extern "C" int32_t b2g_net_get_activation(b2g_net* n, int32_t layer, int32_t batch, float* host) {
  if (!n || !host || layer < 0 || layer >= (int)n->L.size()) return fail(B2G_ERR_ARG, "bad layer index"); CU(cudaSetDevice(n->ctx->device));
  LayerRT& l = n->L[layer]; if (!l.out) return fail(B2G_ERR_ARG, "layer %d has not run", layer);
  return download_act(n, l.out, batch, l.oc, l.oh * l.ow, host);
}

// The columns of the last layer's loss: the channels of a CnnLossLayer (its rows are pixels), else the outputs per example
static int loss_cols(const LayerRT& l) { return l.d.type == B2G_LAYER_CNN_LOSS ? l.oc : (int)std::max<size_t>(1, l.out_elems); }
static bool is_loss_layer(const LayerRT& l) { return l.d.type == B2G_LAYER_OUTPUT || l.d.type == B2G_LAYER_LOSS || l.d.type == B2G_LAYER_CNN_LOSS; }

// The loss of the net's last layer (b2g_loss) on its logits, one launch: dz = dL/dz, loss_sums[g] = the summed scores of group g's rows.  The only
// place that dispatches on the loss: fit, computeGradientAndScore and both losses of the GAN step come here.  A net that does not end in an
// OUTPUT or LOSS layer runs XENT.  mask: [rows][mask_width] in the labels' rows (null: none); with neither a mask nor the net's loss weights the
// unweighted instantiations run, else their weighted / masked ones (the same launches).
static void net_loss(b2g_net* n, const void* logits, const float* labels, void* dz, float* loss_sums, int rows_per_group, int groups,
                     const float* mask = nullptr, int mask_width = 0) {
  const LayerRT& l = n->L.back();
  const bool wm = n->loss_w_on || mask;
  const LossWM q{n->loss_w_on ? n->loss_w : nullptr, mask, mask_width, loss_cols(l)};
  if (l.d.type == B2G_LAYER_CNN_LOSS) {      // rows = the group's pixels, columns = the channels
    const int px = rows_per_group * l.oh * l.ow; cudaStream_t s = n->ctx->stream;
    if (l.d.loss == B2G_LOSS_XENT) {
      if (wm) k_cnn_xent_wm(n->prec, logits, labels, dz, loss_sums, (size_t)rows_per_group * l.out_elems, groups, n->cfg.xent_clip_eps, n->loss_partial, n->loss_ticket, q, s);
      else k_cnn_xent(n->prec, logits, labels, dz, loss_sums, (size_t)rows_per_group * l.out_elems, groups, n->cfg.xent_clip_eps, n->loss_partial, n->loss_ticket, s);
    }
    else if (l.d.loss == B2G_LOSS_MCXENT) {
      if (wm) k_cnn_softmax_xent_wm(n->prec, logits, labels, dz, loss_sums, px, l.oc, groups, n->loss_partial, n->loss_ticket, q, s);
      else k_cnn_softmax_xent(n->prec, logits, labels, dz, nullptr, loss_sums, px, l.oc, groups, n->loss_partial, n->loss_ticket, s);
    }
    else if (l.ext_act) {
      const size_t cnt = (size_t)rows_per_group * groups * l.out_elems;
      k_act_ext_fwd(n->prec, l.ext_act, l.ext_alpha, logits, l.probs, cnt, s);
      if (wm) k_loss_wm(n->prec, l.d.loss, ACT_IDENTITY, 0.f, l.probs, labels, dz, loss_sums, px, l.oc, groups, n->loss_partial, n->loss_ticket, q, s);
      else k_loss(n->prec, l.d.loss, ACT_IDENTITY, 0.f, l.probs, labels, dz, loss_sums, px, l.oc, groups, n->loss_partial, n->loss_ticket, s);
      k_act_ext_bwd(n->prec, l.ext_act, l.ext_alpha, logits, dz, cnt, s);
    }
    else if (wm) k_loss_wm(n->prec, l.d.loss, l.loss_act, l.loss_alpha, logits, labels, dz, loss_sums, px, l.oc, groups, n->loss_partial, n->loss_ticket, q, s);
    else k_loss(n->prec, l.d.loss, l.loss_act, l.loss_alpha, logits, labels, dz, loss_sums, px, l.oc, groups, n->loss_partial, n->loss_ticket, s);
    return;
  }
  const int loss = (l.d.type == B2G_LAYER_OUTPUT || l.d.type == B2G_LAYER_LOSS) ? l.d.loss : B2G_LOSS_XENT;
  cudaStream_t s = n->ctx->stream;
  if (loss == B2G_LOSS_MCXENT) {
    if (wm) k_softmax_xent_wm(n->prec, logits, labels, dz, loss_sums, rows_per_group * groups, l.oc, q, s);
    else k_softmax_xent(n->prec, logits, labels, dz, nullptr, loss_sums, rows_per_group * groups, l.oc, s);
  }
  else if (loss == B2G_LOSS_XENT) {
    if (wm) k_xent_wm(n->prec, logits, labels, dz, loss_sums, rows_per_group, groups, n->cfg.xent_clip_eps, q, s);
    else k_xent(n->prec, logits, labels, dz, loss_sums, rows_per_group, groups, n->cfg.xent_clip_eps, s);
  }
  else if (l.ext_act) {      // activation of codes 5-16: a = f(z) into probs, the loss on a with the identity, then dL/dz = dL/da * f'(z)
    const size_t cnt = (size_t)rows_per_group * groups * l.out_elems;
    k_act_ext_fwd(n->prec, l.ext_act, l.ext_alpha, logits, l.probs, cnt, s);
    if (wm) k_loss_wm(n->prec, loss, ACT_IDENTITY, 0.f, l.probs, labels, dz, loss_sums, rows_per_group, (int)l.out_elems, groups, n->loss_partial, n->loss_ticket, q, s);
    else k_loss(n->prec, loss, ACT_IDENTITY, 0.f, l.probs, labels, dz, loss_sums, rows_per_group, (int)l.out_elems, groups, n->loss_partial, n->loss_ticket, s);
    k_act_ext_bwd(n->prec, l.ext_act, l.ext_alpha, logits, dz, cnt, s);
  }
  else if (wm) k_loss_wm(n->prec, loss, l.loss_act, l.loss_alpha, logits, labels, dz, loss_sums, rows_per_group, (int)l.out_elems, groups, n->loss_partial, n->loss_ticket, q, s);
  else k_loss(n->prec, loss, l.loss_act, l.loss_alpha, logits, labels, dz, loss_sums, rows_per_group, (int)l.out_elems, groups, n->loss_partial, n->loss_ticket, s);
}
// A label mask of width mask_width for the net's loss (b2g_loss): 1 (per example / pixel) or the loss columns (per output)
static int32_t check_loss_mask(const b2g_net* n, int mask_width) {
  const LayerRT& l = n->L.back(); const int cols = loss_cols(l);
  if (mask_width != 1 && mask_width != cols) return fail(B2G_ERR_SHAPE, "label mask width %d: 1 or %d", mask_width, cols);
  if (mask_width > 1 && is_loss_layer(l) && l.d.loss == B2G_LOSS_MCXENT) return fail(B2G_ERR_UNSUPPORTED, "per-output masking for MCXENT + softmax is not supported");
  return 0;
}
// host rows [batch][chans x the map] -> dst on s: labels (chans = 0: the loss columns) or a label mask (chans = its width).  A CnnLossLayer's
// are NCHW: permuted to the engine's NHWC through `stage` when chans > 1 and the map is wider than one pixel (otherwise the orders coincide).
static int32_t upload_labels(b2g_net* n, const float* y, int batch, float* dst, float* stage, cudaStream_t s, int chans = 0) {
  const LayerRT& l = n->L.back(); const int cols = loss_cols(l); if (!chans) chans = cols;
  const size_t cnt = (size_t)batch * (std::max<size_t>(1, l.out_elems) / cols) * chans;
  if (l.d.type == B2G_LAYER_CNN_LOSS && chans > 1 && l.oh * l.ow > 1) {
    if (cnt > n->stage_floats) return fail(B2G_ERR_SHAPE, "labels larger than staging");
    CU(cudaMemcpyAsync(stage, y, sizeof(float) * cnt, cudaMemcpyHostToDevice, s));
    k_nchw_f32_to_nhwc(PREC_F32, stage, dst, batch, chans, l.oh * l.ow, s);
    return 0;
  }
  CU(cudaMemcpyAsync(dst, y, sizeof(float) * cnt, cudaMemcpyHostToDevice, s));
  return 0;
}
// The score's regularization sums L1 and L2 (b2g_regularization): one launch per term that has a non-zero coefficient, copied back on the
// net's stream (complete at its next synchronization); a term without one stays 0 and launches nothing
static int32_t net_reg_sums(b2g_net* n, double* l1, double* l2) {
  cudaStream_t s = n->ctx->stream;
  const int nr = (int)n->reg_seg.size();
  if (n->n_l2) { k_sumsq_segments(n->params, n->reg_off_dev, n->reg_len_dev, n->reg_l2c_dev, nr, n->reg_dev, s); CU(cudaMemcpyAsync(l2, n->reg_dev, sizeof(double), cudaMemcpyDeviceToHost, s)); }
  if (n->n_l1) { k_sumabs_segments(n->params, n->reg_off_dev, n->reg_len_dev, n->reg_l1c_dev, nr, n->reg_dev + 1, s); CU(cudaMemcpyAsync(l1, n->reg_dev + 1, sizeof(double), cudaMemcpyDeviceToHost, s)); }
  return 0;
}
static int32_t train_pass(b2g_net* n, const float* x, const float* y, int batch, bool do_update, float* score, const float* mask = nullptr, int mask_width = 0) {
  cudaStream_t s = n->ctx->stream;
  if (batch < 1 || batch > n->max_rows) return fail(B2G_ERR_SHAPE, "batch %d outside [1,%d]", batch, n->max_rows);
  int lt = n->L.back().d.type;
  if (lt != B2G_LAYER_OUTPUT && lt != B2G_LAYER_LOSS && lt != B2G_LAYER_CNN_LOSS) return fail(B2G_ERR_UNSUPPORTED, "fit needs a net ending in OutputLayer/LossLayer/CnnLossLayer");
  B2(upload_input(n, x, batch, n->input));
  B2(upload_labels(n, y, batch, n->labels_dev, n->stage_f32, s));
  if (mask) { B2(check_loss_mask(n, mask_width)); B2(upload_labels(n, mask, batch, n->mask_dev, n->stage_f32, s, mask_width)); }
  CU(cudaMemsetAsync(n->grads, 0, sizeof(float) * n->n_params, s));
  const void* logits = nullptr; FwdOpts o{batch, 1, true, true, nullptr};
  B2(net_forward(n, n->input, o, &logits));
  net_loss(n, logits, n->labels_dev, n->epsA, n->loss_dev, batch, 1, mask ? n->mask_dev : nullptr, mask_width);
  B2(net_backward(n, n->input, n->epsA, batch, 1, true, false, /*allreduce_follows=*/do_update && !score));
  if (score) {
    double l2 = 0.0, l1 = 0.0; float ls = 0.f;
    B2(net_reg_sums(n, &l1, &l2));
    CU(cudaMemcpyAsync(&ls, n->loss_dev, sizeof(float), cudaMemcpyDeviceToHost, s)); CU(cudaStreamSynchronize(s));
    *score = ls / batch + (float)(l2 + l1);
  }
  if (do_update) { B2(net_allreduce_grads(n)); B2(net_update(n, batch)); }
  return 0;
}
extern "C" int32_t b2g_net_compute_gradient_and_score(b2g_net* n, const float* x, const float* y, int32_t batch, float* score) {
  if (!n || !x || !y) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device)); B2(train_pass(n, x, y, batch, false, score)); CU(cudaStreamSynchronize(n->ctx->stream)); return 0;
}
extern "C" int32_t b2g_net_fit(b2g_net* n, const float* x, const float* y, int32_t batch, float* score) {
  if (!n || !x || !y) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device)); B2(train_pass(n, x, y, batch, true, score)); CU(cudaStreamSynchronize(n->ctx->stream)); return 0;
}
extern "C" int32_t b2g_net_compute_gradient_and_score_masked(b2g_net* n, const float* x, const float* y, int32_t batch, float* score, const float* mask, int32_t mask_width) {
  if (!n || !x || !y) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device)); B2(train_pass(n, x, y, batch, false, score, mask, mask_width)); CU(cudaStreamSynchronize(n->ctx->stream)); return 0;
}
extern "C" int32_t b2g_net_fit_masked(b2g_net* n, const float* x, const float* y, int32_t batch, float* score, const float* mask, int32_t mask_width) {
  if (!n || !x || !y) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device)); B2(train_pass(n, x, y, batch, true, score, mask, mask_width)); CU(cudaStreamSynchronize(n->ctx->stream)); return 0;
}
extern "C" int32_t b2g_net_loss_columns(b2g_net* n, int32_t* cols) {
  if (!n || !cols) return fail(B2G_ERR_ARG, "null");
  *cols = loss_cols(n->L.back()); return 0;
}
extern "C" int32_t b2g_net_set_loss_weights(b2g_net* n, const char* layer, const float* w, int32_t count) {
  if (!n) return fail(B2G_ERR_ARG, "null");
  const LayerRT& l = n->L.back();
  if (!w && !layer) { if (n->loss_w_on) { n->loss_w_on = false; ++n->settings_gen; } return 0; }     // clearing: a no-op on any net without weights
  if (layer && strncmp(l.d.name, layer, B2G_NAME_LEN)) return fail(B2G_ERR_ARG, "layer '%s' is not the net's loss layer", layer);
  if (!is_loss_layer(l)) return fail(B2G_ERR_ARG, "loss weights need a net ending in OutputLayer / LossLayer / CnnLossLayer");
  if (!w) { if (n->loss_w_on) { n->loss_w_on = false; ++n->settings_gen; } return 0; }
  CU(cudaSetDevice(n->ctx->device));
  if (l.d.loss == B2G_LOSS_HINGE || l.d.loss == B2G_LOSS_SQUARED_HINGE || l.d.loss == B2G_LOSS_WASSERSTEIN)
    return fail(B2G_ERR_UNSUPPORTED, "loss %d takes no per-output weights", l.d.loss);
  if (count != loss_cols(l)) return fail(B2G_ERR_SHAPE, "%d loss weights for %d outputs", count, loss_cols(l));
  for (int j = 0; j < count; ++j) if (!isfinite(w[j])) return fail(B2G_ERR_ARG, "loss weight %d is not finite", j);
  CU(cudaMemcpyAsync(n->loss_w, w, sizeof(float) * count, cudaMemcpyHostToDevice, n->ctx->stream)); CU(cudaStreamSynchronize(n->ctx->stream));
  n->loss_w_on = true; ++n->settings_gen;      // a captured step holds which instantiation the loss launches: re-capture
  return 0;
}
extern "C" int32_t b2g_net_get_input_gradient(b2g_net* n, int32_t batch, float* host) {
  if (!n || !host) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device));
  if (!n->input_grad) return fail(B2G_ERR_ARG, "no input gradient available (run b2g_gan_step or a backward that requests it)");
  return download_act(n, n->input_grad, batch, n->cfg.in_c, n->cfg.in_h * n->cfg.in_w, host);
}

// ------------------------------------------------------------------ the fused GAN step -------------------
struct b2g_gan {
  b2g_net *G = nullptr, *D = nullptr; b2g_gan_config cfg{};
  int N = 0;                              // per-step batch (D sees 2N)
  void *z_d = nullptr, *z_g = nullptr;    // T [N][z]
  float *y_d = nullptr, *y_g = nullptr;   // [2N][oe] = y_real | y_fake ; [N][oe]  (oe = the discriminator's outputs per example, NHWC)
  float* loss_dev = nullptr;              // [4]: d_real_sum, d_fake_sum, g_sum
  float* stage = nullptr; size_t stage_floats = 0;
  cudaGraph_t graph = nullptr, graph1 = nullptr; cudaGraphExec_t exec = nullptr, exec1 = nullptr; int graph_batch = 0; uint64_t graph_launches = 0, graph_simt_g = 0, graph_simt_d = 0;
  uint64_t graph_settings_g = 0, graph_settings_d = 0;   // the nets' updater settings generations the captured graph was made with
  float *m_d = nullptr, *m_g = nullptr;   // label masks (b2g_gan_set_label_masks): [2N][mw x map] = m_real | m_fake ; [N][mw x map]; allocated once
  int mask_width = 0, mask_batch = 0, graph_mask_width = 0;   // 0: no masks; graph_mask_width: what the captured graph was made with
  cudaEvent_t ev0 = nullptr, ev1 = nullptr; float last_ms = 0.f; int last_batch = 1; bool nccl_warm = false;
  cudaStream_t copy_stream = nullptr; cudaEvent_t ev_x = nullptr; bool ev1_valid = false;   // x_real's H2D runs under the generator's forward
  std::vector<void*> allocs;
};

// part 1: x_fake = gen.output(z_d) -- needs nothing from the host but z_d.  part 2: everything that touches x_real.
// They are two graphs so that the copy-stream event of x_real's H2D can be waited on between them (a captured stream may not
// wait on work outside its capture).
static int32_t gan_step_part1(b2g_gan* g, int N) {
  b2g_net *G = g->G, *D = g->D;
  const size_t ts = prec_size(D->prec);
  void* fake_dst = (char*)D->input + ts * (size_t)N * D->in_elems;
  FwdOpts og{N, 1, g->cfg.fake_bn_train != 0, false, fake_dst};
  return net_forward(G, g->z_d, og, nullptr);
}
static int32_t gan_step_part2(b2g_gan* g, int N) {
  b2g_net *G = g->G, *D = g->D; cudaStream_t s = G->ctx->stream;
  // 1. (part 1) x_fake = gen.output(z_d) (J:420) was written straight into the second half of D's input batch.
  // x_real arrived (and was converted to the device layout) on the copy stream meanwhile; only the discriminator needs it
  // 3a (hoisted). The generator's train-mode forward on z_g depends only on G's parameters, which the D step does not touch: it runs on a
  // second stream -- on one GPU underneath the whole D step; with a communicator underneath the D gradient all-reduce + updater, where the
  // SMs would otherwise idle on the network.
  // (with sync_bn the generator's BatchNorm all-reduces must keep one issue order with the discriminator's on every rank: no hoisting)
  cudaStream_t s3 = (G->sync_bn || D->sync_bn) ? s : G->ctx->side2;
  const bool under_allreduce = G->ctx->comm && G->ctx->world > 1 && D->grad_allreduce && s3 != s;
  const void* xg = nullptr;
  auto hoisted_g_forward = [&]() -> int32_t {
    CU(cudaEventRecord(G->ctx->ev_a, s)); CU(cudaStreamWaitEvent(s3, G->ctx->ev_a, 0));
    CU(cudaMemsetAsync(G->grads, 0, sizeof(float) * G->n_params, s3));
    FwdOpts og2{N, 1, true, true, nullptr};
    G->fwd_stream = s3; int32_t rg = net_forward(G, g->z_g, og2, &xg); G->fwd_stream = nullptr; B2(rg);
    CU(cudaEventRecord(G->ctx->ev_b, s3)); return 0;
  };
  if (!under_allreduce) B2(hoisted_g_forward());
  // 2. D update on (x_real, y_real) | (x_fake, y_fake): two BN groups, one batched pass (J:414-426)
  CU(cudaMemsetAsync(D->grads, 0, sizeof(float) * D->n_params, s));
  const void* logits = nullptr; FwdOpts od{2 * N, 2, true, true, nullptr};
  B2(net_forward(D, D->input, od, &logits));
  net_loss(D, logits, g->y_d, D->epsA, g->loss_dev, N, 2, g->mask_width ? g->m_d : nullptr, g->mask_width);
  B2(net_backward(D, D->input, D->epsA, 2 * N, 2, true, false, /*allreduce_follows=*/true));
  if (under_allreduce) B2(hoisted_g_forward());
  B2(net_allreduce_grads(D));
  B2(net_update(D, 2 * N));
  // 3. G update through D on (z_g, y_gen) (J:465-471); D's parameters / running stats / updater state untouched
  CU(cudaStreamWaitEvent(s, G->ctx->ev_b, 0));
  // a scheduled DropoutLayer of D reads G's counters here: this pass belongs to the generator's fit (the stacked gan graph counts its own)
  FwdOpts od2{N, 1, true, false, nullptr, G->step_dev, G->epoch_dev};
  B2(net_forward(D, xg, od2, &logits));
  net_loss(D, logits, g->y_g, D->epsA, g->loss_dev + 2, N, 1, g->mask_width ? g->m_g : nullptr, g->mask_width);
  // the generator's output activation (tanh) is differentiated inside D's last input-gradient kernel when that kernel can (EPI_ACTBWD)
  TcEpi ga{}; const LayerRT& gl = G->L.back(); bool ga_done = false;
  const bool ga_can = gl.has_gemm() && gl.d.act != B2G_ACT_IDENTITY && gl.d.type != B2G_LAYER_OUTPUT;
  if (ga_can) { ga.mode = EPI_ACTBWD; ga.aux = (const __nv_bfloat16*)xg; ga.act = gl.d.act; ga.alpha = gl.d.act_alpha; }
  B2(net_backward(D, xg, D->epsA, N, 1, false, true, false, ga_can ? &ga : nullptr, &ga_done));
  B2(net_backward(G, g->z_g, D->input_grad, N, 1, true, false, /*allreduce_follows=*/true, nullptr, nullptr, ga_done));
  B2(net_allreduce_grads(G));
  B2(net_update(G, N));
  return 0;
}

extern "C" int32_t b2g_gan_create(b2g_net* gen, b2g_net* dis, const b2g_gan_config* cfg, b2g_gan** out) {
  if (!gen || !dis || !out) return fail(B2G_ERR_ARG, "null");
  if (gen->ctx != dis->ctx) return fail(B2G_ERR_ARG, "generator and discriminator live on different contexts");
  if (gen->prec != dis->prec) return fail(B2G_ERR_ARG, "generator and discriminator use different precisions");
  if (gen->L.back().out_elems != dis->in_elems) return fail(B2G_ERR_SHAPE, "generator output (%zu) != discriminator input (%zu)", gen->L.back().out_elems, dis->in_elems);
  if (gen->L.back().out_alias || gen->L.back().d.type == B2G_LAYER_DROPOUT) return fail(B2G_ERR_UNSUPPORTED, "generator must end in a layer that owns its output");
  {  // one output per example; XENT or a loss of codes 2-8 (the labels the caller uploads choose the objective)
    const LayerRT& dl = dis->L.back();
    const bool lossy = dl.d.type == B2G_LAYER_OUTPUT || dl.d.type == B2G_LAYER_LOSS;
    if (dl.d.type == B2G_LAYER_CNN_LOSS && dl.d.loss == B2G_LOSS_MCXENT)
      return fail(B2G_ERR_UNSUPPORTED, "the adversarial step needs a CnnLossLayer discriminator with XENT or a loss of codes 2-8 (not MCXENT: one label per patch)");
    if (lossy && dl.d.loss == B2G_LOSS_MCXENT) return fail(B2G_ERR_UNSUPPORTED, "the adversarial step needs a discriminator with one output per example (not MCXENT)");
    if (lossy && dl.out_elems != 1) return fail(B2G_ERR_UNSUPPORTED, "the adversarial step needs a discriminator with one output per example, not %zu", dl.out_elems);
  }
  if (dis->cfg.bn_groups < 2 || dis->max_rows < 2) return fail(B2G_ERR_ARG, "discriminator must be created with bn_groups>=2 and max_batch = 2*N");
  int N = std::min(gen->max_rows, dis->max_rows / 2);
  CU(cudaSetDevice(gen->ctx->device));
  b2g_gan* g = new b2g_gan(); g->G = gen; g->D = dis; if (cfg) g->cfg = *cfg; g->N = N;
  const size_t ts = prec_size(gen->prec);
  auto al = [&](void** p, size_t bytes) -> int32_t { cudaError_t e = cudaMalloc(p, bytes ? bytes : 16); if (e != cudaSuccess) return fail(B2G_ERR_OOM, "cudaMalloc: %s", cudaGetErrorString(e)); g->allocs.push_back(*p); return 0; };
  int32_t r = al(&g->z_d, ts * N * gen->in_elems); if (!r) r = al(&g->z_g, ts * N * gen->in_elems);
  const size_t oe = dis->L.back().out_elems;      // labels per example: 1, or a CnnLossLayer discriminator's patch map
  if (!r) r = al((void**)&g->y_d, sizeof(float) * 2 * N * oe); if (!r) r = al((void**)&g->y_g, sizeof(float) * N * oe); if (!r) r = al((void**)&g->loss_dev, sizeof(float) * 4);
  g->stage_floats = (size_t)N * std::max(dis->in_elems, gen->in_elems); if (!r) r = al((void**)&g->stage, sizeof(float) * g->stage_floats);
  if (!r) { if (cudaEventCreate(&g->ev0) != cudaSuccess || cudaEventCreate(&g->ev1) != cudaSuccess || cudaEventCreateWithFlags(&g->ev_x, cudaEventDisableTiming) != cudaSuccess ||
                cudaStreamCreateWithFlags(&g->copy_stream, cudaStreamNonBlocking) != cudaSuccess) r = fail(B2G_ERR_CUDA, "cudaEventCreate failed"); }
  if (r) { for (void* p : g->allocs) cudaFree(p); delete g; return r; }
  *out = g; return 0;
}
extern "C" int32_t b2g_gan_destroy(b2g_gan* g) {
  if (!g) return 0; cudaSetDevice(g->G->ctx->device); cudaStreamSynchronize(g->G->ctx->stream);
  if (g->exec) cudaGraphExecDestroy(g->exec); if (g->graph) cudaGraphDestroy(g->graph); if (g->exec1) cudaGraphExecDestroy(g->exec1); if (g->graph1) cudaGraphDestroy(g->graph1);
  if (g->ev0) cudaEventDestroy(g->ev0); if (g->ev1) cudaEventDestroy(g->ev1); if (g->ev_x) cudaEventDestroy(g->ev_x); if (g->copy_stream) { cudaStreamSynchronize(g->copy_stream); cudaStreamDestroy(g->copy_stream); }
  for (void* p : g->allocs) cudaFree(p); delete g; return 0;
}
extern "C" int32_t b2g_gan_upload(b2g_gan* g, const float* x_real, const float* z_d, const float* z_g, const float* y_real, const float* y_fake, const float* y_gen, int32_t batch) {
  if (!g || !x_real || !z_d || !z_g || !y_real || !y_fake || !y_gen) return fail(B2G_ERR_ARG, "null");
  if (batch < 1 || batch > g->N) return fail(B2G_ERR_SHAPE, "batch %d outside [1,%d]", batch, g->N);
  b2g_net *G = g->G, *D = g->D; cudaStream_t s = G->ctx->stream; CU(cudaSetDevice(G->ctx->device));
  size_t nx = (size_t)batch * D->in_elems, nz = (size_t)batch * G->in_elems;
  // x_real (the only large input) goes over a separate copy stream, where it is also converted to the device layout;
  // the staging buffer is free once the previous step's conversion has run (ev1 marks the end of that step)
  if (g->ev1_valid) CU(cudaStreamWaitEvent(g->copy_stream, g->ev1, 0));
  CU(cudaMemcpyAsync(g->stage, x_real, sizeof(float) * nx, cudaMemcpyHostToDevice, g->copy_stream));
  k_nchw_f32_to_nhwc(D->prec, g->stage, D->input, batch, D->cfg.in_c, D->cfg.in_h * D->cfg.in_w, g->copy_stream);     // NCHW fp32 -> NHWC in the net's type, off the step's critical path
  CU(cudaEventRecord(g->ev_x, g->copy_stream));
  CU(cudaMemcpyAsync(G->stage_f32, z_d, sizeof(float) * nz, cudaMemcpyHostToDevice, s));
  k_nchw_f32_to_nhwc(G->prec, G->stage_f32, g->z_d, batch, G->cfg.in_c, G->cfg.in_h * G->cfg.in_w, s);
  CU(cudaMemcpyAsync(D->stage_f32, z_g, sizeof(float) * nz, cudaMemcpyHostToDevice, s));
  k_nchw_f32_to_nhwc(G->prec, D->stage_f32, g->z_g, batch, G->cfg.in_c, G->cfg.in_h * G->cfg.in_w, s);
  // [batch][oe] each (NCHW for a CnnLossLayer; D's staging buffer is free again once z_g's conversion above has run on s)
  const size_t oe = D->L.back().out_elems;
  B2(upload_labels(D, y_real, batch, g->y_d, D->stage_f32, s));
  B2(upload_labels(D, y_fake, batch, g->y_d + (size_t)batch * oe, D->stage_f32, s));
  B2(upload_labels(D, y_gen, batch, g->y_g, D->stage_f32, s));
  CHECK_KERNELS();
  return 0;
}
extern "C" int32_t b2g_gan_step_resident(b2g_gan* g, int32_t batch) {
  if (!g) return fail(B2G_ERR_ARG, "null"); if (batch < 1 || batch > g->N) return fail(B2G_ERR_SHAPE, "batch %d outside [1,%d]", batch, g->N);
  b2g_ctx* c = g->G->ctx; cudaStream_t s = c->stream; CU(cudaSetDevice(c->device));
  // With a communicator the first step runs eagerly (NCCL connects lazily on its first collective); after that the whole step,
  // the two ncclAllReduce calls included, is captured and replayed like the single-GPU one.  B2G_GRAPH_NCCL=0 keeps it eager.
  static int graph_nccl = -1; if (graph_nccl < 0) { const char* e = getenv("B2G_GRAPH_NCCL"); graph_nccl = (e && e[0] == '0') ? 0 : 1; }
  bool use_graph = g->cfg.use_cuda_graph && (!c->comm || (graph_nccl && g->nccl_warm));
  if (c->comm) g->nccl_warm = true;
  if (g->mask_width && batch != g->mask_batch) return fail(B2G_ERR_SHAPE, "step batch %d, label masks set for %d", batch, g->mask_batch);
  g->last_batch = batch;
  CU(cudaEventRecord(g->ev0, s));
  if (!use_graph) { B2(gan_step_part1(g, batch)); CU(cudaStreamWaitEvent(s, g->ev_x, 0)); B2(gan_step_part2(g, batch)); }
  else {
    if (!g->exec || g->graph_batch != batch || g->graph_settings_g != g->G->settings_gen || g->graph_settings_d != g->D->settings_gen ||
        g->graph_mask_width != g->mask_width) {
      if (g->exec) { cudaGraphExecDestroy(g->exec); g->exec = nullptr; } if (g->graph) { cudaGraphDestroy(g->graph); g->graph = nullptr; }
      if (g->exec1) { cudaGraphExecDestroy(g->exec1); g->exec1 = nullptr; } if (g->graph1) { cudaGraphDestroy(g->graph1); g->graph1 = nullptr; }
      uint64_t before = g_launch_count; const uint64_t sg0 = g->G->simt_gemm_calls, sd0 = g->D->simt_gemm_calls;
      CU(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
      int32_t r = gan_step_part1(g, batch);
      cudaError_t e = cudaStreamEndCapture(s, &g->graph1);
      if (r) return r; if (e != cudaSuccess) return fail(B2G_ERR_CUDA, "graph capture (generator forward): %s", cudaGetErrorString(e));
      CU(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
      r = gan_step_part2(g, batch);
      e = cudaStreamEndCapture(s, &g->graph);
      g->graph_launches = g_launch_count - before; g_launch_count = before;
      g->graph_simt_g = g->G->simt_gemm_calls - sg0; g->graph_simt_d = g->D->simt_gemm_calls - sd0; g->G->simt_gemm_calls = sg0; g->D->simt_gemm_calls = sd0;
      if (r) return r; if (e != cudaSuccess) return fail(B2G_ERR_CUDA, "graph capture: %s", cudaGetErrorString(e));
      CU(cudaGraphInstantiate(&g->exec1, g->graph1, 0)); CU(cudaGraphInstantiate(&g->exec, g->graph, 0)); g->graph_batch = batch;
      g->graph_settings_g = g->G->settings_gen; g->graph_settings_d = g->D->settings_gen; g->graph_mask_width = g->mask_width;
    }
    CU(cudaGraphLaunch(g->exec1, s));
    CU(cudaStreamWaitEvent(s, g->ev_x, 0));
    CU(cudaGraphLaunch(g->exec, s)); g_launch_count += g->graph_launches; g->G->simt_gemm_calls += g->graph_simt_g; g->D->simt_gemm_calls += g->graph_simt_d;
  }
  CU(cudaEventRecord(g->ev1, s)); g->ev1_valid = true;
  return 0;
}
extern "C" int32_t b2g_gan_set_label_masks(b2g_gan* g, const float* m_real, const float* m_fake, const float* m_gen, int32_t mask_width, int32_t batch) {
  if (!g) return fail(B2G_ERR_ARG, "null");
  if (!m_real && !m_fake && !m_gen) { g->mask_width = 0; g->mask_batch = 0; return 0; }
  if (!m_real || !m_fake || !m_gen) return fail(B2G_ERR_ARG, "label masks: all three or none");
  if (batch < 1 || batch > g->N) return fail(B2G_ERR_SHAPE, "batch %d outside [1,%d]", batch, g->N);
  b2g_net* D = g->D; cudaStream_t s = g->G->ctx->stream; CU(cudaSetDevice(D->ctx->device));
  B2(check_loss_mask(D, mask_width));
  const size_t oe = D->L.back().out_elems;
  if (!g->m_d) {
    for (float** p : {&g->m_d, &g->m_g}) {
      cudaError_t e = cudaMalloc((void**)p, sizeof(float) * (p == &g->m_d ? 2 : 1) * g->N * std::max<size_t>(1, oe));
      if (e != cudaSuccess) return fail(B2G_ERR_OOM, "cudaMalloc: %s", cudaGetErrorString(e));
      g->allocs.push_back(*p);
    }
  }
  // the previous step may still read the masks (and D's staging buffer): the copies wait for it on the step's stream
  const size_t per = (size_t)batch * (std::max<size_t>(1, oe) / loss_cols(D->L.back())) * mask_width;
  B2(upload_labels(D, m_real, batch, g->m_d, D->stage_f32, s, mask_width));
  B2(upload_labels(D, m_fake, batch, g->m_d + per, D->stage_f32, s, mask_width));
  B2(upload_labels(D, m_gen, batch, g->m_g, D->stage_f32, s, mask_width));
  CU(cudaStreamSynchronize(s));
  g->mask_width = mask_width; g->mask_batch = batch;
  return 0;
}
extern "C" int32_t b2g_gan_read_losses(b2g_gan* g, float* losses) {
  if (!g || !losses) return fail(B2G_ERR_ARG, "null"); cudaStream_t s = g->G->ctx->stream; CU(cudaSetDevice(g->G->ctx->device));
  float h[4]; CU(cudaMemcpyAsync(h, g->loss_dev, sizeof(h), cudaMemcpyDeviceToHost, s)); CU(cudaStreamSynchronize(s));
  int N = g->last_batch;
  losses[0] = h[0] / N; losses[1] = h[1] / N; losses[2] = h[2] / N; return 0;
}
extern "C" int32_t b2g_gan_last_step_ms(b2g_gan* g, float* ms) {
  if (!g || !ms) return fail(B2G_ERR_ARG, "null"); CU(cudaEventSynchronize(g->ev1)); CU(cudaEventElapsedTime(ms, g->ev0, g->ev1)); return 0;
}
extern "C" int32_t b2g_gan_step(b2g_gan* g, const float* x_real, const float* z_d, const float* z_g, const float* y_real, const float* y_fake, const float* y_gen, int32_t batch, float* losses) {
  B2(b2g_gan_upload(g, x_real, z_d, z_g, y_real, y_fake, y_gen, batch));
  B2(b2g_gan_step_resident(g, batch));
  if (losses) return b2g_gan_read_losses(g, losses);
  return 0;
}

// ------------------------------------------------------------------ iteration counter / dispatch evidence ----
// The updater's iteration counter (Adam's t, DL4J's BaseMultiLayerUpdater iteration) lives on the device so that CUDA graphs replay;
// a checkpoint must carry it, or a resumed Adam restarts its bias correction at t = 1 with warm moments.
extern "C" int32_t b2g_net_get_iteration(b2g_net* n, int64_t* out) {
  if (!n || !out) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device));
  int v = 0; CU(cudaMemcpyAsync(&v, n->step_dev, sizeof(int), cudaMemcpyDeviceToHost, n->ctx->stream)); CU(cudaStreamSynchronize(n->ctx->stream)); *out = v; return 0;
}
extern "C" int32_t b2g_net_set_iteration(b2g_net* n, int64_t it) {
  if (!n || it < 0 || it > 0x7fffffff) return fail(B2G_ERR_ARG, "bad iteration"); CU(cudaSetDevice(n->ctx->device));
  int v = (int)it; CU(cudaMemcpyAsync(n->step_dev, &v, sizeof(int), cudaMemcpyHostToDevice, n->ctx->stream)); CU(cudaStreamSynchronize(n->ctx->stream)); return 0;
}
// The dropout pass counter P lives on the device for the same reason; a checkpoint carries it so that a resumed run draws the masks of an
// uninterrupted one.
extern "C" int32_t b2g_net_get_dropout_pass(b2g_net* n, int64_t* out) {
  if (!n || !out) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device));
  unsigned long long v = 0; CU(cudaMemcpyAsync(&v, n->drop_pass, sizeof(v), cudaMemcpyDeviceToHost, n->ctx->stream)); CU(cudaStreamSynchronize(n->ctx->stream)); *out = (int64_t)v; return 0;
}
extern "C" int32_t b2g_net_set_dropout_pass(b2g_net* n, int64_t pass) {
  if (!n || pass < 0) return fail(B2G_ERR_ARG, "bad dropout pass"); CU(cudaSetDevice(n->ctx->device));
  unsigned long long v = (unsigned long long)pass; CU(cudaMemcpyAsync(n->drop_pass, &v, sizeof(v), cudaMemcpyHostToDevice, n->ctx->stream)); CU(cudaStreamSynchronize(n->ctx->stream)); return 0;
}
extern "C" int32_t b2g_net_set_gradient_normalization(b2g_net* n, int32_t mode, float threshold) {
  if (!n) return fail(B2G_ERR_ARG, "null");
  if (mode == B2G_GN_CLIP_ELEMENTWISE) return fail(B2G_ERR_ARG, "ClipElementWiseAbsoluteValue is b2g_net_config.grad_clip, set when the net is created");
  if (mode != B2G_GN_NONE && mode != B2G_GN_RENORM_L2_LAYER && mode != B2G_GN_RENORM_L2_PARAM && mode != B2G_GN_CLIP_L2_LAYER && mode != B2G_GN_CLIP_L2_PARAM)
    return fail(B2G_ERR_ARG, "unknown gradient normalization %d", mode);
  if (mode != B2G_GN_NONE && n->cfg.grad_clip > 0.f)
    return fail(B2G_ERR_ARG, "the net was created with grad_clip %g (ClipElementWiseAbsoluteValue): one gradient normalization per layer", (double)n->cfg.grad_clip);
  const bool clip = mode == B2G_GN_CLIP_L2_LAYER || mode == B2G_GN_CLIP_L2_PARAM;
  if (clip && !(threshold > 0.f && isfinite(threshold))) return fail(B2G_ERR_ARG, "gradient normalization threshold %g: the clip modes need a finite threshold > 0", (double)threshold);
  if (!clip) threshold = 1.0f;      // the renormalize modes ignore it
  if (mode != n->gn_mode || threshold != n->gn_threshold) { n->gn_mode = mode; n->gn_threshold = threshold; ++n->settings_gen; }
  return 0;
}

// ------------------------------------------------------------------ weight constraints --------------------
// A parameter's internal axes [A][kH][kW][B] and where its DL4J dimensions land on them (b2g_constraint): conv W [nOut, nIn, kH, kW] and deconv
// W [nIn, nOut, kH, kW] are [A][taps][B] with dims (0, 1, 2, 3) -> (A, B, kH, kW); dense / output W [nIn, nOut] is [nOut][nIn] = [A][B] with
// dims (0, 1) -> (B, A); a [1, n] vector is [1][n] with dims (0, 1) -> (A, B).
struct ConAxes { int ax[4]; int map[4]; int rank; };
static ConAxes con_axes(const b2g_net* n, const ParamRef& r, const char* param) {
  const LayerRT& l = n->L[r.layer];
  ConAxes c{};
  if (!strcmp(param, "W") && (l.d.type == B2G_LAYER_CONV2D || l.d.type == B2G_LAYER_DECONV2D)) c = ConAxes{{l.wA, l.d.k_h, l.d.k_w, l.wB}, {0, 3, 1, 2}, 4};
  else if (!strcmp(param, "W")) c = ConAxes{{l.wA, 1, 1, l.wB}, {3, 0, 0, 0}, 2};
  else c = ConAxes{{1, 1, 1, (int)r.len}, {0, 3, 0, 0}, 2};
  return c;
}
// Rebuilds the job plan from n->con (include/b200gan.h for the rules, kernels.h ConJob for the paths).  Frozen layers' tensors are skipped.
static int32_t net_build_constraints(b2g_net* n) {
  cudaStream_t s = n->ctx->stream;
  CU(cudaStreamSynchronize(s));                  // nothing in flight reads the old plan
  cudaFree(n->con_jobs); cudaFree(n->con_partial); cudaFree(n->con_mult);
  n->con_jobs = nullptr; n->con_partial = nullptr; n->con_mult = nullptr; n->con_rounds.clear();
  std::vector<ConJob> jobs; int64_t parts = 0, mults = 0;
  for (int round = 0; round < 4; ++round) {
    std::vector<ConJob> one, two;
    for (const auto& t : n->con) {
      if ((int)t.list.size() <= round || n->L[t.layer].d.frozen) continue;     // FrozenLayer: no update, no constraint
      const b2g_constraint& k = t.list[round];
      const LayerRT& l = n->L[t.layer];
      ParamRef r; B2(find_param(n, l.d.name, t.param, &r));
      const ConAxes a = con_axes(n, r, t.param);
      bool red[4] = {false, false, false, false};
      for (int d = 0; d < a.rank; ++d) if (!k.dims_mask || (k.dims_mask >> d) & 1) red[a.map[d]] = true;
      // [K0][R0][K1][R1][K2]: the runs of kept / reduced axes (size-1 axes dropped); a kept innermost run after a reduced one is K2 (strided
      // groups, lane per group), the other runs fill K0, R0, K1, R1 in order
      int run_f[4], run_n[4], nr = 0;
      for (int x = 0; x < 4; ++x) {
        if (a.ax[x] == 1) continue;
        const int f = red[x] ? 1 : 0;
        if (nr && run_f[nr - 1] == f) run_n[nr - 1] *= a.ax[x];
        else { run_f[nr] = f; run_n[nr] = a.ax[x]; ++nr; }
      }
      int slot[5] = {1, 1, 1, 1, 1};
      if (nr >= 2 && run_f[nr - 1] == 0) slot[4] = run_n[--nr];
      for (int i = 0, si = -1; i < nr; ++i) { si = si < 0 ? run_f[i] : si + 1; slot[si] = run_n[i]; }
      ConJob j{};
      const bool w = !strcmp(t.param, "W");
      j.sg.off = r.off; j.sg.len = r.len; j.sg.off_bf = (w && l.off_W_bf >= 0) ? l.off_W_bf : -1; j.sg.off_ps = (w && l.off_Wps_bf >= 0) ? l.off_Wps_bf : -1;
      j.sg.ps_O = l.geom.O; j.sg.ps_C = l.geom.C;
      j.kind = k.kind; j.max_norm = k.max_norm; j.min_norm = k.min_norm; j.rate = k.kind == B2G_CONSTRAINT_MIN_MAX_NORM ? k.rate : 1.0;
      j.K0 = slot[0]; j.R0 = slot[1]; j.K1 = slot[2]; j.R1 = slot[3]; j.K2 = slot[4]; j.groups = j.K0 * j.K1 * j.K2; j.R = j.R0 * j.R1;
      j.chunks = 1;
      if (k.kind == B2G_CONSTRAINT_NON_NEGATIVE) { j.path = CON_ELEMWISE; j.blocks = (int)((r.len + CON_CHUNK - 1) / CON_CHUNK); one.push_back(j); }
      else if (j.K2 == 1 && j.R <= CON_CHUNK) { j.path = CON_ONEPASS; j.blocks = j.groups; one.push_back(j); }
      else {
        j.path = CON_TWOPASS;
        if (j.K2 == 1) { j.chunks = (j.R + CON_CHUNK - 1) / CON_CHUNK; j.blocks = j.groups * j.chunks; }
        else { j.chunks = (j.R + CON_SCHUNK - 1) / CON_SCHUNK; j.blocks = j.K0 * j.K1 * ((j.K2 + 31) / 32) * j.chunks; }
        j.blocks2 = (int)((r.len + CON_CHUNK - 1) / CON_CHUNK);
        j.part_begin = parts; parts += (int64_t)j.groups * j.chunks; j.mult_begin = mults; mults += j.groups;
        two.push_back(j);
      }
    }
    if (one.empty() && two.empty()) break;
    b2g_net::ConRound rd{};
    rd.j0 = (int)jobs.size();
    for (auto& j : one) { j.blk_begin = rd.onepass_blocks; rd.onepass_blocks += j.blocks; jobs.push_back(j); }
    rd.j1 = rd.t0 = (int)jobs.size();
    for (auto& j : two) { j.blk_begin = rd.norm_blocks; rd.norm_blocks += j.blocks; j.blk2_begin = rd.scale_blocks; rd.scale_blocks += j.blocks2; jobs.push_back(j); }
    rd.t1 = (int)jobs.size();
    n->con_rounds.push_back(rd);
  }
  if (!jobs.empty()) {
    CU(cudaMalloc(&n->con_jobs, sizeof(ConJob) * jobs.size()));
    CU(cudaMalloc(&n->con_partial, sizeof(double) * std::max<int64_t>(1, parts))); CU(cudaMalloc(&n->con_mult, sizeof(float) * std::max<int64_t>(1, mults)));
    if (!n->con_ticket) { B2(dalloc(n, &n->con_ticket, sizeof(unsigned))); CU(cudaMemsetAsync(n->con_ticket, 0, sizeof(unsigned), s)); }
    CU(cudaMemcpyAsync(n->con_jobs, jobs.data(), sizeof(ConJob) * jobs.size(), cudaMemcpyHostToDevice, s));
    CU(cudaStreamSynchronize(s));
  }
  ++n->settings_gen;
  return 0;
}
extern "C" int32_t b2g_net_set_constraints(b2g_net* n, const char* layer, const char* param, const b2g_constraint* list, int32_t cnt) {
  if (!n || !layer || !param || cnt < 0 || (cnt > 0 && !list)) return fail(B2G_ERR_ARG, "b2g_net_set_constraints: null argument or negative count");
  if (cnt > 4) return fail(B2G_ERR_ARG, "%s.%s: %d constraints, at most 4 per tensor", layer, param, cnt);
  CU(cudaSetDevice(n->ctx->device));
  ParamRef r; B2(find_param(n, layer, param, &r));
  if (n->L[r.layer].d.type == B2G_LAYER_PRELU) return fail(B2G_ERR_ARG, "layer %s: constraints on a PReLU's slopes are not supported", layer);
  const ConAxes a = con_axes(n, r, param);
  for (int i = 0; i < cnt; ++i) {
    const b2g_constraint& k = list[i];
    if (k.kind < B2G_CONSTRAINT_MAX_NORM || k.kind > B2G_CONSTRAINT_NON_NEGATIVE) return fail(B2G_ERR_ARG, "%s.%s: unknown constraint kind %d", layer, param, k.kind);
    if (k.dims_mask < 0 || (k.dims_mask >> a.rank) != 0) return fail(B2G_ERR_ARG, "%s.%s: dims mask 0x%x outside the parameter's %d dimensions", layer, param, k.dims_mask, a.rank);
    const bool maxk = k.kind == B2G_CONSTRAINT_MAX_NORM || k.kind == B2G_CONSTRAINT_MIN_MAX_NORM, mink = k.kind == B2G_CONSTRAINT_MIN_MAX_NORM;
    if (maxk && !(std::isfinite(k.max_norm) && k.max_norm >= 0.0)) return fail(B2G_ERR_ARG, "%s.%s: max norm %g is not finite and >= 0", layer, param, k.max_norm);
    if (mink && !(std::isfinite(k.min_norm) && k.min_norm >= 0.0)) return fail(B2G_ERR_ARG, "%s.%s: min norm %g is not finite and >= 0", layer, param, k.min_norm);
    if (mink && k.min_norm > k.max_norm) return fail(B2G_ERR_ARG, "%s.%s: min norm %g > max norm %g", layer, param, k.min_norm, k.max_norm);
    if (mink && !(k.rate >= 0.0 && k.rate <= 1.0)) return fail(B2G_ERR_ARG, "%s.%s: rate %g outside [0, 1]", layer, param, k.rate);
  }
  size_t at = 0;
  while (at < n->con.size() && !(n->con[at].layer == r.layer && !strcmp(n->con[at].param, param))) ++at;
  if (at == n->con.size()) {
    if (!cnt) return 0;
    b2g_net::ConTensor t{}; t.layer = r.layer; snprintf(t.param, sizeof(t.param), "%s", param);
    n->con.push_back(t);
    std::sort(n->con.begin(), n->con.end(), [&](const b2g_net::ConTensor& x, const b2g_net::ConTensor& y) {
      ParamRef px, py; find_param(n, n->L[x.layer].d.name, x.param, &px); find_param(n, n->L[y.layer].d.name, y.param, &py); return px.off < py.off; });
    at = 0; while (!(n->con[at].layer == r.layer && !strcmp(n->con[at].param, param))) ++at;
  }
  if (cnt) n->con[at].list.assign(list, list + cnt); else n->con.erase(n->con.begin() + at);
  return net_build_constraints(n);
}
extern "C" int32_t b2g_net_apply_constraints(b2g_net* n) {
  if (!n) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device));
  net_launch_constraints(n, n->ctx->stream); CHECK_KERNELS();
  CU(cudaStreamSynchronize(n->ctx->stream)); return 0;
}

// ------------------------------------------------------------------ learning-rate schedules ---------------
// A layer has a learning rate when it is not frozen, has parameters and its updater is neither NoOp nor AdaDelta: when it owns an updater
// segment of another kind (frozen layers own no segments; a NoOp updater and BatchNorm mean/var make NoOp segments; AdaDelta has no learning
// rate).  The Python layer specs apply the same rule (engine.py layer_has_lr); b2g_net_get_learning_rate reads the layer's first such segment.
static int lr_segment(const b2g_net* n, int li) {
  for (size_t i = 0; i < n->segs.size(); ++i) if (n->seg_layer[i] == li && n->segs[i].kind != 3 && n->segs[i].kind != 9) return (int)i;
  return -1;
}
static bool layer_has_lr(const b2g_net* n, int li) { return lr_segment(n, li) >= 0; }
static int32_t find_lr_layer(const b2g_net* n, const char* layer, int* li) {
  for (size_t i = 0; i < n->L.size(); ++i) if (!strncmp(n->L[i].d.name, layer, B2G_NAME_LEN)) {
    if (!layer_has_lr(n, (int)i)) return fail(B2G_ERR_ARG, "layer %s has no learning rate (frozen, no parameters, NoOp or AdaDelta)", layer);
    *li = (int)i; return 0;
  }
  return fail(B2G_ERR_ARG, "no layer named %s", layer);
}
// Rebuilds the per-segment table from the per-layer schedules: MAP entries go to sched_map (values, then keys), every segment of a layer with
// a learning rate carries the layer's schedule (the BatchNorm mean/var segments too; their NoOp update ignores it).
static int32_t net_upload_schedules(b2g_net* n) {
  cudaStream_t s = n->ctx->stream;
  size_t nv = 0; for (auto& ls : n->layer_sched) nv += ls.vals.size();
  const size_t bytes = nv * (sizeof(double) + sizeof(int32_t));
  CU(cudaStreamSynchronize(s));                  // nothing in flight reads the old table or map
  if (bytes > n->sched_map_bytes) {
    if (n->sched_map) { cudaFree(n->sched_map); n->sched_map = nullptr; n->sched_map_bytes = 0; }
    cudaError_t e = cudaMalloc(&n->sched_map, bytes);
    if (e != cudaSuccess) { n->sched_map = nullptr; return fail(B2G_ERR_OOM, "cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e)); }
    n->sched_map_bytes = bytes;
  }
  std::vector<char> host(bytes); double* dv = (double*)n->sched_map; int32_t* dk = (int32_t*)((char*)n->sched_map + nv * sizeof(double));
  std::vector<UpdSched> per_layer(n->L.size()); size_t at = 0;
  for (size_t li = 0; li < n->L.size(); ++li) {
    const auto& ls = n->layer_sched[li]; per_layer[li] = ls.sc;
    if (ls.sc.kind == B2G_SCHED_MAP) {
      memcpy(host.data() + at * sizeof(double), ls.vals.data(), ls.vals.size() * sizeof(double));
      memcpy(host.data() + nv * sizeof(double) + at * sizeof(int32_t), ls.keys.data(), ls.keys.size() * sizeof(int32_t));
      per_layer[li].vals = dv + at; per_layer[li].keys = dk + at; at += ls.vals.size();
    }
  }
  std::vector<UpdSched> seg(n->segs.size()); bool on = false;
  for (size_t i = 0; i < n->segs.size(); ++i) { seg[i] = per_layer[n->seg_layer[i]]; on = on || seg[i].kind != B2G_SCHED_NONE; }
  if (bytes) CU(cudaMemcpyAsync(n->sched_map, host.data(), bytes, cudaMemcpyHostToDevice, s));
  if (!seg.empty()) CU(cudaMemcpyAsync(n->sched_dev, seg.data(), sizeof(UpdSched) * seg.size(), cudaMemcpyHostToDevice, s));
  CU(cudaStreamSynchronize(s));
  n->sched_on = on; ++n->settings_gen;
  return 0;
}
// A b2g_lr_schedule checked and copied (null or NONE: no schedule); shared by the learning-rate and the DropoutLayer schedules
static int32_t parse_schedule(const b2g_lr_schedule* s, b2g_net::LayerSched* out) {
  b2g_net::LayerSched ls;
  if (s && s->kind != B2G_SCHED_NONE) {
    if (s->kind < B2G_SCHED_EXPONENTIAL || s->kind > B2G_SCHED_MAP) return fail(B2G_ERR_ARG, "unknown schedule kind %d (PolySchedule is not supported)", s->kind);
    if (s->type != B2G_SCHED_ITERATION && s->type != B2G_SCHED_EPOCH) return fail(B2G_ERR_ARG, "unknown schedule type %d", s->type);
    if (!std::isfinite(s->initial) || !std::isfinite(s->gamma) || !std::isfinite(s->power) || !std::isfinite(s->step) || !std::isfinite(s->decay_rate))
      return fail(B2G_ERR_ARG, "schedule parameters must be finite");
    if (s->kind == B2G_SCHED_STEP && !(s->step > 0.0)) return fail(B2G_ERR_ARG, "StepSchedule step %g: must be > 0", s->step);
    if (s->kind == B2G_SCHED_INVERSE && s->gamma < 0.0) return fail(B2G_ERR_ARG, "InverseSchedule gamma %g: must be >= 0", s->gamma);
    UpdSched& sc = ls.sc; sc.kind = s->kind; sc.type = s->type;
    sc.initial = s->initial; sc.gamma = s->gamma; sc.power = s->power; sc.step = s->step; sc.decay = s->decay_rate;
    if (s->kind == B2G_SCHED_MAP) {
      if (s->n_map < 1 || !s->map_keys || !s->map_values) return fail(B2G_ERR_ARG, "MapSchedule needs at least one entry");
      bool has0 = false;
      for (int j = 0; j < s->n_map; ++j) {
        if (j > 0 && s->map_keys[j] <= s->map_keys[j - 1]) return fail(B2G_ERR_ARG, "MapSchedule keys must strictly increase");
        if (!std::isfinite(s->map_values[j])) return fail(B2G_ERR_ARG, "MapSchedule values must be finite");
        has0 = has0 || s->map_keys[j] == 0;
      }
      if (!has0) return fail(B2G_ERR_ARG, "MapSchedule has no value for key 0");
      ls.keys.assign(s->map_keys, s->map_keys + s->n_map); ls.vals.assign(s->map_values, s->map_values + s->n_map); sc.n_map = s->n_map;
    }
  }
  *out = ls;
  return 0;
}
extern "C" int32_t b2g_net_set_lr_schedule(b2g_net* n, const char* layer, const b2g_lr_schedule* s) {
  if (!n) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device));
  b2g_net::LayerSched ls; B2(parse_schedule(s, &ls));
  if (layer) { int li = 0; B2(find_lr_layer(n, layer, &li)); n->layer_sched[li] = ls; }
  else for (size_t li = 0; li < n->L.size(); ++li) if (layer_has_lr(n, (int)li)) n->layer_sched[li] = ls;
  return net_upload_schedules(n);
}
extern "C" int32_t b2g_net_get_learning_rate(b2g_net* n, const char* layer, float* out) {
  if (!n || !layer || !out) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device));
  int li = 0; B2(find_lr_layer(n, layer, &li));
  const int seg = lr_segment(n, li);
  k_sched_lr(n->segs_dev, n->sched_dev, seg, n->step_dev, n->epoch_dev, n->lr_out, n->ctx->stream); CHECK_KERNELS();
  CU(cudaMemcpyAsync(out, n->lr_out, sizeof(float), cudaMemcpyDeviceToHost, n->ctx->stream)); CU(cudaStreamSynchronize(n->ctx->stream));
  return 0;
}
// ------------------------------------------------------------------ DropoutLayer schedules (b2g_net_set_dropout_schedule) ---------------
static int32_t find_dropout_layer(const b2g_net* n, const char* layer, int* li) {
  for (size_t i = 0; i < n->L.size(); ++i) if (!strncmp(n->L[i].d.name, layer, B2G_NAME_LEN)) {
    if (n->L[i].d.type != B2G_LAYER_DROPOUT) return fail(B2G_ERR_ARG, "layer %s is not a DropoutLayer", layer);
    *li = (int)i; return 0;
  }
  return fail(B2G_ERR_ARG, "no layer named %s", layer);
}
// A layer's schedule to its device slot `dev`, MAP entries (values, then keys) to a buffer of its own (*map, replaced)
static int32_t upload_schedule(b2g_net* n, UpdSched* dev, void** map, const b2g_net::LayerSched& ls) {
  cudaStream_t s = n->ctx->stream;
  CU(cudaStreamSynchronize(s));                  // nothing in flight reads the old schedule or map
  if (*map) { CU(cudaFree(*map)); *map = nullptr; }
  UpdSched sc = ls.sc;
  if (sc.kind == B2G_SCHED_MAP) {
    const size_t nv = ls.vals.size(), bytes = nv * (sizeof(double) + sizeof(int32_t));
    cudaError_t e = cudaMalloc(map, bytes);
    if (e != cudaSuccess) { *map = nullptr; return fail(B2G_ERR_OOM, "cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e)); }
    CU(cudaMemcpyAsync(*map, ls.vals.data(), nv * sizeof(double), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync((char*)*map + nv * sizeof(double), ls.keys.data(), nv * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    sc.vals = (const double*)*map; sc.keys = (const int32_t*)((char*)*map + nv * sizeof(double));
  }
  CU(cudaMemcpyAsync(dev, &sc, sizeof(sc), cudaMemcpyHostToDevice, s));
  CU(cudaStreamSynchronize(s));
  return 0;
}
static int32_t upload_dropout_schedule(b2g_net* n, LayerRT& l, const b2g_net::LayerSched& ls) {
  B2(upload_schedule(n, l.drop_sched_dev, &l.drop_map, ls));
  l.drop_sched = ls.sc.kind != B2G_SCHED_NONE;
  return 0;
}
extern "C" int32_t b2g_net_set_dropout_schedule(b2g_net* n, const char* layer, const b2g_lr_schedule* s) {
  if (!n) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device));
  b2g_net::LayerSched ls; B2(parse_schedule(s, &ls));
  if (layer) { int li = 0; B2(find_dropout_layer(n, layer, &li)); B2(upload_dropout_schedule(n, n->L[li], ls)); }
  else for (auto& l : n->L) if (l.d.type == B2G_LAYER_DROPOUT && !l.d.frozen) B2(upload_dropout_schedule(n, l, ls));
  ++n->settings_gen;           // a captured step holds which kernels the layers launch: re-capture
  return 0;
}
extern "C" int32_t b2g_net_get_dropout_value(b2g_net* n, const char* layer, float* out) {
  if (!n || !layer || !out) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device));
  int li = 0; B2(find_dropout_layer(n, layer, &li));
  const LayerRT& l = n->L[li];
  k_noise_value(l.d.act, l.d.act_alpha, noise_sched(n, l, nullptr, nullptr), n->lr_out, n->ctx->stream); CHECK_KERNELS();
  CU(cudaMemcpyAsync(out, n->lr_out, sizeof(float), cudaMemcpyDeviceToHost, n->ctx->stream)); CU(cudaStreamSynchronize(n->ctx->stream));
  return 0;
}
// ------------------------------------------------------------------ weight noise (b2g_net_set_weight_noise) --------------------------------
static int32_t check_weight_noise(const b2g_weight_noise& w) {
  if (w.kind == B2G_WEIGHT_NOISE_NONE) return 0;
  if (w.kind == B2G_WEIGHT_NOISE_DROPCONNECT) {
    if (!(w.p > 0.f && w.p <= 1.f)) return fail(B2G_ERR_ARG, "DropConnect retain probability %g outside (0, 1]", (double)w.p);
    return 0;
  }
  if (w.kind != B2G_WEIGHT_NOISE_WEIGHTNOISE) return fail(B2G_ERR_ARG, "unknown weight noise kind %d", w.kind);
  if (!std::isfinite(w.a) || !std::isfinite(w.b)) return fail(B2G_ERR_ARG, "WeightNoise distribution parameters must be finite");
  if (w.dist == B2G_DIST_NORMAL) { if (w.b < 0.f) return fail(B2G_ERR_ARG, "NormalDistribution std %g < 0", (double)w.b); }
  else if (w.dist == B2G_DIST_UNIFORM) { if (w.b < w.a) return fail(B2G_ERR_ARG, "UniformDistribution upper %g < lower %g", (double)w.b, (double)w.a); }
  else return fail(B2G_ERR_ARG, "unknown distribution %d (NORMAL or UNIFORM)", w.dist);
  return 0;
}
// The layer's noisy operands, once: W' (fp32, or bf16 straight | packed pixel-shuffle copy) and b' when the bias is perturbed
static int32_t wn_alloc(b2g_net* n, LayerRT& l) {
  cudaStream_t s = n->ctx->stream;
  if (!l.wn_w) {
    if (n->prec == PREC_BF16) {
      const int64_t straight = (l.n_W + 63) / 64 * 64, ps = l.off_Wps_bf >= 0 ? (int64_t)k_tc_deconv_ps_weight_elems(l.geom) : 0;
      B2(dalloc(n, &l.wn_w, sizeof(__nv_bfloat16) * (straight + ps)));
      // the packed operand's slots no weight element maps to stay zero, as k_pack_deconv_ps leaves them
      CU(cudaMemsetAsync(l.wn_w, 0, sizeof(__nv_bfloat16) * (straight + ps), s));
      l.wn_ps = ps ? straight : -1;
    } else B2(dalloc(n, &l.wn_w, sizeof(float) * l.n_W));
  }
  if (l.wn.apply_to_bias && l.off_b >= 0 && !l.wn_b) B2(dalloc(n, &l.wn_b, sizeof(float) * l.d.n_out));
  return 0;
}
// The job table of one draw: a W job per drawing layer and a b job per perturbed bias, each of ceil(n / WN_CHUNK) blocks
static int32_t wn_build_jobs(b2g_net* n) {
  if (!n->wn_jobs) B2(dalloc(n, &n->wn_jobs, sizeof(WnJob) * 2 * n->L.size()));
  std::vector<WnJob> jobs; int blocks = 0;
  for (size_t i = 0; i < n->L.size(); ++i) {
    const LayerRT& l = n->L[i];
    if (!l.wn_active()) continue;
    WnJob j{}; j.layer = (int)i; j.kind = l.wn.kind; j.dist = l.wn.dist; j.additive = l.wn.additive; j.p = l.wn.p; j.a = l.wn.a; j.b = l.wn.b;
    j.sched = l.wn_sched ? l.wn_sched_dev : nullptr; j.sg.off_bf = 0; j.sg.off_ps = -1;
    WnJob w = j; w.src = n->params + l.off_W; w.n = l.n_W; w.j0 = 0;
    if (n->prec == PREC_BF16) { w.dst_bf16 = (__nv_bfloat16*)l.wn_w; w.sg.len = l.n_W; w.sg.off_ps = l.wn_ps; w.sg.ps_O = l.geom.O; w.sg.ps_C = l.geom.C; }
    else w.dst_f32 = (float*)l.wn_w;
    w.blk_begin = blocks; w.blocks = (int)((w.n + WN_CHUNK - 1) / WN_CHUNK); blocks += w.blocks; jobs.push_back(w);
    if (l.wn.apply_to_bias && l.off_b >= 0) {
      WnJob b = j; b.src = n->params + l.off_b; b.n = l.d.n_out; b.j0 = 4 * ((l.n_W + 3) / 4); b.dst_f32 = l.wn_b;
      b.blk_begin = blocks; b.blocks = (int)((b.n + WN_CHUNK - 1) / WN_CHUNK); blocks += b.blocks; jobs.push_back(b);
    }
  }
  if (!jobs.empty()) { CU(cudaMemcpyAsync(n->wn_jobs, jobs.data(), sizeof(WnJob) * jobs.size(), cudaMemcpyHostToDevice, n->ctx->stream)); CU(cudaStreamSynchronize(n->ctx->stream)); }
  n->wn_njobs = (int)jobs.size(); n->wn_blocks = blocks;
  return 0;
}
extern "C" int32_t b2g_net_set_weight_noise(b2g_net* n, const char* layer, const b2g_weight_noise* wn) {
  if (!n) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device));
  b2g_weight_noise w{}; if (wn && wn->kind != B2G_WEIGHT_NOISE_NONE) w = *wn;
  B2(check_weight_noise(w));
  b2g_net::LayerSched ls;
  if (w.kind == B2G_WEIGHT_NOISE_DROPCONNECT) B2(parse_schedule(w.p_schedule, &ls));
  w.p_schedule = nullptr;
  std::vector<int> targets;
  if (layer) {
    for (size_t i = 0; i < n->L.size() && targets.empty(); ++i) if (!strncmp(n->L[i].d.name, layer, B2G_NAME_LEN)) {
      if (!n->L[i].has_gemm()) return fail(B2G_ERR_ARG, "layer %s: weight noise needs a conv, deconv, dense or output layer (not supported on a PReLU's slopes)", layer);
      targets.push_back((int)i);
    }
    if (targets.empty()) return fail(B2G_ERR_ARG, "no layer named %s", layer);
  } else for (size_t i = 0; i < n->L.size(); ++i) if (n->L[i].has_gemm() && !n->L[i].d.frozen) targets.push_back((int)i);
  CU(cudaStreamSynchronize(n->ctx->stream));      // nothing in flight reads the old job table or operands
  for (int i : targets) {
    LayerRT& l = n->L[i];
    l.wn = w; l.wn_drawn = false; l.wn_sched = false;
    if (w.kind == B2G_WEIGHT_NOISE_NONE) continue;
    B2(wn_alloc(n, l));
    if (w.kind == B2G_WEIGHT_NOISE_DROPCONNECT && ls.sc.kind != B2G_SCHED_NONE) {
      if (!l.wn_sched_dev) B2(dalloc(n, &l.wn_sched_dev, sizeof(UpdSched)));
      B2(upload_schedule(n, l.wn_sched_dev, &l.wn_map, ls));
      l.wn_sched = true;
    }
  }
  B2(wn_build_jobs(n));
  ++n->settings_gen;           // a captured step holds the launch and its job count: re-capture
  return 0;
}

// ------------------------------------------------------------------ weight initialization (b2g_net_init_weights) --------------------------
static int32_t check_weight_init(const b2g_weight_init& w) {
  if (w.scheme < B2G_WI_DISTRIBUTION || w.scheme > B2G_WI_VAR_SCALING_UNIFORM_FAN_AVG) return fail(B2G_ERR_ARG, "unknown weight init scheme %d", w.scheme);
  if (!std::isfinite(w.bias_init)) return fail(B2G_ERR_ARG, "biasInit %g is not finite", (double)w.bias_init);
  if (w.scheme != B2G_WI_DISTRIBUTION) return 0;
  if (w.dist < B2G_DIST_NORMAL || w.dist > B2G_DIST_ORTHOGONAL) return fail(B2G_ERR_ARG, "unknown distribution %d", w.dist);
  if (w.dist == B2G_DIST_ORTHOGONAL) return fail(B2G_ERR_UNSUPPORTED, "OrthogonalDistribution is not supported (it needs an SVD)");
  if (!std::isfinite(w.a) || (w.dist != B2G_DIST_CONSTANT && !std::isfinite(w.b))) return fail(B2G_ERR_ARG, "distribution parameters must be finite");
  switch (w.dist) {
    case B2G_DIST_NORMAL: case B2G_DIST_TRUNCATED_NORMAL: case B2G_DIST_LOG_NORMAL:
      if (w.b < 0.f) return fail(B2G_ERR_ARG, "distribution std %g < 0", (double)w.b);
      break;
    case B2G_DIST_UNIFORM: if (w.b < w.a) return fail(B2G_ERR_ARG, "UniformDistribution upper %g < lower %g", (double)w.b, (double)w.a); break;
    case B2G_DIST_BINOMIAL:
      if (!(w.a >= 0.f && w.a <= 65536.f && w.a == floorf(w.a))) return fail(B2G_ERR_ARG, "BinomialDistribution nTrials %g is not a whole number in [0, 65536]", (double)w.a);
      if (!(w.b >= 0.f && w.b <= 1.f)) return fail(B2G_ERR_ARG, "BinomialDistribution p %g outside [0, 1]", (double)w.b);
      break;
    default: break;
  }
  return 0;
}
// The draw of one layer's W under the scheme, from the desc's fans (the internal geometry of a 1x1-map deconv or whole-input conv aside)
static int32_t weight_init_draw(const b2g_weight_init& w, const LayerRT& l, WiDraw* out) {
  const b2g_layer_desc& d = l.d;
  if (d.type == B2G_LAYER_PRELU && w.scheme != B2G_WI_ZERO && w.scheme != B2G_WI_ONES && w.scheme != B2G_WI_DISTRIBUTION)
    return fail(B2G_ERR_ARG, "layer %s: weight init %d needs fans, which a PReLU's slopes do not have (ZERO, ONES or DISTRIBUTION)", d.name, w.scheme);
  const bool conv = d.type == B2G_LAYER_CONV2D || d.type == B2G_LAYER_DECONV2D;
  const double fi = (double)d.n_in * l.wTaps, fo = (double)d.n_out * l.wTaps / (conv ? (double)(d.s_h * d.s_w) : 1.0);
  WiDraw r{}; double sd = -1.0, lim = -1.0, tsd = -1.0;
  switch (w.scheme) {
    case B2G_WI_DISTRIBUTION:
      r.kind = w.dist; r.a = w.a; r.b = w.b;
      if (w.dist == B2G_DIST_BINOMIAL) { r.trials = (int)w.a; r.thr = (uint64_t)floor((double)w.b * 4294967296.0); }
      break;
    case B2G_WI_ZERO: r.kind = WI_CONSTANT; r.a = 0.f; break;
    case B2G_WI_ONES: r.kind = WI_CONSTANT; r.a = 1.f; break;
    case B2G_WI_SIGMOID_UNIFORM: lim = 4.0 * sqrt(6.0 / (fi + fo)); break;
    case B2G_WI_NORMAL: case B2G_WI_LECUN_NORMAL: case B2G_WI_XAVIER_FAN_IN: sd = 1.0 / sqrt(fi); break;
    case B2G_WI_UNIFORM: lim = 1.0 / sqrt(fi); break;
    case B2G_WI_XAVIER: sd = sqrt(2.0 / (fi + fo)); break;
    case B2G_WI_XAVIER_UNIFORM: lim = sqrt(6.0) / sqrt(fi + fo); break;
    case B2G_WI_XAVIER_LEGACY: sd = 1.0 / sqrt((double)d.n_in + d.n_out); break;
    case B2G_WI_RELU: sd = sqrt(2.0 / fi); break;
    case B2G_WI_RELU_UNIFORM: lim = sqrt(6.0 / fi); break;
    case B2G_WI_IDENTITY:
      if (conv) return fail(B2G_ERR_SHAPE, "layer %s: WeightInit.IDENTITY needs a dense or output layer, not a convolution", d.name);
      if (d.n_in != d.n_out) return fail(B2G_ERR_SHAPE, "layer %s: WeightInit.IDENTITY needs a square W, got nIn %d != nOut %d", d.name, d.n_in, d.n_out);
      r.kind = WI_IDENTITY; break;
    case B2G_WI_LECUN_UNIFORM: case B2G_WI_VAR_SCALING_UNIFORM_FAN_IN: lim = 3.0 / sqrt(fi); break;
    case B2G_WI_VAR_SCALING_NORMAL_FAN_IN: tsd = sqrt(1.0 / fi); break;
    case B2G_WI_VAR_SCALING_NORMAL_FAN_OUT: tsd = sqrt(1.0 / fo); break;
    case B2G_WI_VAR_SCALING_NORMAL_FAN_AVG: tsd = sqrt(2.0 / (fi + fo)); break;
    case B2G_WI_VAR_SCALING_UNIFORM_FAN_OUT: lim = 3.0 / sqrt(fo); break;
    case B2G_WI_VAR_SCALING_UNIFORM_FAN_AVG: lim = 3.0 / sqrt((fi + fo) / 2.0); break;
    default: return fail(B2G_ERR_ARG, "unknown weight init scheme %d", w.scheme);
  }
  if (sd >= 0.0) { r.kind = WI_NORMAL; r.a = 0.f; r.b = (float)sd; }
  if (tsd >= 0.0) { r.kind = WI_TRUNCATED_NORMAL; r.a = 0.f; r.b = (float)tsd; }
  if (lim >= 0.0) { r.kind = WI_UNIFORM; r.a = -(float)lim; r.b = (float)lim; }
  *out = r;
  return 0;
}
extern "C" int32_t b2g_net_init_weights(b2g_net* n, const char* layer, const b2g_weight_init* wi) {
  if (!n || !wi) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device));
  const b2g_weight_init w = *wi;
  B2(check_weight_init(w));
  std::vector<int> targets;
  if (layer) {
    for (size_t i = 0; i < n->L.size() && targets.empty(); ++i) if (!strncmp(n->L[i].d.name, layer, B2G_NAME_LEN)) {
      if (!n->L[i].has_reg()) return fail(B2G_ERR_ARG, "layer %s has no W (weight init needs a conv, deconv, dense, output or PReLU layer)", layer);
      targets.push_back((int)i);
    }
    if (targets.empty()) return fail(B2G_ERR_ARG, "no layer named %s", layer);
  } else for (size_t i = 0; i < n->L.size(); ++i) if (n->L[i].has_gemm()) targets.push_back((int)i);
  std::vector<WiDraw> draws(targets.size());
  for (size_t k = 0; k < targets.size(); ++k) B2(weight_init_draw(w, n->L[targets[k]], &draws[k]));    // every target checked before any write
  cudaStream_t s = n->ctx->stream;
  const uint64_t seed = n->cfg.seed ? n->cfg.seed : 666;
  for (size_t k = 0; k < targets.size(); ++k) {
    const LayerRT& l = n->L[targets[k]];
    k_weight_init(n->params + l.off_W, l.wA, l.wTaps, l.wB, draws[k], l.off_b >= 0 ? n->params + l.off_b : nullptr, l.d.n_out, w.bias_init, seed, targets[k], s);
    net_refresh_shadow(n, targets[k]);
  }
  CU(cudaStreamSynchronize(s)); CHECK_KERNELS();
  return 0;
}

// ------------------------------------------------------------------ regularization (b2g_net_set_regularization) --------------------------
// The coefficients live in the updater's segment table and the score table, both read from device memory at run time: a new value needs
// no new launch, and a captured GAN step picks it up at its next replay without a re-capture.
static int32_t find_reg_layer(const b2g_net* n, const char* layer, int* li) {
  for (size_t i = 0; i < n->L.size(); ++i) if (!strncmp(n->L[i].d.name, layer, B2G_NAME_LEN)) {
    if (!n->L[i].has_reg()) return fail(B2G_ERR_ARG, "layer %s has no W (regularization needs a conv, deconv, dense, output or PReLU layer)", layer);
    *li = (int)i; return 0;
  }
  return fail(B2G_ERR_ARG, "no layer named %s", layer);
}
extern "C" int32_t b2g_net_set_regularization(b2g_net* n, const char* layer, const b2g_regularization* r) {
  if (!n || !r) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device));
  const float v[4] = {r->l1, r->l2, r->l1_bias, r->l2_bias};
  for (float x : v) if (!(std::isfinite(x) && x >= 0.f)) return fail(B2G_ERR_ARG, "regularization coefficient %g: must be finite and >= 0", (double)x);
  if (layer) { int li = 0; B2(find_reg_layer(n, layer, &li)); n->L[li].reg = *r; }
  else for (auto& l : n->L) if (l.has_reg() && !l.d.frozen) l.reg = *r;
  for (size_t i = 0; i < n->segs.size(); ++i) {        // frozen layers own no segment: they take no term
    const LayerRT& l = n->L[n->seg_layer[i]];
    if (!l.has_reg()) continue;
    const bool weight = n->segs[i].off == l.off_W;
    n->segs[i].l2 = weight ? l.reg.l2 : l.reg.l2_bias; n->segs[i].l1 = weight ? l.reg.l1 : l.reg.l1_bias;
  }
  n->n_l2 = n->n_l1 = 0;
  for (size_t k = 0; k < n->reg_seg.size(); ++k) {
    const UpdSeg& sg = n->segs[n->reg_seg[k]];
    n->reg_l2c[k] = 0.5f * sg.l2; n->reg_l1c[k] = sg.l1; n->n_l2 += sg.l2 != 0.f; n->n_l1 += sg.l1 != 0.f;
  }
  cudaStream_t s = n->ctx->stream;
  CU(cudaStreamSynchronize(s));                  // nothing in flight reads the old tables
  if (!n->segs.empty()) CU(cudaMemcpyAsync(n->segs_dev, n->segs.data(), sizeof(UpdSeg) * n->segs.size(), cudaMemcpyHostToDevice, s));
  if (!n->reg_seg.empty()) {
    CU(cudaMemcpyAsync(n->reg_l2c_dev, n->reg_l2c.data(), sizeof(float) * n->reg_seg.size(), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(n->reg_l1c_dev, n->reg_l1c.data(), sizeof(float) * n->reg_seg.size(), cudaMemcpyHostToDevice, s));
  }
  CU(cudaStreamSynchronize(s));
  return 0;
}
extern "C" int32_t b2g_net_get_regularization(b2g_net* n, const char* layer, b2g_regularization* out) {
  if (!n || !layer || !out) return fail(B2G_ERR_ARG, "null");
  int li = 0; B2(find_reg_layer(n, layer, &li)); *out = n->L[li].reg; return 0;
}
extern "C" int32_t b2g_net_calc_regularization(b2g_net* n, double* l1, double* l2) {
  if (!n) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device));
  double a = 0.0, b = 0.0;
  B2(net_reg_sums(n, &a, &b)); CU(cudaStreamSynchronize(n->ctx->stream));
  if (l1) *l1 = a;
  if (l2) *l2 = b;
  return 0;
}

// The epoch word lives on the device like the iteration counter: a replayed graph reads the value set last, no re-capture needed.
extern "C" int32_t b2g_net_get_epoch(b2g_net* n, int64_t* out) {
  if (!n || !out) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device));
  int64_t v = 0; CU(cudaMemcpyAsync(&v, n->epoch_dev, sizeof(v), cudaMemcpyDeviceToHost, n->ctx->stream)); CU(cudaStreamSynchronize(n->ctx->stream)); *out = v; return 0;
}
extern "C" int32_t b2g_net_set_epoch(b2g_net* n, int64_t epoch) {
  if (!n || epoch < 0) return fail(B2G_ERR_ARG, "bad epoch"); CU(cudaSetDevice(n->ctx->device));
  CU(cudaMemcpyAsync(n->epoch_dev, &epoch, sizeof(epoch), cudaMemcpyHostToDevice, n->ctx->stream)); CU(cudaStreamSynchronize(n->ctx->stream)); return 0;
}
extern "C" int32_t b2g_net_simt_gemm_calls(b2g_net* n, uint64_t* out) { if (!n || !out) return fail(B2G_ERR_ARG, "null"); *out = n->simt_gemm_calls; return 0; }

// ------------------------------------------------------------------ data parallel ------------------------
extern "C" int32_t b2g_comm_unique_id(void* id128) { if (!id128) return fail(B2G_ERR_ARG, "null"); B2(nccl_load()); NcclId id; NC(g_nccl.uid(&id)); memcpy(id128, &id, sizeof(id)); return 0; }
extern "C" int32_t b2g_ctx_comm_init(b2g_ctx* c, int32_t world, int32_t rank, const void* id128) {
  if (!c || !id128 || world < 1 || rank < 0 || rank >= world) return fail(B2G_ERR_ARG, "bad communicator arguments");
  B2(nccl_load()); CU(cudaSetDevice(c->device));
  NcclId id; memcpy(&id, id128, sizeof(id));
  NC(g_nccl.init(&c->comm, world, id, rank)); c->world = world; c->rank = rank; return 0;
}
extern "C" int32_t b2g_ctx_comm_destroy(b2g_ctx* c) { if (c && c->comm) { g_nccl.destroy(c->comm); c->comm = nullptr; c->world = 1; c->rank = 0; } return 0; }
extern "C" int32_t b2g_net_set_grad_allreduce(b2g_net* n, int32_t enabled) { if (!n) return fail(B2G_ERR_ARG, "null"); n->grad_allreduce = enabled != 0; return 0; }
extern "C" int32_t b2g_net_set_sync_bn(b2g_net* n, int32_t enabled) { if (!n) return fail(B2G_ERR_ARG, "null"); if (enabled && n->prec != PREC_BF16) return fail(B2G_ERR_UNSUPPORTED, "sync_bn rides on the fused BatchNorm path (BF16 nets)"); n->sync_bn = enabled != 0; return 0; }
extern "C" int32_t b2g_net_set_grad_payload_bf16(b2g_net* n, int32_t enabled) {
  if (!n) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device));
  if (enabled && !n->ar_buf) B2(dalloc(n, &n->ar_buf, sizeof(__nv_bfloat16) * (size_t)n->n_params));
  n->ar_bf16 = enabled != 0; return 0;
}
// COLLECTIVE (every rank, same order of nets): maps every rank's gradient vector and flag words into this process (cudaIpc*, handles
// exchanged with ncclAllGather) and switches the net's gradient all-reduce to the peer-memory kernel (kernels_ew.cu p2p_allreduce_kernel).
// If any rank cannot map (different nodes, IPC disabled) every rank stays on ncclAllReduce; *enabled reports the common outcome.
extern "C" int32_t b2g_net_enable_p2p_allreduce(b2g_net* n, int32_t* enabled) {
  if (!n) return fail(B2G_ERR_ARG, "null"); b2g_ctx* c = n->ctx; CU(cudaSetDevice(c->device)); if (enabled) *enabled = 0;
  if (!c->comm || c->world < 2) return 0;
  if (c->world > 8 || !g_nccl.ag) return 0;
  cudaStream_t s = c->stream;
  if (!c->p2p_flags) { CU(cudaMalloc(&c->p2p_flags, 16 * sizeof(unsigned))); CU(cudaMalloc(&c->p2p_state, 2 * sizeof(unsigned)));
                       CU(cudaMemsetAsync(c->p2p_flags, 0, 16 * sizeof(unsigned), s)); CU(cudaMemsetAsync(c->p2p_state, 0, 2 * sizeof(unsigned), s)); CU(cudaStreamSynchronize(s)); }
  struct Pair { cudaIpcMemHandle_t flags, grads; };
  Pair mine; memset(&mine, 0, sizeof(mine)); float ok = 1.f;
  if (cudaIpcGetMemHandle(&mine.flags, c->p2p_flags) != cudaSuccess || cudaIpcGetMemHandle(&mine.grads, n->grads) != cudaSuccess) { cudaGetLastError(); ok = 0.f; }
  std::vector<Pair> all(c->world);
  char *d_send = nullptr, *d_recv = nullptr; float* d_ok = nullptr;
  CU(cudaMalloc(&d_send, sizeof(Pair))); CU(cudaMalloc(&d_recv, sizeof(Pair) * c->world)); CU(cudaMalloc(&d_ok, sizeof(float)));
  CU(cudaMemcpyAsync(d_send, &mine, sizeof(Pair), cudaMemcpyHostToDevice, s));
  NC(g_nccl.ag(d_send, d_recv, sizeof(Pair), /*ncclChar*/ 0, c->comm, s));
  CU(cudaMemcpyAsync(all.data(), d_recv, sizeof(Pair) * c->world, cudaMemcpyDeviceToHost, s)); CU(cudaStreamSynchronize(s));
  float* pg[8] = {}; unsigned* pf[8] = {};
  for (int r = 0; r < c->world && ok > 0.f; ++r) {
    if (r == c->rank) { pg[r] = n->grads; pf[r] = c->p2p_flags; continue; }
    void* q = nullptr;
    if (cudaIpcOpenMemHandle(&q, all[r].grads, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); ok = 0.f; break; }
    pg[r] = (float*)q;
    if (c->p2p_flags_mapped) pf[r] = c->p2p_peer_flags[r];
    else { if (cudaIpcOpenMemHandle(&q, all[r].flags, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); ok = 0.f; break; } pf[r] = (unsigned*)q; }
  }
  // the decision must be common: sum of the ranks' verdicts
  CU(cudaMemcpyAsync(d_ok, &ok, sizeof(float), cudaMemcpyHostToDevice, s)); NC(g_nccl.ar(d_ok, d_ok, 1, 7, 0, c->comm, s));
  float sum = 0.f; CU(cudaMemcpyAsync(&sum, d_ok, sizeof(float), cudaMemcpyDeviceToHost, s)); CU(cudaStreamSynchronize(s));
  cudaFree(d_send); cudaFree(d_recv); cudaFree(d_ok);
  if (sum < (float)c->world - 0.5f) {      // somebody failed: undo the mappings made here
    for (int r = 0; r < c->world; ++r) { if (r == c->rank) continue; if (pg[r]) cudaIpcCloseMemHandle(pg[r]); if (!c->p2p_flags_mapped && pf[r]) cudaIpcCloseMemHandle(pf[r]); }
    return 0;
  }
  for (int r = 0; r < c->world; ++r) { n->p2p_peer_grads[r] = pg[r]; c->p2p_peer_flags[r] = pf[r]; }
  c->p2p_flags_mapped = true; n->p2p = true; if (enabled) *enabled = 1;
  return 0;
}
extern "C" int32_t b2g_net_average_parameters(b2g_net* n) {
  if (!n) return fail(B2G_ERR_ARG, "null"); b2g_ctx* c = n->ctx; CU(cudaSetDevice(c->device));
  if (!c->comm || c->world == 1) return 0;
  const float inv = 1.0f / (float)c->world; cudaStream_t s = c->stream;
  float* bufs[4] = {n->params, n->st0, n->st1, n->st2};
  for (float* b : bufs) { if (!b) continue; NC(g_nccl.ar(b, b, (size_t)n->n_params, 7, 0, c->comm, s)); k_scale_f32(b, inv, (size_t)n->n_params, s); }
  net_refresh_shadow(n);
  CU(cudaStreamSynchronize(s)); return 0;
}

// ------------------------------------------------------------------ test hooks ----------------------------
namespace {
// Every device buffer and event of one test-hook call, released on every return.  Copies run on stream s; T is the call's precision.
struct HookMem {
  cudaStream_t s; int prec;
  std::vector<void*> bufs; std::vector<cudaEvent_t> events;
  HookMem(cudaStream_t s_, int prec_) : s(s_), prec(prec_) {}
  HookMem(const HookMem&) = delete; HookMem& operator=(const HookMem&) = delete;
  ~HookMem() { for (void* p : bufs) cudaFree(p); for (cudaEvent_t e : events) cudaEventDestroy(e); }
  // count es-byte elements, off elements past a 256-byte aligned allocation (as a layer's W and dW sit in the flattened parameter vectors)
  int32_t dev(size_t count, size_t es, void** p, size_t off = 0) {
    void* b = nullptr; *p = nullptr; CU(cudaMalloc(&b, es * (count + off) + 16)); bufs.push_back(b); *p = (char*)b + es * off; return 0; }
  // fp32 host -> fp32 device; h null: the buffer only
  int32_t upF(const float* h, size_t count, float** p, size_t off = 0) {
    B2(dev(count, 4, (void**)p, off)); if (h) CU(cudaMemcpyAsync(*p, h, 4 * count, cudaMemcpyHostToDevice, s)); return 0; }
  // fp32 device -> T device (bf16: rounded)
  int32_t toT(const float* f, void* t, size_t count) {
    if (prec == PREC_F32) CU(cudaMemcpyAsync(t, f, 4 * count, cudaMemcpyDeviceToDevice, s)); else k_cast_f32_to_bf16(f, (__nv_bfloat16*)t, count, s); return 0; }
  // fp32 host -> T device (bf16: rounded on the device from an fp32 copy); h null: the buffer only
  int32_t upT(const float* h, size_t count, void** p, size_t off = 0) {
    B2(dev(count, prec_size(prec), p, off)); if (!h) return 0;
    if (prec == PREC_F32) { CU(cudaMemcpyAsync(*p, h, 4 * count, cudaMemcpyHostToDevice, s)); return 0; }
    float* f = nullptr; B2(upF(h, count, &f)); return toT(f, *p, count); }
  // fp32 device -> host; h null: nothing
  int32_t downF(float* h, const float* d, size_t count) { if (h) CU(cudaMemcpyAsync(h, d, 4 * count, cudaMemcpyDeviceToHost, s)); return 0; }
  // T device -> fp32 host (bf16: widened on the device into an fp32 copy); h null: nothing
  int32_t downT(float* h, const void* d, size_t count) {
    if (!h || prec == PREC_F32) return downF(h, (const float*)d, count);
    float* f = nullptr; B2(upF(nullptr, count, &f)); k_nhwc_to_nchw_f32(prec, d, f, 1, 1, (int)count, s); return downF(h, f, count); }
  int32_t event(cudaEvent_t* e) { CU(cudaEventCreate(e)); events.push_back(*e); return 0; }
};
}  // namespace

extern "C" int32_t b2g_ctx_allreduce_test(b2g_ctx* c, float* host, int64_t n) {
  if (!c || !host || n < 1) return fail(B2G_ERR_ARG, "null"); if (!c->comm) return fail(B2G_ERR_NCCL, "no communicator"); CU(cudaSetDevice(c->device));
  HookMem m(c->stream, PREC_F32); float* d = nullptr;
  B2(m.upF(host, (size_t)n, &d));
  NC(g_nccl.ar(d, d, (size_t)n, 7, 0, c->comm, c->stream));
  B2(m.downF(host, d, (size_t)n)); CU(cudaStreamSynchronize(c->stream)); return 0;
}

// The tile-width / grid / split-count overrides of the tensor-core kernels hold for the hook's own launch loop only: reset right after it, and on
// every early return.
struct TcTestSchedule {
  TcTestSchedule(int bn, int max_ctas, int per_tap, int splits) { g_tc_test_bn = bn; g_tc_test_max_ctas = max_ctas; g_tc_test_per_tap = per_tap; g_tc_test_splits = splits; }
  ~TcTestSchedule() { reset(); }
  void reset() { g_tc_test_bn = 0; g_tc_test_max_ctas = 0; g_tc_test_per_tap = 0; g_tc_test_splits = 0; }
};
// What b2g_test_conv_ex takes for one (impl, kind): the precision and shapes its kernel runs, and the options it accepts.  Bits 1-3 of opts
// are the fused epilogues EPI_STATS / EPI_BNBWD / EPI_ACTBWD; bit 0 stands for an epi value no kernel has.
enum : unsigned { CO_STATS = 1u << EPI_STATS, CO_BNBWD = 1u << EPI_BNBWD, CO_ACTBWD = 1u << EPI_ACTBWD, CO_BIAS_ACT = 1u << 4, CO_SCALE = 1u << 5,
                  CO_POFF = 1u << 6, CO_BN = 1u << 7, CO_MAX_CTAS = 1u << 8, CO_PER_TAP = 1u << 9, CO_W_MN = 1u << 10, CO_SPLITS = 1u << 11,
                  CO_DEFER = 1u << 12, CO_DB = 1u << 13 };
struct ConvHookImpl {
  const char* kernel;                 // names the kernels in a refusal
  bool bf16, tma;                     // BF16 only; needs the tensor-map encoder (c->tc_ok)
  struct { bool (*shape)(const ConvGeom&); unsigned opts; } kind[3];      // fprop, dgrad, wgrad: the geometries it runs, the options it takes
};
static bool any_shape(const ConvGeom&) { return true; }
static bool dense_bwd_shape(const ConvGeom& g) { return dense_small_o_supported(g) || dense_small_k_supported(g); }
static bool tc_edge_conv_shape(const ConvGeom& g) { return edge_conv_small_cin_supported(g) && tc_edge_conv_supported(g); }
static bool tc_edge_wgrad_shape(const ConvGeom& g) { return edge_wgrad_small_cin_supported(g) && tc_edge_wgrad_supported(g); }
static const unsigned CO_TC = CO_STATS | CO_BNBWD | CO_ACTBWD | CO_BIAS_ACT | CO_SCALE | CO_BN | CO_MAX_CTAS | CO_PER_TAP;
static const ConvHookImpl kConvHook[6] = {
  {"SIMT kernel", false, false, {{any_shape, CO_BIAS_ACT | CO_SCALE | CO_POFF}, {any_shape, CO_BIAS_ACT | CO_SCALE | CO_POFF}, {any_shape, CO_POFF}}},
  {"tensor-core kernel (BF16, a working tensor-map encoder)", true, true,
   {{tc_fprop_supported, CO_TC | CO_W_MN}, {tc_dgrad_supported, CO_TC}, {tc_wgrad_supported, CO_POFF | CO_SPLITS | CO_DEFER}}},
  {"skinny-layer kernel (<= 4 image channels)", false, false,
   {{edge_conv_small_cin_supported, CO_BIAS_ACT | CO_POFF}, {edge_deconv_small_c_supported, CO_BIAS_ACT | CO_POFF}, {edge_wgrad_small_cin_supported, CO_POFF}}},
  // kind 1 is the pixel-shuffle deconv: the training step runs it wherever tc_deconv_ps_supported holds, also where the SIMT kernel has no
  // variant (O > 128)
  {"skinny-layer tensor-core kernel (BF16, <= 4 image channels, a working tensor-map encoder)", true, true,
   {{tc_edge_conv_shape, CO_BIAS_ACT | CO_MAX_CTAS}, {tc_deconv_ps_supported, CO_ACTBWD | CO_BIAS_ACT | CO_MAX_CTAS},
    {tc_edge_wgrad_shape, CO_POFF | CO_SPLITS | CO_DEFER | CO_DB}}},
  {"dense kernel (1x1 geometry: <= 4 output units, or a short reduction in the input / weight gradient)", false, false,
   {{dense_small_o_supported, CO_BIAS_ACT | CO_POFF}, {dense_bwd_shape, CO_BIAS_ACT | CO_POFF}, {dense_bwd_shape, CO_POFF}}},
  {"few-output conv kernel (BF16, O <= 4, C % 8 == 0, k x k)", true, false,
   {{head_conv_supported, CO_BIAS_ACT | CO_POFF}, {head_conv_supported, CO_BIAS_ACT | CO_POFF}, {head_conv_supported, CO_POFF | CO_SPLITS | CO_DB}}},
};
static constexpr int ik(int impl, int kind) { return 3 * impl + kind; }

extern "C" int32_t b2g_test_conv_ex(b2g_ctx* c, int32_t kind, int32_t impl, int32_t precision, const b2g_conv_geom* gg, const float* a_host, const float* b_host, float* out, int32_t iters, float* ms_per_iter,
                                    b2g_test_conv_opts* opt) {
  if (!c || !gg || !a_host || !b_host || !out) return fail(B2G_ERR_ARG, "null");
  if (kind < 0 || kind > 2 || impl < 0 || impl > 5) return fail(B2G_ERR_ARG, "kind %d / impl %d: kind is 0-2, impl 0-5", kind, impl);
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream; int prec = precision == B2G_PREC_BF16 ? PREC_BF16 : PREC_F32; size_t ts = prec_size(prec);
  ConvGeom g{gg->n, gg->h, gg->w, gg->c, gg->oh, gg->ow, gg->o, gg->kh, gg->kw, gg->sh, gg->sw, gg->ph, gg->pw};
  size_t nx = (size_t)g.N * g.H * g.W * g.C, ny = (size_t)g.N * g.OH * g.OW * g.O, nw = (size_t)g.O * g.KH * g.KW * g.C;
  // operands: kind 0: a = x (NHWC), b = w [O][KH][KW][C] -> out y ; kind 1: a = dy, b = w -> out dx ; kind 2: a = x, b = dy -> out dw (fp32)
  size_t na = kind == 1 ? ny : nx, nb = kind == 2 ? ny : nw, no = kind == 0 ? ny : kind == 1 ? nx : nw;
  const int oc = kind == 0 ? g.O : g.C;       // channels of the result (kinds 0 / 1)
  const ConvHookImpl& im = kConvHook[impl];
  if ((im.bf16 && prec != PREC_BF16) || (im.tma && !c->tc_ok) || !im.kind[kind].shape(g))
    return fail(B2G_ERR_UNSUPPORTED, "impl %d kind %d: no %s for this shape", impl, kind, im.kernel);
  const b2g_test_conv_opts none{}; const b2g_test_conv_opts& o = opt ? *opt : none;
  const struct { unsigned flag; bool set; const char* what; } asked[] = {
    {o.epi >= EPI_STATS && o.epi <= EPI_ACTBWD ? 1u << o.epi : 1u, o.epi != 0,
     "fused epilogue (epi 1-3: the tensor-core fprop / dgrad, impl 1 kind 0 / 1; epi 3: the pixel-shuffle deconv, impl 3 kind 1)"},
    {CO_BIAS_ACT, o.bias || o.act, "bias / activation (kinds 0 / 1; impl 4 kind 1 on its short-reduction kernel)"},
    {CO_SCALE, o.scale != nullptr, "scale (the SIMT and tensor-core fprop / dgrad, impl 0 / 1 kind 0 / 1)"},
    {CO_POFF, o.param_offset != 0, "param_offset (impl 0 / 2 / 4 / 5, and the tensor-core weight gradients, impl 1 / 3 kind 2)"},
    {CO_BN, o.bn != 0, "bn (the tile width of the tensor-core fprop / dgrad, impl 1 kind 0 / 1)"},
    {CO_MAX_CTAS, o.max_ctas != 0, "max_ctas (a grid cap of tc_conv_kernel and tc_edge_conv_kernel launches, impl 1 / 3 kind 0 / 1)"},
    {CO_PER_TAP, o.per_tap != 0, "per_tap (the tensor-core fprop / dgrad, impl 1 kind 0 / 1)"},
    {CO_W_MN, o.w_mn != 0, "w_mn (the [C][O] weight operand of the 1x1 tensor-core fprop, impl 1 kind 0)"},
    {CO_SPLITS, o.splits != 0, "splits (a forced split count of the weight gradients of impl 1 / 3 / 5)"},
    {CO_DEFER, o.defer != 0, "defer (the tensor-core weight gradients, impl 1 / 3 kind 2)"},
    {CO_DB, o.db != nullptr, "db (the bias column of the edge tensor-core and few-output weight gradients, impl 3 / 5 kind 2)"},
  };
  for (const auto& a : asked) if (a.set && !(im.kind[kind].opts & a.flag)) return fail(B2G_ERR_UNSUPPORTED, "impl %d kind %d takes no %s", impl, kind, a.what);
  if (o.param_offset < 0 || o.max_ctas < 0 || o.splits < 0)
    return fail(B2G_ERR_UNSUPPORTED, "param_offset %d, max_ctas %d, splits %d: none may be negative", o.param_offset, o.max_ctas, o.splits);
  if (o.bn && ((o.bn != 64 && o.bn != 128) || oc % o.bn))
    return fail(B2G_ERR_UNSUPPORTED, "bn %d: the tensor-core fprop / dgrad tile is 64 or 128 columns and must divide the %d output channels", o.bn, oc);
  // as in gemm_dgrad, a dense input gradient with an epilogue runs the short-reduction kernel
  if (impl == 4 && kind == 1 && (o.bias || o.act) && !dense_small_k_supported(g))
    return fail(B2G_ERR_UNSUPPORTED, "impl 4 kind 1: bias / activation run on the short-reduction kernel only, which has no variant for this shape");
  if (o.w_mn && (g.KH != 1 || g.KW != 1)) return fail(B2G_ERR_UNSUPPORTED, "w_mn: the [C][O] weight operand exists for the 1x1 tensor-core fprop only");
  const bool gemm = impl == 0 || impl == 2 || impl >= 4, tc_wg = kind == 2 && (impl == 1 || impl == 3);    // which globals name the launch
  const int force_splits = o.splits;
  size_t sc = std::max(std::max(std::max(k_simt_wgrad_scratch_floats(g), k_tc_wgrad_scratch_floats(g)), std::max(k_edge_wgrad_scratch_floats(g), k_tc_edge_wgrad_scratch_floats(g))), k_dense_small_o_wgrad_scratch_floats(g)) + 16;
  // a forced split count needs room for that many partials: [splits][dw] (tc_wgrad_kernel), [ctas][dw] + [ctas][db] with ctas <= splits (tc_edge_wgrad_kernel)
  if (force_splits) sc = std::max(sc, (size_t)force_splits * (impl == 1 || impl == 5 ? nw : (size_t)64 * 16 * g.C + 64) + 16);
  if (impl == 5) sc = std::max(sc, std::max(k_head_wgrad_scratch_floats(g), k_colsum_scratch_floats(g.O)) + 16);
  // param_offset: the fp32 weight operand (FP32, kinds 0 / 1) and the weight gradient and db (kind 2) start param_offset elements past the
  // 256-byte aligned base of their allocation, as W and dW do in a net's flattened parameter / gradient vectors
  const size_t woff = (prec == PREC_F32 && kind != 2) ? (size_t)o.param_offset : 0, dwoff = kind == 2 ? (size_t)o.param_offset : 0;
  // the fp32 copies, then the T operands: the layout bench.py's per-kernel times rest on (a different order moves some by ~3% on an H100)
  HookMem m(s, prec);
  float *fa, *fb, *fres, *scratch, *dbres = nullptr, *bias = nullptr, *scale = nullptr; void *ta, *tb, *to; __nv_bfloat16* wps = nullptr;
  B2(m.upF(a_host, na, &fa)); B2(m.upF(b_host, nb, &fb)); B2(m.upF(nullptr, no, &fres, dwoff)); B2(m.upF(nullptr, sc, &scratch));
  B2(m.dev(na, ts, &ta)); B2(m.dev(nb, ts, &tb, woff)); B2(m.dev(no, ts, &to)); B2(m.toT(fa, ta, na)); B2(m.toT(fb, tb, nb));
  if (impl == 3 && kind == 1) { B2(m.dev(k_tc_deconv_ps_weight_elems(g), 2, (void**)&wps)); k_pack_deconv_ps(fb, wps, g.O, g.C, s); }    // its packed weight operand
  if (o.db) B2(m.upF(nullptr, g.O, &dbres, dwoff));
  if (o.bias) B2(m.upF(o.bias, oc, &bias));
  if (o.scale) B2(m.upF(o.scale, oc, &scale));
  const int groups = o.groups > 0 ? o.groups : 1, act = o.act; const float alpha = o.alpha;
  TcEpi epi{}; unsigned long long* d_acc = nullptr;
  epi.mode = o.epi; epi.scale = scale; epi.imgs_per_group = g.N / groups; epi.act = act; epi.alpha = alpha;
  if (o.epi == EPI_STATS || o.epi == EPI_BNBWD) { B2(m.dev(k_bn_acc_elems(oc, groups), 8, (void**)&d_acc)); epi.acc = d_acc; }
  if (o.epi == EPI_BNBWD || o.epi == EPI_ACTBWD) {
    if (!o.aux) return fail(B2G_ERR_ARG, "epilogue %d needs aux", o.epi);
    void* aux = nullptr; B2(m.upT(o.aux, no, &aux)); epi.aux = (const __nv_bfloat16*)aux;
  }
  if (o.epi == EPI_BNBWD) {      // aux = the BatchNorm(+activation) output y, aux2 = its input z
    if (!o.aux2) return fail(B2G_ERR_ARG, "epilogue 2 needs aux2 (the BatchNorm input z)");
    void* aux2 = nullptr; B2(m.upT(o.aux2, no, &aux2)); epi.aux2 = (const __nv_bfloat16*)aux2;
  }
  const TcEpi* pe = o.epi || o.scale ? &epi : nullptr;
  const __nv_bfloat16 *ba = (const __nv_bfloat16*)ta, *bb = (const __nv_bfloat16*)tb; __nv_bfloat16* bo = (__nv_bfloat16*)to;
  ReduceList rl{}; ReduceList* prl = o.defer ? &rl : nullptr;
  cudaEvent_t e0, e1; B2(m.event(&e0)); B2(m.event(&e1));
  int reps = iters < 1 ? 1 : iters; int rc = 0, db_written = 0;
  g_tc_last_kernel = ""; g_tc_last_slab = false; g_tc_last_splits = 0; g_gemm_last_kernel = ""; g_gemm_last_splits = 0;
  TcTestSchedule schedule(o.bn, o.max_ctas, o.per_tap != 0, force_splits);
  for (int it = -1; it < reps; ++it) {       // it = -1: warm-up
    if (it == 0) CU(cudaEventRecord(e0, s));
    if (d_acc) CU(cudaMemsetAsync(d_acc, 0, 8 * k_bn_acc_elems(oc, groups), s));
    if (o.poison) CU(cudaMemsetAsync(to, 0xFF, ts * no, s));       // a tile this launch does not write reads back as NaN, not as the warm-up's values
    if (o.poison && kind == 2) { CU(cudaMemsetAsync(fres, 0xFF, 4 * no, s)); CU(cudaMemsetAsync(scratch, 0xFF, 4 * sc, s)); }   // fp32 NaN: dw and the split-K partials
    if (o.poison && dbres) CU(cudaMemsetAsync(dbres, 0xFF, 4 * (size_t)g.O, s));
    switch (ik(impl, kind)) {
      case ik(0, 0): k_simt_fprop(prec, prec, g, ta, tb, bias, to, act, alpha, s, scale); break;
      case ik(0, 1): k_simt_dgrad(prec, prec, g, ta, tb, bias, to, act, alpha, s, scale); break;
      case ik(0, 2): k_simt_wgrad(prec, g, ta, tb, fres, scratch, sc, 0, s); break;
      case ik(1, 0): rc = k_tc_fprop(g, ba, bb, bias, bo, act, alpha, s, pe, o.w_mn ? 1 : 0); break;
      case ik(1, 1): rc = k_tc_dgrad(g, ba, bb, bias, bo, act, alpha, s, pe); break;
      case ik(1, 2): rc = k_tc_wgrad(g, ba, bb, fres, scratch, sc, 0, s, prl); break;
      case ik(2, 0): k_edge_conv_small_cin(prec, prec, g, ta, tb, bias, to, act, alpha, s); break;
      case ik(2, 1): k_edge_deconv_small_c(prec, prec, g, ta, tb, bias, to, act, alpha, s); break;
      case ik(2, 2): k_edge_wgrad_small_cin(prec, g, ta, tb, fres, scratch, 0, s); break;
      case ik(3, 0): rc = k_tc_edge_conv(g, ba, bb, bias, bo, act, alpha, s); break;
      case ik(3, 1): rc = k_tc_deconv_ps(g, ba, wps, bias, bo, act, alpha, s, pe); break;
      case ik(3, 2): rc = k_tc_edge_wgrad(g, ba, bb, fres, dbres, scratch, sc, 0, s, prl); if (rc >= 0) { db_written = rc; rc = 0; } break;
      case ik(4, 0): k_dense_small_o_fwd(prec, prec, g, ta, tb, bias, to, act, alpha, s); break;
      case ik(4, 1):
        if (dense_small_o_supported(g) && !bias && !act) k_dense_small_o_dgrad(prec, prec, g, ta, tb, to, s);
        else k_dense_small_k_dgrad(prec, prec, g, ta, tb, bias, to, act, alpha, s);
        break;
      case ik(4, 2): if (dense_small_o_supported(g)) k_dense_small_o_wgrad(prec, g, ta, tb, fres, scratch, 0, s); else k_dense_small_k_wgrad(prec, g, ta, tb, fres, s); break;
      case ik(5, 0): k_head_fwd(g, ba, bb, bias, bo, act, alpha, s); break;
      case ik(5, 1): k_head_dgrad(g, ba, bb, bias, bo, act, alpha, s); break;
      case ik(5, 2): {      // the weight gradient's split sums as the backward pass runs them: one reduce-list launch; db = the column sums of dy
        ReduceList hl{};
        if (k_head_wgrad(g, ba, bb, fres, scratch, sc, force_splits, s, &hl)) { rc = -5; break; }
        const int hs = g_gemm_last_splits; k_reduce_multi(hl, s); g_gemm_last_splits = hs;
        if (dbres) { k_colsum(PREC_BF16, tb, g.N * g.OH * g.OW, g.O, scratch, dbres, 0, s); db_written = 1; }
        break;
      }
    }
    if (rc) break;
    if (o.defer) {      // the backward pass's one reduce-list launch over the partials the wgrad kernel left in scratch
      if (!rl.count) { rc = -4; break; }
      k_reduce_multi(rl, s); rl.count = 0;
    }
  }
  schedule.reset();
  CU(cudaEventRecord(e1, s));
  if (rc == -4) return fail(B2G_ERR_CUDA, "defer: the weight gradient queued no reduction");
  if (rc == -5) return fail(B2G_ERR_ARG, "splits %d: the partials do not fit the scratch", force_splits);
  if (rc) return fail(B2G_ERR_CUDA, "tensor-core kernel launch failed (%d)", rc);
  if (opt) {
    strncpy(opt->kernel, gemm ? g_gemm_last_kernel : g_tc_last_kernel, sizeof(opt->kernel) - 1); opt->kernel[sizeof(opt->kernel) - 1] = 0; opt->slab = g_tc_last_slab;
    opt->splits = gemm ? g_gemm_last_splits : tc_wg ? g_tc_last_splits : 0;
  }
  if (o.db) {
    if (!db_written) return fail(B2G_ERR_UNSUPPORTED, "the edge weight gradient produces no bias column for C = %d", g.C);
    B2(m.downF(o.db, dbres, g.O));
  }
  B2(kind == 2 ? m.downF(out, fres, no) : m.downT(out, to, no));
  CU(cudaStreamSynchronize(s)); CHECK_KERNELS();
  if (d_acc && o.stats) {      // [groups][2][C] doubles from the [groups][2][2][C] hi | lo words
    std::vector<long long> h(k_bn_acc_elems(oc, groups)); CU(cudaMemcpy(h.data(), d_acc, 8 * h.size(), cudaMemcpyDeviceToHost));
    for (int gi = 0; gi < groups; ++gi) for (int st = 0; st < 2; ++st) for (int ch = 0; ch < oc; ++ch)
      o.stats[((size_t)gi * 2 + st) * oc + ch] = (double)h[((size_t)(gi * 2 + st) * 2 + 0) * oc + ch] / 1024.0 + (double)h[((size_t)(gi * 2 + st) * 2 + 1) * oc + ch] / 1152921504606846976.0;
  }
  float ms = 0.f; CU(cudaEventElapsedTime(&ms, e0, e1)); if (ms_per_iter) *ms_per_iter = ms / reps;
  return 0;
}
extern "C" int32_t b2g_test_conv(b2g_ctx* c, int32_t kind, int32_t impl, int32_t precision, const b2g_conv_geom* gg, const float* a_host, const float* b_host, float* out, int32_t iters, float* ms_per_iter) {
  return b2g_test_conv_ex(c, kind, impl, precision, gg, a_host, b_host, out, iters, ms_per_iter, nullptr);
}

// One BatchNorm(+activation) forward and backward on [groups][rows][C] host tensors through the kernels the training step uses.
// path 0: k_bn_stats -> k_bn_apply -> k_bn_bwd (fp32 or bf16); path 1: the 128-bit accumulator kernels, backward statistics from
// k_bn_bwd_stats_acc; path 2: the accumulator kernels in the state the EPI_BNBWD epilogue leaves them (eps_out already holds dy' =
// eps * act', the backward accumulator holds (sum dy', sum dy'*z)).  g_gamma / g_beta are in/out (accumulated into, as in a backward pass).
extern "C" int32_t b2g_test_bn(b2g_ctx* c, int32_t precision, int32_t path, int32_t groups, int32_t rows, int32_t C, const float* x, const float* eps_out,
                               const float* gamma, const float* beta, const float* run_mean, const float* run_var, int32_t act, float alpha, float eps, float decay,
                               int32_t want_param_grads, float* y, float* eps_in, float* g_gamma, float* g_beta, float* g_mean, float* g_var, float* mean, float* invstd) {
  if (!c || !x || !eps_out || !gamma || !beta || !run_mean || !run_var || !y || !eps_in || !g_gamma || !g_beta || !g_mean || !g_var || !mean || !invstd) return fail(B2G_ERR_ARG, "null");
  if (groups < 1 || rows < 1 || C < 1 || path < 0 || path > 2) return fail(B2G_ERR_ARG, "bad BatchNorm test arguments");
  const int prec = precision == B2G_PREC_BF16 ? PREC_BF16 : PREC_F32;
  if (path != 0 && !k_bn_vec_ok(prec, C)) return fail(B2G_ERR_UNSUPPORTED, "the accumulator BatchNorm kernels need bf16 and C %% 8 == 0 with 256 %% (C/8) == 0 (C = %d)", C);
  CU(cudaSetDevice(c->device)); cudaStream_t s = c->stream;
  const size_t n = (size_t)groups * rows * C, gc = (size_t)groups * C, ts = prec_size(prec), na = k_bn_acc_elems(C, groups);
  HookMem m(s, prec);
  float *d_gamma, *d_beta, *d_rm, *d_rv, *d_gg, *d_gb, *d_gm, *d_gv, *d_mean, *d_is, *scratch, *coef, *unit; void *tx, *te, *ty, *tei; unsigned long long* acc;
  B2(m.upT(x, n, &tx)); B2(m.upT(eps_out, n, &te)); B2(m.dev(n, ts, &ty)); B2(m.dev(n, ts, &tei));
  B2(m.upF(gamma, C, &d_gamma)); B2(m.upF(beta, C, &d_beta)); B2(m.upF(run_mean, C, &d_rm)); B2(m.upF(run_var, C, &d_rv));
  B2(m.upF(g_gamma, C, &d_gg)); B2(m.upF(g_beta, C, &d_gb)); B2(m.upF(nullptr, C, &d_gm)); B2(m.upF(nullptr, C, &d_gv));
  B2(m.upF(nullptr, gc, &d_mean)); B2(m.upF(nullptr, gc, &d_is)); B2(m.upF(nullptr, k_bn_scratch_floats(C, groups), &scratch));
  B2(m.upF(nullptr, 4 * gc, &coef)); B2(m.upF(nullptr, 4 * gc, &unit)); B2(m.dev(2 * na, 8, (void**)&acc)); CU(cudaMemsetAsync(acc, 0, 8 * 2 * na, s));
  unsigned long long *acc_f = acc, *acc_b = acc + na;
  const int want = want_param_grads ? 1 : 0;
  if (path == 0) {
    k_bn_stats(prec, tx, rows, C, groups, scratch, d_mean, d_is, eps, d_rm, d_rv, d_gm, d_gv, decay, s);
    k_bn_apply(prec, tx, ty, rows, C, groups, d_mean, d_is, d_gamma, d_beta, act, alpha, s);
    k_bn_bwd(prec, tx, te, tei, rows, C, groups, d_mean, d_is, d_gamma, d_beta, act, alpha, scratch, d_gg, d_gb, want, s);
  } else {
    k_bn_stats_acc(tx, rows, C, groups, acc_f, s);
    k_bn_apply_acc(tx, ty, rows, C, groups, acc_f, d_gamma, d_beta, act, alpha, eps, coef, d_rm, d_rv, d_gm, d_gv, decay, s, 1);
    if (path == 1) k_bn_bwd_stats_acc(tx, te, rows, C, groups, coef, act, alpha, acc_b, s);
    else {      // (scale 1, shift 0, mean 0, invstd 1) makes xhat = z: the accumulator receives (sum dy', sum dy'*z) exactly as the epilogue writes it
      for (int g = 0; g < groups; ++g) for (int k = 0; k < 4; ++k) k_fill_f32(unit + (size_t)(g * 4 + k) * C, (k == 0 || k == 3) ? 1.f : 0.f, C, s);
      k_bn_bwd_stats_acc(tx, te, rows, C, groups, unit, ACT_IDENTITY, 0.f, acc_b, s);
    }
    k_bn_bwd_apply_acc(tx, te, tei, rows, C, groups, coef, act, alpha, path == 2 ? 1 : 0, acc_b, d_gg, d_gb, want, s, 1);
    for (int g = 0; g < groups; ++g) {
      cudaMemcpyAsync(d_mean + (size_t)g * C, coef + (size_t)(g * 4 + 2) * C, 4 * C, cudaMemcpyDeviceToDevice, s);
      cudaMemcpyAsync(d_is + (size_t)g * C, coef + (size_t)(g * 4 + 3) * C, 4 * C, cudaMemcpyDeviceToDevice, s);
    }
  }
  B2(m.downT(y, ty, n)); B2(m.downT(eps_in, tei, n));
  B2(m.downF(g_gamma, d_gg, C)); B2(m.downF(g_beta, d_gb, C)); B2(m.downF(g_mean, d_gm, C)); B2(m.downF(g_var, d_gv, C));
  B2(m.downF(mean, d_mean, gc)); B2(m.downF(invstd, d_is, gc));
  CU(cudaStreamSynchronize(s)); CHECK_KERNELS();
  return 0;
}

// Cross-replica BatchNorm on one device (include/b200gan.h b2g_test_bn_ex): every replica's accumulator kernels on its own rows, the
// replicas' 128-bit words summed on the host as the ncclUint64 sum all-reduce sums them (uint64, modulo 2^64), the sum handed back to every
// replica's buffer, the apply kernels run with replicas = R.
extern "C" int32_t b2g_test_bn_ex(b2g_ctx* c, const b2g_test_bn_opts* o, const float* x, const float* eps_out, const float* gamma, const float* beta,
                                  const float* run_mean, const float* run_var, const float* g_gamma0, const float* g_beta0, float* y, float* eps_in,
                                  float* g_gamma, float* g_beta, float* g_mean, float* g_var, float* mean, float* invstd) {
  if (!c || !o || !x || !eps_out || !gamma || !beta || !run_mean || !run_var || !g_gamma0 || !g_beta0 || !y || !eps_in || !g_gamma || !g_beta || !g_mean ||
      !g_var || !mean || !invstd) return fail(B2G_ERR_ARG, "null");
  const int R = o->replicas, groups = o->groups, rows = o->rows, C = o->C, path = o->path;
  if (R < 1 || groups < 1 || rows < 1 || C < 1 || path < 1 || path > 2) return fail(B2G_ERR_ARG, "bad cross-replica BatchNorm test arguments");
  if (!k_bn_vec_ok(PREC_BF16, C)) return fail(B2G_ERR_UNSUPPORTED, "the accumulator BatchNorm kernels need C %% 8 == 0 with 256 %% (C/8) == 0 (C = %d)", C);
  if ((int64_t)R * groups * rows * C > 0x7fffffff) return fail(B2G_ERR_ARG, "the cross-replica BatchNorm test takes at most 2^31 - 1 elements");
  CU(cudaSetDevice(c->device)); cudaStream_t s = c->stream;
  const size_t per = (size_t)groups * rows * C, n = per * R, gc = (size_t)groups * C, na = k_bn_acc_elems(C, groups);
  HookMem m(s, PREC_BF16);
  float *d_gamma, *d_beta, *d_rm, *d_rv, *d_gg, *d_gb, *d_gm, *d_gv, *coef, *unit; void *tx, *te, *ty, *tei; unsigned long long *acc_f, *acc_b;
  B2(m.upT(x, n, &tx)); B2(m.upT(eps_out, n, &te)); B2(m.dev(n, 2, &ty)); B2(m.dev(n, 2, &tei));
  B2(m.upF(gamma, C, &d_gamma)); B2(m.upF(beta, C, &d_beta)); B2(m.upF(run_mean, C, &d_rm)); B2(m.upF(run_var, C, &d_rv));
  B2(m.upF(nullptr, (size_t)R * C, &d_gg)); B2(m.upF(nullptr, (size_t)R * C, &d_gb)); B2(m.upF(nullptr, (size_t)R * C, &d_gm)); B2(m.upF(nullptr, (size_t)R * C, &d_gv));
  for (int r = 0; r < R; ++r) {
    CU(cudaMemcpyAsync(d_gg + (size_t)r * C, g_gamma0, 4 * C, cudaMemcpyHostToDevice, s)); CU(cudaMemcpyAsync(d_gb + (size_t)r * C, g_beta0, 4 * C, cudaMemcpyHostToDevice, s));
  }
  B2(m.upF(nullptr, 4 * gc * R, &coef)); B2(m.upF(nullptr, 4 * gc, &unit));
  B2(m.dev(na * R, 8, (void**)&acc_f)); B2(m.dev(na * R, 8, (void**)&acc_b)); CU(cudaMemsetAsync(acc_f, 0, 8 * na * R, s)); CU(cudaMemsetAsync(acc_b, 0, 8 * na * R, s));
  auto X = [&](void* t, int r) { return (void*)((__nv_bfloat16*)t + per * r); };
  auto CF = [&](int r) { return coef + 4 * gc * r; };
  std::vector<unsigned long long> words(na * R), sum(na);
  auto allreduce = [&](unsigned long long* acc) -> int32_t {      // every replica's buffer <- the word-wise sum of all of them
    CU(cudaMemcpyAsync(words.data(), acc, 8 * na * R, cudaMemcpyDeviceToHost, s)); CU(cudaStreamSynchronize(s));
    std::fill(sum.begin(), sum.end(), 0ull);
    for (int r = 0; r < R; ++r) for (size_t i = 0; i < na; ++i) sum[i] += words[na * r + i];
    for (int r = 0; r < R; ++r) CU(cudaMemcpyAsync(acc + na * r, sum.data(), 8 * na, cudaMemcpyHostToDevice, s));
    return 0;
  };
  const int want = o->want_param_grads ? 1 : 0;
  for (int r = 0; r < R; ++r) k_bn_stats_acc(X(tx, r), rows, C, groups, acc_f + na * r, s);
  B2(allreduce(acc_f));
  for (int r = 0; r < R; ++r)
    k_bn_apply_acc(X(tx, r), X(ty, r), rows, C, groups, acc_f + na * r, d_gamma, d_beta, o->act, o->alpha, o->eps, CF(r), d_rm, d_rv, d_gm + (size_t)r * C,
                   d_gv + (size_t)r * C, o->decay, s, R);
  if (path == 2)      // (scale 1, shift 0, mean 0, invstd 1): the accumulator receives (sum dy', sum dy'*z), as b2g_test_bn's path 2
    for (int g = 0; g < groups; ++g) for (int k = 0; k < 4; ++k) k_fill_f32(unit + (size_t)(g * 4 + k) * C, (k == 0 || k == 3) ? 1.f : 0.f, C, s);
  for (int r = 0; r < R; ++r) {
    if (path == 1) k_bn_bwd_stats_acc(X(tx, r), X(te, r), rows, C, groups, CF(r), o->act, o->alpha, acc_b + na * r, s);
    else k_bn_bwd_stats_acc(X(tx, r), X(te, r), rows, C, groups, unit, ACT_IDENTITY, 0.f, acc_b + na * r, s);
  }
  B2(allreduce(acc_b));
  for (int r = 0; r < R; ++r)
    k_bn_bwd_apply_acc(X(tx, r), X(te, r), X(tei, r), rows, C, groups, CF(r), o->act, o->alpha, path == 2 ? 1 : 0, acc_b + na * r, d_gg + (size_t)r * C,
                       d_gb + (size_t)r * C, want, s, R);
  B2(m.downT(y, ty, n)); B2(m.downT(eps_in, tei, n));
  B2(m.downF(g_gamma, d_gg, (size_t)R * C)); B2(m.downF(g_beta, d_gb, (size_t)R * C)); B2(m.downF(g_mean, d_gm, (size_t)R * C)); B2(m.downF(g_var, d_gv, (size_t)R * C));
  std::vector<float> cf(4 * gc * R); CU(cudaMemcpyAsync(cf.data(), coef, 4 * 4 * gc * R, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s)); CHECK_KERNELS();
  for (int r = 0; r < R; ++r) for (int g = 0; g < groups; ++g) {      // coef rows per group: scale, beta, mean, invstd
    memcpy(mean + ((size_t)r * groups + g) * C, cf.data() + 4 * gc * r + (size_t)(g * 4 + 2) * C, 4 * C);
    memcpy(invstd + ((size_t)r * groups + g) * C, cf.data() + 4 * gc * r + (size_t)(g * 4 + 3) * C, 4 * C);
  }
  return 0;
}

// One DropoutLayer forward (pass counter `pass`, advanced by the kernel) and backward on rows*h*w*c host tensors in NHWC element order,
// through the kernels the training step uses.
extern "C" int32_t b2g_test_dropout(b2g_ctx* c, int32_t precision, uint64_t seed, int32_t layer, int32_t rank, int64_t pass, int32_t rows, int32_t h, int32_t w, int32_t ch,
                                    float p, const float* x, const float* dy, float* y, float* dx) {
  if (!c || !x || !dy || !y || !dx) return fail(B2G_ERR_ARG, "null");
  if (!(p > 0.f && p <= 1.f)) return fail(B2G_ERR_ARG, "dropout retain probability %g outside (0, 1]", (double)p);
  if (rows < 1 || h < 1 || w < 1 || ch < 1 || layer < 0 || layer > 0xffff || rank < 0 || rank > 0xffff || pass < 0) return fail(B2G_ERR_ARG, "bad dropout test arguments");
  const size_t n = (size_t)rows * h * w * ch;
  if (n > 0x7fffffff) return fail(B2G_ERR_UNSUPPORTED, "the dropout test hook takes at most 2^31 - 1 elements (%zu)", n);
  const int prec = precision == B2G_PREC_BF16 ? PREC_BF16 : PREC_F32; const size_t ts = prec_size(prec);
  CU(cudaSetDevice(c->device)); cudaStream_t s = c->stream;
  HookMem m(s, prec);
  void *tx, *te, *ty; uint32_t* mask; unsigned long long* dpass; unsigned* ticket;
  const unsigned long long p0 = (unsigned long long)pass;
  B2(m.upT(x, n, &tx)); B2(m.upT(dy, n, &te)); B2(m.dev(n, ts, &ty)); B2(m.dev((n + 31) / 32, 4, (void**)&mask));
  B2(m.dev(1, sizeof(p0), (void**)&dpass)); B2(m.dev(1, sizeof(unsigned), (void**)&ticket));
  CU(cudaMemcpyAsync(dpass, &p0, sizeof(p0), cudaMemcpyHostToDevice, s)); CU(cudaMemsetAsync(ticket, 0, sizeof(unsigned), s));
  const DropoutArgs a = make_dropout_args(seed, layer, rank, p);
  k_dropout_fwd(prec, tx, ty, mask, n, a, dpass, ticket, 1, s);
  k_dropout_bwd(prec, te, te, mask, n, a.scale, s);
  unsigned long long p1 = 0;
  B2(m.downT(y, ty, n)); B2(m.downT(dx, te, n)); CU(cudaMemcpyAsync(&p1, dpass, sizeof(p1), cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s)); CHECK_KERNELS();
  if (p1 != p0 + 1) return fail(B2G_ERR_CUDA, "dropout test: the forward left the pass counter at %llu, expected %llu", p1, p0 + 1);
  return 0;
}

// One DropoutLayer forward and backward of any b2g_dropout_kind, as b2g_test_dropout (include/b200gan.h b2g_test_dropout_kind).
extern "C" int32_t b2g_test_dropout_kind(b2g_ctx* c, int32_t precision, int32_t kind, uint64_t seed, int32_t layer, int32_t rank, int64_t pass, int32_t rows,
                                         int32_t h, int32_t w, int32_t ch, float v, const float* x, const float* dy, float* y, float* dx) {
  if (!c || !x || !dy || !y || !dx) return fail(B2G_ERR_ARG, "null");
  bool identity = false;
  switch (kind) {
    case B2G_DROPOUT: case B2G_DROPOUT_ALPHA: case B2G_DROPOUT_SPATIAL:
      if (!(v > 0.f && v <= 1.f)) return fail(B2G_ERR_ARG, "dropout retain probability %g outside (0, 1]", (double)v);
      identity = v >= 1.f; break;
    case B2G_DROPOUT_GAUSSIAN_DROPOUT: if (!(v >= 0.f && v < 1.f)) return fail(B2G_ERR_ARG, "GaussianDropout rate %g outside [0, 1)", (double)v); identity = v == 0.f; break;
    case B2G_DROPOUT_GAUSSIAN_NOISE: if (!(v >= 0.f && std::isfinite(v))) return fail(B2G_ERR_ARG, "GaussianNoise stddev %g not finite and >= 0", (double)v); identity = v == 0.f; break;
    default: return fail(B2G_ERR_ARG, "unknown dropout kind %d", kind);
  }
  if (kind == B2G_DROPOUT) return b2g_test_dropout(c, precision, seed, layer, rank, pass, rows, h, w, ch, v, x, dy, y, dx);
  if (rows < 1 || h < 1 || w < 1 || ch < 1 || layer < 0 || layer > 0xffff || rank < 0 || rank > 0xffff || pass < 0) return fail(B2G_ERR_ARG, "bad dropout test arguments");
  const size_t n = (size_t)rows * h * w * ch;
  if (n > 0x7fffffff) return fail(B2G_ERR_UNSUPPORTED, "the dropout test hook takes at most 2^31 - 1 elements (%zu)", n);
  if (identity) { memcpy(y, x, n * sizeof(float)); memcpy(dx, dy, n * sizeof(float)); return 0; }
  const int prec = precision == B2G_PREC_BF16 ? PREC_BF16 : PREC_F32; const size_t ts = prec_size(prec);
  CU(cudaSetDevice(c->device)); cudaStream_t s = c->stream;
  HookMem m(s, prec);
  void *tx, *te, *ty; uint32_t* mask; unsigned long long* dpass; NoiseRec* rec; unsigned* ticket;
  const unsigned long long p0 = (unsigned long long)pass;
  B2(m.upT(x, n, &tx)); B2(m.upT(dy, n, &te)); B2(m.dev(n, ts, &ty)); B2(m.dev((n + 31) / 32, 4, (void**)&mask));
  B2(m.dev(1, sizeof(p0), (void**)&dpass)); B2(m.dev(1, sizeof(NoiseRec), (void**)&rec)); B2(m.dev(1, sizeof(unsigned), (void**)&ticket));
  CU(cudaMemcpyAsync(dpass, &p0, sizeof(p0), cudaMemcpyHostToDevice, s)); CU(cudaMemsetAsync(ticket, 0, sizeof(unsigned), s));
  const NoiseArgs a = make_noise_args(seed, layer, rank, kind, v, h * w, ch);
  k_noise_fwd(prec, kind, tx, ty, mask, rec, n, a, NoiseSched{}, dpass, ticket, 1, s);
  k_noise_bwd(prec, kind, te, te, mask, rec, n, a, NoiseSched{}, s);
  unsigned long long p1 = 0;
  B2(m.downT(y, ty, n)); B2(m.downT(dx, te, n)); CU(cudaMemcpyAsync(&p1, dpass, sizeof(p1), cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s)); CHECK_KERNELS();
  if (p1 != p0 + 1) return fail(B2G_ERR_CUDA, "dropout test: the forward left the pass counter at %llu, expected %llu", p1, p0 + 1);
  return 0;
}

// One reduction / loss / element-wise kernel through its production wrapper on host tensors (include/b200gan.h, b2g_test_ew).  The kernel
// names come from the wrappers (g_ew_last_kernel): this hook never decides which path a shape takes.
// b2g_test_pool runs through the same code as two private ops, its own options in po (null for every b2g_test_ew call)
enum { EW_POOL2D = 100, EW_GLOBAL_POOL = 101 };
static int32_t test_ew_impl(b2g_ctx* c, int32_t precision, b2g_test_ew_opts* o, b2g_test_pool_opts* po, const float* in0, const float* in1, float* out0,
                            float* out1, float* out2) {
  if (!c || !o) return fail(B2G_ERR_ARG, "null");
  const int prec = precision == B2G_PREC_BF16 ? PREC_BF16 : PREC_F32; const size_t ts = prec_size(prec);
  const int off = o->offset;
  if (off < 0 || off > 64) return fail(B2G_ERR_ARG, "offset %d outside [0, 64]", off);
  if (o->poison && o->accumulate) return fail(B2G_ERR_ARG, "poison would overwrite the initial destination accumulate adds to");
  CU(cudaSetDevice(c->device)); cudaStream_t s = c->stream;
  HookMem m(s, prec);
  auto poison = [&](void* d, size_t bytes) -> int32_t { if (o->poison) CU(cudaMemsetAsync(d, 0xFF, bytes, s)); return 0; };     // fp32 and bf16 NaN
  std::string names;
  auto ran = [&]() { if (!names.empty()) names += ","; names += g_ew_last_kernel; g_ew_last_kernel = ""; };
  const int64_t lim = 0x7fffffff;
  g_ew_last_kernel = "";
  switch (o->op) {
    case B2G_EW_REDUCE_SPLITS: {
      if (!in0 || o->n < 1 || o->n > lim || o->splits < 1 || o->stride < o->n || (o->accumulate && !in1)) return fail(B2G_ERR_ARG, "bad REDUCE_SPLITS arguments");
      float *src = nullptr, *dst = nullptr; B2(m.upF(in0, (size_t)o->splits * o->stride, &src, off)); B2(m.upF(in1, (size_t)o->n, &dst, off)); B2(poison(dst, 4 * o->n));
      k_reduce_splits(src, dst, (size_t)o->n, o->splits, (size_t)o->stride, o->accumulate ? 1 : 0, s); ran();
      B2(m.downF(out0, dst, (size_t)o->n));
      break;
    }
    case B2G_EW_REDUCE_MULTI: {
      if (!in0 || o->n < 1 || o->n > lim || o->n_jobs < 1 || o->n_jobs > ReduceList::MAX_JOBS || !o->jobs) return fail(B2G_ERR_ARG, "bad REDUCE_MULTI arguments");
      const b2g_ew_reduce_job* J = o->jobs;
      auto src_end = [&](int i) { return J[i].src_off + (int64_t)(J[i].splits - 1) * J[i].stride + J[i].n; };
      for (int i = 0; i < o->n_jobs; ++i) {
        if (J[i].n < 1 || J[i].splits < 1 || J[i].stride < J[i].n || J[i].src_off < 0 || J[i].dst_off < 0 || src_end(i) > o->n || J[i].dst_off + J[i].n > o->n)
          return fail(B2G_ERR_ARG, "reduce job %d outside the buffer", i);
        for (int k = 0; k < o->n_jobs; ++k) {      // a destination shared with any source or another destination would race
          const bool src_hit = J[i].dst_off < src_end(k) && J[k].src_off < J[i].dst_off + J[i].n;
          const bool dst_hit = k != i && J[i].dst_off < J[k].dst_off + J[k].n && J[k].dst_off < J[i].dst_off + J[i].n;
          if (src_hit || dst_hit) return fail(B2G_ERR_ARG, "reduce job %d's destination overlaps job %d", i, k);
        }
      }
      float* buf = nullptr; B2(m.upF(in0, (size_t)o->n, &buf, off));
      ReduceList rl{};
      for (int i = 0; i < o->n_jobs; ++i) {
        reduce_list_push(&rl, buf + J[i].src_off, buf + J[i].dst_off, J[i].n, J[i].splits, J[i].stride);
        o->jobs[i].wide = rl.jobs[i].blocks < 0 ? 1 : 0;
        B2(poison(buf + J[i].dst_off, 4 * (size_t)J[i].n));
      }
      if (rl.count != o->n_jobs) return fail(B2G_ERR_ARG, "the reduce list took %d of %d jobs", rl.count, o->n_jobs);
      k_reduce_multi(rl, s); ran();
      B2(m.downF(out0, buf, (size_t)o->n));
      break;
    }
    case B2G_EW_COLSUM: {
      if (!in0 || o->rows < 1 || o->cols < 1 || (int64_t)o->rows * o->cols > lim || (o->accumulate && !in1)) return fail(B2G_ERR_ARG, "bad COLSUM arguments");
      void* x = nullptr; float *out = nullptr, *scratch = nullptr; B2(m.upT(in0, (size_t)o->rows * o->cols, &x, off)); B2(m.upF(in1, (size_t)o->cols, &out, off)); B2(poison(out, 4 * (size_t)o->cols));
      B2(m.upF(nullptr, k_colsum_scratch_floats(o->cols), &scratch));
      k_colsum(prec, x, o->rows, o->cols, scratch, out, o->accumulate ? 1 : 0, s); ran();
      B2(m.downF(out0, out, (size_t)o->cols));
      break;
    }
    case B2G_EW_XENT: {
      const size_t n = (size_t)o->rows * o->groups;
      if (!in0 || !in1 || o->rows < 1 || o->groups < 1 || (int64_t)n > lim) return fail(B2G_ERR_ARG, "bad XENT arguments");
      void *z = nullptr, *dz = nullptr; float *y = nullptr, *loss = nullptr; B2(m.upT(in0, n, &z, off)); B2(m.upF(in1, n, &y, off)); B2(m.dev(n, ts, &dz, off)); B2(m.upF(nullptr, (size_t)o->groups, &loss, off));
      B2(poison(dz, ts * n)); B2(poison(loss, 4 * (size_t)o->groups));
      k_xent(prec, z, y, dz, loss, o->rows, o->groups, o->clip_eps, s); ran();
      B2(m.downT(out0, dz, n)); B2(m.downF(out1, loss, (size_t)o->groups));
      break;
    }
    case B2G_EW_SOFTMAX_XENT: {
      const size_t n = (size_t)o->rows * o->cols;
      if (!in0 || o->rows < 1 || o->cols < 1 || (int64_t)n > lim) return fail(B2G_ERR_ARG, "bad SOFTMAX_XENT arguments");
      void *z = nullptr, *dz = nullptr, *p = nullptr; float *y = nullptr, *loss = nullptr; B2(m.upT(in0, n, &z, off)); if (in1) B2(m.upF(in1, n, &y, off));
      B2(m.dev(n, ts, &dz, off)); B2(m.dev(n, ts, &p, off)); B2(m.upF(nullptr, 1, &loss, off));
      B2(poison(dz, ts * n)); B2(poison(p, ts * n)); B2(poison(loss, 4));
      k_softmax_xent(prec, z, y, y ? dz : nullptr, p, y ? loss : nullptr, o->rows, o->cols, s); ran();       // no labels: the inference call
      B2(m.downT(out0, dz, n)); B2(m.downF(out1, loss, 1)); B2(m.downT(out2, p, n));
      break;
    }
    case B2G_EW_LOSS: {
      const size_t per = (size_t)o->rows * o->cols, n = per * o->groups;
      if (!in0 || !in1 || o->rows < 1 || o->cols < 1 || o->groups < 1 || (int64_t)n > lim || o->loss < B2G_LOSS_MSE || o->loss > B2G_LOSS_WASSERSTEIN ||
          o->act < B2G_ACT_IDENTITY || o->act > B2G_ACT_LRELU) return fail(B2G_ERR_ARG, "bad LOSS arguments");
      void *z = nullptr, *dz = nullptr; float *y = nullptr, *loss = nullptr; double* partial = nullptr; unsigned* ticket = nullptr;
      B2(m.upT(in0, n, &z, off)); B2(m.upF(in1, n, &y, off)); B2(m.dev(n, ts, &dz, off)); B2(m.upF(nullptr, (size_t)o->groups, &loss, off));
      B2(m.dev((size_t)o->groups * k_loss_blocks(per, o->groups), 8, (void**)&partial, off)); B2(m.dev(1, 4, (void**)&ticket, off)); CU(cudaMemsetAsync(ticket, 0, 4, s));
      B2(poison(dz, ts * n)); B2(poison(loss, 4 * (size_t)o->groups));
      k_loss(prec, o->loss, o->act, o->alpha, z, y, dz, loss, o->rows, o->cols, o->groups, partial, ticket, s); ran();
      B2(m.downT(out0, dz, n)); B2(m.downF(out1, loss, (size_t)o->groups));
      break;
    }
    case B2G_EW_CNN_XENT: case B2G_EW_CNN_SOFTMAX_XENT: {
      const bool sm = o->op == B2G_EW_CNN_SOFTMAX_XENT;
      const size_t per = (size_t)o->rows * o->cols, n = per * o->groups;
      if (!in0 || (!in1 && !sm) || o->rows < 1 || o->cols < 1 || o->groups < 1 || (int64_t)n > lim) return fail(B2G_ERR_ARG, "bad CNN loss arguments");
      const int bpg = sm ? k_cnn_softmax_blocks(o->rows, o->groups) : k_loss_blocks(per, o->groups);
      void *z = nullptr, *dz = nullptr, *p = nullptr; float *y = nullptr, *loss = nullptr; double* partial = nullptr; unsigned* ticket = nullptr;
      B2(m.upT(in0, n, &z, off)); if (in1) B2(m.upF(in1, n, &y, off)); B2(m.dev(n, ts, &dz, off)); B2(m.dev(n, ts, &p, off)); B2(m.upF(nullptr, (size_t)o->groups, &loss, off));
      B2(m.dev((size_t)o->groups * bpg, 8, (void**)&partial, off)); B2(m.dev(1, 4, (void**)&ticket, off)); CU(cudaMemsetAsync(ticket, 0, 4, s));
      B2(poison(dz, ts * n)); B2(poison(p, ts * n)); B2(poison(loss, 4 * (size_t)o->groups));
      if (sm) k_cnn_softmax_xent(prec, z, y, y ? dz : nullptr, p, y ? loss : nullptr, o->rows, o->cols, o->groups, partial, ticket, s);     // no labels: the inference call
      else k_cnn_xent(prec, z, y, dz, loss, per, o->groups, o->clip_eps, partial, ticket, s);
      ran();
      B2(m.downT(out0, dz, n)); B2(m.downF(out1, loss, (size_t)o->groups)); if (sm) B2(m.downT(out2, p, n));
      unsigned t = 1; CU(cudaMemcpyAsync(&t, ticket, 4, cudaMemcpyDeviceToHost, s)); CU(cudaStreamSynchronize(s));
      if (t != 0) return fail(B2G_ERR_CUDA, "CNN loss: the kernel left its ticket word at %u", t);
      break;
    }
    case B2G_EW_VERTEX_FWD: case B2G_EW_VERTEX_BWD: case B2G_EW_SKIP_ADD: {
      const size_t n = (size_t)o->n; const int order = o->groups;
      if (!in0 || !in1 || o->n < 1 || o->n > lim) return fail(B2G_ERR_ARG, "bad vertex arguments");
      if (o->op != B2G_EW_SKIP_ADD && (o->act < B2G_EW_OP_ADD || o->act > B2G_EW_OP_MAX || (order != 0 && order != 1))) return fail(B2G_ERR_ARG, "bad vertex op / order");
      if (o->op == B2G_EW_VERTEX_FWD) {
        void *a = nullptr, *b = nullptr, *y = nullptr; B2(m.upT(in0, n, &a, off)); B2(m.upT(in1, n, &b, off)); B2(m.dev(n, ts, &y, off)); B2(poison(y, ts * n));
        k_vertex_ew_fwd(prec, o->act, order ? b : a, order ? a : b, y, n, s); ran();
        B2(m.downT(out0, y, n));
      } else if (o->op == B2G_EW_VERTEX_BWD) {
        void *sp = nullptr, *sk = nullptr, *e = nullptr; float* acc = nullptr;
        B2(m.upT(in0, n, &sp, off)); B2(m.upT(in0 + n, n, &sk, off)); B2(m.upT(in1, n, &e, off)); B2(m.upF(o->accumulate ? in1 + n : nullptr, n, &acc, off)); B2(poison(acc, 4 * n));
        k_vertex_ew_bwd(prec, o->act, order, e, sp, sk, acc, o->accumulate ? 1 : 0, n, s); ran();
        B2(m.downT(out0, e, n)); B2(m.downF(out1, acc, n));
      } else {
        void* e = nullptr; float* acc = nullptr; B2(m.upT(in0, n, &e, off)); B2(m.upF(in1, n, &acc, off));
        k_skip_add(prec, e, acc, n, s); ran();
        B2(m.downT(out0, e, n));
      }
      break;
    }
    case B2G_EW_MERGE_FWD: case B2G_EW_MERGE_BWD: {
      const int Cs = o->cols, Ck = o->C, order = o->groups; const size_t P = (size_t)o->rows, nt = P * (Cs + Ck);
      if (!in0 || (!in1 && (o->op == B2G_EW_MERGE_FWD || o->accumulate)) || o->rows < 1 || Cs < 1 || Ck < 1 || (order != 0 && order != 1) || nt > (size_t)lim)
        return fail(B2G_ERR_ARG, "bad merge arguments");
      if (o->op == B2G_EW_MERGE_FWD) {
        void *a = nullptr, *b = nullptr, *y = nullptr; B2(m.upT(in0, P * Cs, &a, off)); B2(m.upT(in1, P * Ck, &b, off)); B2(m.dev(nt, ts, &y, off)); B2(poison(y, ts * nt));
        if (order) k_merge_fwd(prec, b, a, y, P, Ck, Cs, s); else k_merge_fwd(prec, a, b, y, P, Cs, Ck, s);
        ran(); B2(m.downT(out0, y, nt));
      } else {
        void *e = nullptr, *d = nullptr; float* acc = nullptr;
        B2(m.upT(in0, nt, &e, off)); B2(m.dev(P * Cs, ts, &d, off)); B2(m.upF(o->accumulate ? in1 : nullptr, P * Ck, &acc, off)); B2(poison(d, ts * P * Cs)); B2(poison(acc, 4 * P * Ck));
        k_merge_bwd(prec, e, d, acc, P, order ? Ck : Cs, order ? Cs : Ck, order == 0, o->accumulate ? 1 : 0, s); ran();
        B2(m.downT(out0, d, P * Cs)); B2(m.downF(out1, acc, P * Ck));
      }
      break;
    }
    case B2G_EW_ACT_FWD: case B2G_EW_ACT_BWD: {
      const size_t n = (size_t)o->n; const bool bwd = o->op == B2G_EW_ACT_BWD;
      if (!in0 || (bwd && !in1) || o->n < 1 || o->n > lim || o->act < B2G_ACT_IDENTITY || o->act > B2G_ACT_LRELU) return fail(B2G_ERR_ARG, "bad activation arguments");
      void *a = nullptr, *e = nullptr, *r = nullptr; B2(m.upT(in0, n, &a, off));
      if (bwd) B2(m.upT(in1, n, &e, off));
      if (bwd && o->in_place) r = e;
      else { B2(m.dev(n, ts, &r, off)); B2(poison(r, ts * n)); }
      if (bwd) k_act_bwd_from_output(prec, a, e, r, n, o->act, o->alpha, s);      // in place: eps_in == eps_out, as the backward pass calls it
      else k_act_fwd(prec, a, r, n, o->act, o->alpha, s);
      ran();
      B2(m.downT(out0, r, n));
      break;
    }
    case B2G_EW_ACT_EXT_FWD: case B2G_EW_ACT_EXT_BWD: {
      const size_t n = (size_t)o->n; const bool bwd = o->op == B2G_EW_ACT_EXT_BWD;
      if (!in0 || (bwd && !in1) || o->n < 1 || o->n > lim || !act_ext_kind(o->act) || !std::isfinite(o->alpha)) return fail(B2G_ERR_ARG, "bad activation arguments");
      void *z = nullptr, *r = nullptr; B2(m.upT(in0, n, &z, off));
      if (bwd) B2(m.upT(in1, n, &r, off));      // eps_out, overwritten in place with eps_in
      else { B2(m.dev(n, ts, &r, off)); B2(poison(r, ts * n)); }
      if (bwd) k_act_ext_bwd(prec, o->act, o->alpha, z, r, n, s);
      else k_act_ext_fwd(prec, o->act, o->alpha, z, r, n, s);
      ran();
      B2(m.downT(out0, r, n));
      break;
    }
    case B2G_EW_MAXPOOL: {
      if (!in0 || !in1 || o->N < 1 || o->C < 1 || o->KH < 1 || o->KW < 1 || o->SH < 1 || o->SW < 1 || o->H < o->KH || o->W < o->KW || o->KH * o->KW > 255)
        return fail(B2G_ERR_ARG, "bad MAXPOOL arguments");
      const int OH = (o->H - o->KH) / o->SH + 1, OW = (o->W - o->KW) / o->SW + 1;
      const size_t ni = (size_t)o->N * o->H * o->W * o->C, no = (size_t)o->N * OH * OW * o->C;
      if (ni > (size_t)lim) return fail(B2G_ERR_ARG, "MAXPOOL input too large");
      void *x = nullptr, *eo = nullptr, *y = nullptr, *ei = nullptr; uint8_t* arg = nullptr;
      B2(m.upT(in0, ni, &x, off)); B2(m.upT(in1, no, &eo, off)); B2(m.dev(no, ts, &y, off)); B2(m.dev(ni, ts, &ei, off)); B2(m.dev(no, 1, (void**)&arg, off));
      B2(poison(y, ts * no)); B2(poison(ei, ts * ni)); B2(poison(arg, no));        // 0xFF: no window of <= 255 elements has that argmax
      k_maxpool_fwd(prec, x, y, arg, o->N, o->H, o->W, o->C, OH, OW, o->KH, o->KW, o->SH, o->SW, s); ran();
      k_maxpool_bwd(prec, eo, arg, ei, o->N, o->H, o->W, o->C, OH, OW, o->KH, o->KW, o->SH, o->SW, s); ran();
      B2(m.downT(out0, y, no)); B2(m.downT(out1, ei, ni));
      if (out2) {
        std::vector<uint8_t> h(no); CU(cudaMemcpyAsync(h.data(), arg, no, cudaMemcpyDeviceToHost, s)); CU(cudaStreamSynchronize(s));
        for (size_t i = 0; i < no; ++i) out2[i] = (float)h[i];
      }
      break;
    }
    case EW_POOL2D: {
      if (!po) return fail(B2G_ERR_ARG, "unknown op %d", o->op);
      if (!in0 || !in1 || o->N < 1 || o->H < 1 || o->W < 1 || o->C < 1 || o->KH < 1 || o->KW < 1 || o->SH < 1 || o->SW < 1 || po->PH < 0 || po->PW < 0 ||
          po->PH >= o->KH || po->PW >= o->KW || o->H + 2 * po->PH < o->KH || o->W + 2 * po->PW < o->KW || po->pool < B2G_POOL_AVG || po->pool > B2G_POOL_PNORM ||
          (po->pool == B2G_POOL_PNORM && !(po->pnorm >= 1.f && po->pnorm <= 1024.f && po->pnorm == floorf(po->pnorm))))
        return fail(B2G_ERR_ARG, "bad POOL2D arguments");
      const int OH = (o->H + 2 * po->PH - o->KH) / o->SH + 1, OW = (o->W + 2 * po->PW - o->KW) / o->SW + 1;
      const size_t ni = (size_t)o->N * o->H * o->W * o->C, no = (size_t)o->N * OH * OW * o->C;
      if (ni > (size_t)lim || no > (size_t)lim) return fail(B2G_ERR_ARG, "POOL2D tensors too large");
      void *x = nullptr, *eo = nullptr, *y = nullptr, *ei = nullptr;
      B2(m.upT(in0, ni, &x, off)); B2(m.upT(in1, no, &eo, off)); B2(m.dev(no, ts, &y, off)); B2(m.dev(ni, ts, &ei, off)); B2(poison(y, ts * no)); B2(poison(ei, ts * ni));
      const int pn = po->pool == B2G_POOL_PNORM ? (int)po->pnorm : 0;
      k_pool2d_fwd(prec, po->pool, pn, x, y, o->N, o->H, o->W, o->C, OH, OW, o->KH, o->KW, o->SH, o->SW, po->PH, po->PW, s); ran();
      k_pool2d_bwd(prec, po->pool, pn, eo, x, y, ei, o->N, o->H, o->W, o->C, OH, OW, o->KH, o->KW, o->SH, o->SW, po->PH, po->PW, s); ran();
      B2(m.downT(out0, y, no)); B2(m.downT(out1, ei, ni));
      break;
    }
    case EW_GLOBAL_POOL: {
      if (!po) return fail(B2G_ERR_ARG, "unknown op %d", o->op);
      if (!in0 || !in1 || o->N < 1 || o->H < 1 || o->W < 1 || o->C < 1 || po->pool < B2G_POOL_MAX || po->pool > B2G_POOL_PNORM ||
          (po->pool == B2G_POOL_PNORM && !(po->pnorm >= 1.f && po->pnorm <= 1024.f && po->pnorm == floorf(po->pnorm))))
        return fail(B2G_ERR_ARG, "bad GLOBAL_POOL arguments");
      const int HW = o->H * o->W;
      const size_t ni = (size_t)o->N * HW * o->C, no = (size_t)o->N * o->C;
      if (ni > (size_t)lim) return fail(B2G_ERR_ARG, "GLOBAL_POOL input too large");
      void *x = nullptr, *eo = nullptr, *y = nullptr, *ei = nullptr; int32_t *idx = nullptr, *part_idx = nullptr; float* part = nullptr; unsigned* ticket = nullptr;
      B2(m.upT(in0, ni, &x, off)); B2(m.upT(in1, no, &eo, off)); B2(m.dev(no, ts, &y, off)); B2(m.dev(ni, ts, &ei, off)); B2(m.dev(no, 4, (void**)&idx, off));
      const size_t np = std::max<size_t>(1, k_global_pool_partial_elems(prec, o->N, HW, o->C));
      B2(m.dev(np, 4, (void**)&part, off)); B2(m.dev(np, 4, (void**)&part_idx, off)); B2(m.dev(1, 4, (void**)&ticket, off)); CU(cudaMemsetAsync(ticket, 0, 4, s));
      B2(poison(y, ts * no)); B2(poison(ei, ts * ni)); B2(poison(idx, 4 * no));      // 0xFF..: index -1, no pixel
      const int pn = po->pool == B2G_POOL_PNORM ? (int)po->pnorm : 0;
      k_global_pool_fwd(prec, po->pool, pn, x, y, po->pool == B2G_POOL_MAX ? idx : nullptr, o->N, HW, o->C, part, part_idx, ticket, s); ran();
      po->splits = g_pool_last_splits;
      k_global_pool_bwd(prec, po->pool, pn, eo, x, y, idx, ei, o->N, HW, o->C, s); ran();
      B2(m.downT(out0, y, no)); B2(m.downT(out1, ei, ni));
      if (out2) {
        std::vector<int32_t> h(no); CU(cudaMemcpyAsync(h.data(), idx, 4 * no, cudaMemcpyDeviceToHost, s)); CU(cudaStreamSynchronize(s));
        for (size_t i = 0; i < no; ++i) out2[i] = (float)h[i];
      }
      unsigned t = 1; CU(cudaMemcpyAsync(&t, ticket, 4, cudaMemcpyDeviceToHost, s)); CU(cudaStreamSynchronize(s));
      if (t != 0) return fail(B2G_ERR_CUDA, "GLOBAL_POOL: the forward left its ticket word at %u", t);
      break;
    }
    case B2G_EW_UPSAMPLE: {
      const int f = o->KH;
      if (!in0 || !in1 || o->N < 1 || o->H < 1 || o->W < 1 || o->C < 1 || f < 1) return fail(B2G_ERR_ARG, "bad UPSAMPLE arguments");
      const size_t ni = (size_t)o->N * o->H * o->W * o->C, no = ni * f * f;
      if (no > (size_t)lim) return fail(B2G_ERR_ARG, "UPSAMPLE output too large");
      void *x = nullptr, *eo = nullptr, *y = nullptr, *ei = nullptr;
      B2(m.upT(in0, ni, &x, off)); B2(m.upT(in1, no, &eo, off)); B2(m.dev(no, ts, &y, off)); B2(m.dev(ni, ts, &ei, off)); B2(poison(y, ts * no)); B2(poison(ei, ts * ni));
      k_upsample_fwd(prec, x, y, o->N, o->H, o->W, o->C, f, s); ran();
      k_upsample_bwd(prec, eo, ei, o->N, o->H, o->W, o->C, f, s); ran();
      B2(m.downT(out0, y, no)); B2(m.downT(out1, ei, ni));
      break;
    }
    case B2G_EW_PRELU_FWD: case B2G_EW_PRELU_BWD: {      // in0 = [x | alpha], act = the shared-axes mask, the map in N, H, W, C
      const bool bwd = o->op == B2G_EW_PRELU_BWD;
      if (!in0 || (bwd && !in1) || o->N < 1 || o->H < 1 || o->W < 1 || o->C < 1 || o->act < 0 || o->act > 7) return fail(B2G_ERR_ARG, "bad PRELU arguments");
      const PreluGeom g{o->H, o->W, o->C, o->act};
      const size_t n = (size_t)o->N * o->H * o->W * o->C, K = prelu_slopes(g);
      if (n > (size_t)lim) return fail(B2G_ERR_ARG, "PRELU tensors too large");
      void* x = nullptr; float* alpha = nullptr; B2(m.upT(in0, n, &x, off)); B2(m.upF(in0 + n, K, &alpha, off));
      if (!bwd) {
        void* y = nullptr; B2(m.dev(n, ts, &y, off)); B2(poison(y, ts * n));
        k_prelu_fwd(prec, x, y, alpha, o->N, g, s); ran();
        B2(m.downT(out0, y, n));
      } else {        // out0 = dx in eps's buffer (in place; NULL: not written), out1 = dalpha (NULL: no slope gradient)
        void* e = nullptr; float *part = nullptr, *da = nullptr; B2(m.upT(in1, n, &e, off));
        if (out1) {
          const size_t np = k_prelu_part_floats(o->N, g);
          B2(m.upF(nullptr, np, &part, off)); B2(m.upF(nullptr, K, &da, off)); B2(poison(part, 4 * np)); B2(poison(da, 4 * K));
        }
        k_prelu_bwd(prec, x, e, alpha, part, out0 ? 1 : 0, o->N, g, s); ran();
        if (out1) { ReduceList rl{}; prelu_queue_reduce(&rl, part, da, o->N, g); k_reduce_multi(rl, s); ran(); }
        B2(m.downT(out0, e, n)); B2(m.downF(out1, da, K));
      }
      break;
    }
    case B2G_EW_SUMSQ: {
      if (!in0 || o->n < 1 || o->n_seg < 1 || !o->seg_off || !o->seg_len || !o->seg_coef) return fail(B2G_ERR_ARG, "bad SUMSQ arguments");
      for (int i = 0; i < o->n_seg; ++i)
        if (o->seg_off[i] < 0 || o->seg_len[i] < 0 || o->seg_off[i] + o->seg_len[i] > o->n) return fail(B2G_ERR_ARG, "segment %d outside the tensor", i);
      float *p = nullptr, *coef = nullptr; int64_t *so = nullptr, *sl = nullptr; double* res = nullptr;
      B2(m.upF(in0, (size_t)o->n, &p, off)); B2(m.upF(o->seg_coef, (size_t)o->n_seg, &coef, off)); B2(m.dev((size_t)o->n_seg, 8, (void**)&so, off)); B2(m.dev((size_t)o->n_seg, 8, (void**)&sl, off)); B2(m.dev(1, 8, (void**)&res, off));
      CU(cudaMemcpyAsync(so, o->seg_off, 8 * (size_t)o->n_seg, cudaMemcpyHostToDevice, s)); CU(cudaMemcpyAsync(sl, o->seg_len, 8 * (size_t)o->n_seg, cudaMemcpyHostToDevice, s));
      B2(poison(res, 8));
      k_sumsq_segments(p, so, sl, coef, o->n_seg, res, s); ran();
      CU(cudaMemcpyAsync(&o->sumsq, res, 8, cudaMemcpyDeviceToHost, s));
      break;
    }
    case B2G_EW_NCHW_TO_NHWC: case B2G_EW_NHWC_TO_NCHW: case B2G_EW_PERMUTE: {
      const size_t n = (size_t)o->N * o->C * o->H * o->W;
      if (!in0 || o->N < 1 || o->C < 1 || o->H < 1 || o->W < 1 || n > (size_t)lim || (o->op == B2G_EW_PERMUTE && o->groups != 0 && o->groups != 1))
        return fail(B2G_ERR_ARG, "bad layout arguments");
      const int HW = o->H * o->W;
      if (o->op == B2G_EW_NCHW_TO_NHWC) {
        float* x = nullptr; void* y = nullptr; B2(m.upF(in0, n, &x, off)); B2(m.dev(n, ts, &y, off)); B2(poison(y, ts * n));
        k_nchw_f32_to_nhwc(prec, x, y, o->N, o->C, HW, s); ran();
        B2(m.downT(out0, y, n));
      } else if (o->op == B2G_EW_NHWC_TO_NCHW) {
        void* x = nullptr; float* y = nullptr; B2(m.upT(in0, n, &x, off)); B2(m.upF(nullptr, n, &y, off)); B2(poison(y, 4 * n));
        k_nhwc_to_nchw_f32(prec, x, y, o->N, o->C, HW, s); ran();
        B2(m.downF(out0, y, n));
      } else {
        void *x = nullptr, *y = nullptr; B2(m.upT(in0, n, &x, off)); B2(m.dev(n, ts, &y, off)); B2(poison(y, ts * n));
        k_permute(prec, x, y, o->N, o->C, HW, o->groups, s); ran();
        B2(m.downT(out0, y, n));
      }
      break;
    }
    case B2G_EW_CAST_BF16: {      // the bf16 result comes back raw (widened on the host), and through the device widen the gradient payload uses
      const size_t n = (size_t)o->n;
      if (!in0 || o->n < 1 || o->n > lim) return fail(B2G_ERR_ARG, "bad CAST_BF16 arguments");
      float *x = nullptr, *w = nullptr; __nv_bfloat16* y = nullptr;
      B2(m.upF(in0, n, &x, off)); B2(m.dev(n, 2, (void**)&y, off)); B2(m.upF(nullptr, n, &w, off)); B2(poison(y, 2 * n)); B2(poison(w, 4 * n));
      k_cast_f32_to_bf16(x, y, n, s); ran();
      k_nhwc_to_nchw_f32(PREC_BF16, y, w, 1, 1, (int)n, s); ran();
      if (out0) {
        std::vector<uint16_t> h(n); CU(cudaMemcpyAsync(h.data(), y, 2 * n, cudaMemcpyDeviceToHost, s)); CU(cudaStreamSynchronize(s));
        for (size_t i = 0; i < n; ++i) { const uint32_t u = (uint32_t)h[i] << 16; memcpy(out0 + i, &u, 4); }
      }
      B2(m.downF(out1, w, n));
      break;
    }
    default: return fail(B2G_ERR_ARG, "unknown op %d", o->op);
  }
  CU(cudaStreamSynchronize(s)); CHECK_KERNELS();
  strncpy(o->kernel, names.c_str(), sizeof(o->kernel) - 1); o->kernel[sizeof(o->kernel) - 1] = 0;
  return 0;
}
extern "C" int32_t b2g_test_ew(b2g_ctx* c, int32_t precision, b2g_test_ew_opts* o, const float* in0, const float* in1, float* out0, float* out1, float* out2) {
  return test_ew_impl(c, precision, o, nullptr, in0, in1, out0, out1, out2);
}
extern "C" int32_t b2g_test_loss(b2g_ctx* c, int32_t precision, b2g_test_loss_opts* o, const float* zh, const float* yh, const float* wh, const float* mh,
                                  float* dzh, float* lossh) {
  if (!c || !o || !zh || !yh) return fail(B2G_ERR_ARG, "null");
  const int prec = precision == B2G_PREC_BF16 ? PREC_BF16 : PREC_F32; const size_t ts = prec_size(prec);
  const int off = o->offset, k = o->kernel;
  if (off < 0 || off > 64) return fail(B2G_ERR_ARG, "offset %d outside [0, 64]", off);
  if (k < B2G_TEST_LOSS_XENT || k > B2G_TEST_LOSS_CNN_SOFTMAX_XENT || o->rows < 1 || o->cols < 1 || o->groups < 1 ||
      (k == B2G_TEST_LOSS_XENT && o->cols != 1) || (k == B2G_TEST_LOSS_SOFTMAX_XENT && o->groups != 1) ||
      (int64_t)o->rows * o->cols * o->groups > 0x7fffffff) return fail(B2G_ERR_ARG, "bad loss test arguments");
  if (k == B2G_TEST_LOSS_CODES && (o->loss < B2G_LOSS_MSE || o->loss > B2G_LOSS_WASSERSTEIN || o->act < B2G_ACT_IDENTITY || o->act > B2G_ACT_LRELU))
    return fail(B2G_ERR_ARG, "bad loss / activation");
  if (mh && o->mask_width != 1 && o->mask_width != o->cols) return fail(B2G_ERR_SHAPE, "mask width %d: 1 or %d", o->mask_width, o->cols);
  CU(cudaSetDevice(c->device)); cudaStream_t s = c->stream;
  HookMem m(s, prec);
  const size_t per = (size_t)o->rows * o->cols, n = per * o->groups, rows = (size_t)o->rows * o->groups;
  void *z = nullptr, *dz = nullptr; float *y = nullptr, *w = nullptr, *mk = nullptr, *loss = nullptr; double* partial = nullptr; unsigned* ticket = nullptr;
  B2(m.upT(zh, n, &z, off)); B2(m.upF(yh, n, &y, off)); B2(m.dev(n, ts, &dz, off)); B2(m.upF(nullptr, (size_t)o->groups, &loss, off));
  if (wh) B2(m.upF(wh, (size_t)o->cols, &w, off));
  if (mh) B2(m.upF(mh, rows * o->mask_width, &mk, off));
  B2(m.dev((size_t)1024 + (size_t)o->groups, 8, (void**)&partial, off)); B2(m.dev(1, 4, (void**)&ticket, off)); CU(cudaMemsetAsync(ticket, 0, 4, s));
  if (o->poison) { CU(cudaMemsetAsync(dz, 0xFF, ts * n, s)); CU(cudaMemsetAsync(loss, 0xFF, 4 * (size_t)o->groups, s)); }
  const LossWM q{w, mk, mh ? o->mask_width : 0, o->cols};
  g_ew_last_kernel = "";
  switch (k) {
    case B2G_TEST_LOSS_XENT: k_xent_wm(prec, z, y, dz, loss, o->rows, o->groups, o->clip_eps, q, s); break;
    case B2G_TEST_LOSS_SOFTMAX_XENT: k_softmax_xent_wm(prec, z, y, dz, loss, o->rows, o->cols, q, s); break;
    case B2G_TEST_LOSS_CODES: k_loss_wm(prec, o->loss, o->act, o->alpha, z, y, dz, loss, o->rows, o->cols, o->groups, partial, ticket, q, s); break;
    case B2G_TEST_LOSS_CNN_XENT: k_cnn_xent_wm(prec, z, y, dz, loss, per, o->groups, o->clip_eps, partial, ticket, q, s); break;
    default: k_cnn_softmax_xent_wm(prec, z, y, dz, loss, o->rows, o->cols, o->groups, partial, ticket, q, s); break;
  }
  snprintf(o->kernel_name, sizeof(o->kernel_name), "%s", g_ew_last_kernel); g_ew_last_kernel = "";
  B2(m.downT(dzh, dz, n)); B2(m.downF(lossh, loss, (size_t)o->groups));
  unsigned t = 1; CU(cudaMemcpyAsync(&t, ticket, 4, cudaMemcpyDeviceToHost, s)); CU(cudaStreamSynchronize(s));
  if (t != 0) return fail(B2G_ERR_CUDA, "loss test: the kernel left its ticket word at %u", t);
  return 0;
}
extern "C" int32_t b2g_test_pool(b2g_ctx* c, int32_t precision, b2g_test_pool_opts* po, const float* in0, const float* in1, float* out0, float* out1, float* out2) {
  if (!c || !po) return fail(B2G_ERR_ARG, "null");
  if (po->op != B2G_TEST_POOL2D && po->op != B2G_TEST_GLOBAL_POOL) return fail(B2G_ERR_ARG, "unknown pooling op %d", po->op);
  b2g_test_ew_opts o{};
  o.op = po->op == B2G_TEST_POOL2D ? EW_POOL2D : EW_GLOBAL_POOL;
  o.N = po->N; o.H = po->H; o.W = po->W; o.C = po->C; o.KH = po->KH; o.KW = po->KW; o.SH = po->SH; o.SW = po->SW;
  o.offset = po->offset; o.poison = po->poison;
  po->splits = 1;
  B2(test_ew_impl(c, precision, &o, po, in0, in1, out0, out1, out2));
  memcpy(po->kernel, o.kernel, sizeof(po->kernel));
  return 0;
}

// Copies one of the bf16 weight operands the updater keeps beside the fp32 master, widened to fp32: which = 0 the straight copy of W
// (internal [A][taps][B] order), which = 1 the packed [(py,px,c)][(dyr,dxc)][O] operand of the pixel-shuffle transposed conv.
extern "C" int32_t b2g_test_net_shadow(b2g_net* n, int32_t layer, int32_t which, float* out, int64_t count) {
  if (!n || !out) return fail(B2G_ERR_ARG, "null");
  if (layer < 0 || layer >= (int)n->L.size()) return fail(B2G_ERR_ARG, "layer %d out of range", layer);
  if (n->prec != PREC_BF16) return fail(B2G_ERR_UNSUPPORTED, "FP32 nets keep no bf16 weight copies");
  const LayerRT& l = n->L[layer];
  int64_t off = -1, len = 0;
  if (which == 0) { off = l.off_W_bf; len = l.n_W; }
  else if (which == 1) { off = l.off_Wps_bf; len = (int64_t)k_tc_deconv_ps_weight_elems(l.geom); }
  else return fail(B2G_ERR_ARG, "which = %d (0 straight copy, 1 pixel-shuffle operand)", which);
  if (off < 0) return fail(B2G_ERR_UNSUPPORTED, "layer %d has no %s", layer, which ? "pixel-shuffle operand" : "bf16 weight copy");
  if (count != len) return fail(B2G_ERR_SHAPE, "layer %d operand has %lld elements, %lld requested", layer, (long long)len, (long long)count);
  CU(cudaSetDevice(n->ctx->device)); cudaStream_t s = n->ctx->stream;
  if ((size_t)len > n->stage_floats) return fail(B2G_ERR_SHAPE, "operand larger than the staging buffer");
  k_nhwc_to_nchw_f32(PREC_BF16, n->shadow + off, n->stage_f32, 1, 1, (int)len, s);
  CU(cudaMemcpyAsync(out, n->stage_f32, sizeof(float) * len, cudaMemcpyDeviceToHost, s)); CU(cudaStreamSynchronize(s)); CHECK_KERNELS();
  return 0;
}

// The noisy operands of the layer's latest drawing pass (b2g_weight_noise), widened to fp32: which = 0 W' (fp32 or the bf16 straight copy),
// 1 the packed pixel-shuffle W', 2 b'.
extern "C" int32_t b2g_test_net_noisy_operand(b2g_net* n, int32_t layer, int32_t which, float* out, int64_t count) {
  if (!n || !out) return fail(B2G_ERR_ARG, "null");
  if (layer < 0 || layer >= (int)n->L.size()) return fail(B2G_ERR_ARG, "layer %d out of range", layer);
  const LayerRT& l = n->L[layer];
  if (!l.wn_drawn) return fail(B2G_ERR_UNSUPPORTED, "layer %d drew no weight noise", layer);
  const void* src = nullptr; int64_t len = 0; int prec = PREC_F32;
  if (which == 0) { src = l.wn_w; len = l.n_W; prec = n->prec; }
  else if (which == 1) {
    if (l.wn_ps < 0) return fail(B2G_ERR_UNSUPPORTED, "layer %d has no pixel-shuffle operand", layer);
    src = (const __nv_bfloat16*)l.wn_w + l.wn_ps; len = (int64_t)k_tc_deconv_ps_weight_elems(l.geom); prec = PREC_BF16;
  } else if (which == 2) {
    if (!l.wn.apply_to_bias || !l.wn_b) return fail(B2G_ERR_UNSUPPORTED, "layer %d perturbs no bias", layer);
    src = l.wn_b; len = l.d.n_out;
  } else return fail(B2G_ERR_ARG, "which = %d (0 W', 1 pixel-shuffle W', 2 b')", which);
  if (count != len) return fail(B2G_ERR_SHAPE, "layer %d operand has %lld elements, %lld requested", layer, (long long)len, (long long)count);
  CU(cudaSetDevice(n->ctx->device)); cudaStream_t s = n->ctx->stream;
  if (prec == PREC_BF16) {
    if ((size_t)len > n->stage_floats) return fail(B2G_ERR_SHAPE, "operand larger than the staging buffer");
    k_nhwc_to_nchw_f32(PREC_BF16, src, n->stage_f32, 1, 1, (int)len, s); src = n->stage_f32;
  }
  CU(cudaMemcpyAsync(out, src, sizeof(float) * len, cudaMemcpyDeviceToHost, s)); CU(cudaStreamSynchronize(s)); CHECK_KERNELS();
  return 0;
}

// Times the HBM-bound kernels of the step in isolation (bench.py's `hbm` roofline entries): every launch is bracketed by its own CUDA events
// on the library stream and preceded by an L2 flush (a 256 MiB memset), so the operands really come from HBM as they do inside a step.
// ms[0] = one updater pass over `net` (Adam: 28 B/param + 2 B bf16 operand copy; the net's parameters are perturbed -- bench only),
// ms[1] = BatchNorm apply (read + write a [groups*rows x C] bf16 tensor), ms[2] = BatchNorm backward apply (two reads + one write).
extern "C" int32_t b2g_test_hbm_kernels(b2g_net* n, int32_t rows, int32_t channels, int32_t iters, float* ms3) {
  if (!n || !ms3 || rows < 8 || iters < 1) return fail(B2G_ERR_ARG, "bad arguments"); b2g_ctx* c = n->ctx; CU(cudaSetDevice(c->device)); cudaStream_t s = c->stream;
  if (!k_bn_vec_ok(PREC_BF16, channels)) return fail(B2G_ERR_UNSUPPORTED, "channels %d not supported by the vector BatchNorm kernels", channels);
  const size_t ne = (size_t)rows * channels; __nv_bfloat16 *x = nullptr, *e = nullptr, *y = nullptr; float *coef = nullptr, *gb = nullptr; unsigned long long* acc = nullptr;
  HookMem m(s, PREC_BF16);
  B2(m.dev(ne, 2, (void**)&x)); B2(m.dev(ne, 2, (void**)&e)); B2(m.dev(ne, 2, (void**)&y)); B2(m.upF(nullptr, 4 * (size_t)channels, &coef)); B2(m.upF(nullptr, 4 * (size_t)channels, &gb));
  B2(m.dev(k_bn_acc_elems(channels, 1), 8, (void**)&acc));
  CU(cudaMemsetAsync(x, 0x3c, 2 * ne, s)); CU(cudaMemsetAsync(e, 0x3c, 2 * ne, s)); CU(cudaMemsetAsync(acc, 0, 8 * k_bn_acc_elems(channels, 1), s)); k_fill_f32(coef, 1.0f, 4 * channels, s); k_fill_f32(gb, 1.0f, 4 * channels, s);
  cudaEvent_t e0, e1; B2(m.event(&e0)); B2(m.event(&e1));
  ms3[0] = ms3[1] = ms3[2] = 0.f;
  for (int which = 0; which < 3; ++which) for (int it = -1; it < iters; ++it) {
    B2(b2g_flush_l2(c));
    CU(cudaEventRecord(e0, s));
    if (which == 0) k_updater(n->params, n->grads, n->st0, n->st1, n->st2, n->segs_dev, n->chunk_seg_dev, n->chunk_off_dev, n->nchunks, 1.0f, 1.0f, n->step_dev, n->upd_ticket,
                              n->shadow, nullptr, nullptr, nullptr, n->upd_ext, s);
    else if (which == 1) k_bn_apply_acc(x, y, rows, channels, 1, acc, gb, gb + channels, ACT_LRELU, 0.2f, 1e-5f, coef, gb + 2 * channels, gb + 3 * channels, nullptr, nullptr, 0.9f, s);
    else k_bn_bwd_apply_acc(x, e, y, rows, channels, 1, coef, ACT_LRELU, 0.2f, 1, acc, gb, gb + channels, 0, s);
    CU(cudaEventRecord(e1, s)); CU(cudaEventSynchronize(e1));
    float ms = 0.f; CU(cudaEventElapsedTime(&ms, e0, e1)); if (it >= 0) ms3[which] += ms / iters;
  }
  CHECK_KERNELS();
  return 0;
}
