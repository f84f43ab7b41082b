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
  int64_t off_W_bf = -1;                                       // bf16 operand copy [A][taps][B] (written by the updater itself); serves fprop, dgrad (MN-major tiles) and wgrad
  int64_t off_Wps_bf = -1;                                     // packed [16][9][O] weights of the tensor-core pixel-shuffle transposed conv (<= 4 image channels)
  int wA = 0, wTaps = 0, wB = 0;                               // internal weight layout [A][taps][B]
  void* out = nullptr; bool out_alias = false;
  void* probs = nullptr;                                       // OUTPUT / LOSS: sigmoid(logits)
  uint8_t* argmax = nullptr;
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
  bool drop_active() const { return d.type == B2G_LAYER_DROPOUT && !d.frozen && d.act_alpha < 1.f; }   // FrozenLayer: test mode, identity
  bool has_gemm() const { return d.type == B2G_LAYER_CONV2D || d.type == B2G_LAYER_DECONV2D || d.type == B2G_LAYER_DENSE || d.type == B2G_LAYER_OUTPUT; }
};

struct b2g_net {
  b2g_ctx* ctx = nullptr;
  b2g_net_config cfg{};
  std::vector<LayerRT> L;
  int prec = PREC_F32;
  int64_t n_params = 0;
  float *params = nullptr, *grads = nullptr, *st0 = nullptr, *st1 = nullptr;
  __nv_bfloat16* shadow = nullptr; int64_t n_shadow = 0;
  std::vector<UpdSeg> segs; UpdSeg* segs_dev = nullptr; int32_t* chunk_seg_dev = nullptr; int64_t* chunk_off_dev = nullptr; int nchunks = 0;
  int64_t *l2_off_dev = nullptr, *l2_len_dev = nullptr; float* l2_coef_dev = nullptr; int n_l2 = 0;
  int* step_dev = nullptr;
  int max_rows = 0;                    // cfg.max_batch
  size_t in_elems = 0;
  void* input = nullptr;               // T NHWC [max_rows][in_elems]
  float* stage_f32 = nullptr; size_t stage_floats = 0;   // host<->device fp32 staging (inputs, outputs, params)
  float* labels_dev = nullptr;         // [max_rows]
  void *epsA = nullptr, *epsB = nullptr, *epsC = nullptr; size_t eps_elems = 0;
  float* scratch2 = nullptr;           // split-K / colsum partials of the side stream
  std::vector<cudaEvent_t> ev_fork, ev_done; cudaEvent_t ev_join = nullptr;
  unsigned long long* bn_acc = nullptr; size_t bn_acc_bytes = 0;  // every BatchNorm layer's accumulators, zeroed by one memset per train-mode forward
  unsigned* upd_ticket = nullptr;                                  // block-completion counter of the updater kernel (the last block bumps step_dev)
  unsigned long long* drop_pass = nullptr;                         // dropout pass counter P (device): read by every dropout kernel of a train-mode pass
  unsigned* drop_ticket = nullptr;                                 // block-completion counter of the pass's last dropout kernel (its last block bumps P)
  // L2 gradient normalization (b2g_net_set_gradient_normalization): mode, threshold and a generation bumped on every change (a captured GAN
  // step holds the mode's launches, so it is re-captured when the generation differs); norm groups per layer and per segment; the norm
  // kernel's per-chunk partial sums, block-completion counter and per-segment multipliers
  int gn_mode = B2G_GN_NONE; float gn_threshold = 1.0f; uint64_t gn_gen = 0;
  GnGroup *gn_layer_groups = nullptr, *gn_param_groups = nullptr; int gn_n_layer_groups = 0, gn_n_param_groups = 0;
  double* gn_partial = nullptr; unsigned* gn_ticket = nullptr; float* gn_mult = nullptr;
  ReduceList pending{};                                            // split-K partial sums queued by this backward pass
  uint64_t simt_gemm_calls = 0;                                    // BF16 nets: GEMM-shaped ops that ran on the SIMT kernels (skinny / unsupported shapes) -- reported, never silent
  float* scratch = nullptr; size_t scratch_floats = 0;
  float* loss_dev = nullptr;           // [8]
  double* l2_dev = nullptr;
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
        if (d.type == B2G_LAYER_OUTPUT) { d.act = B2G_ACT_IDENTITY; if (d.loss == B2G_LOSS_XENT && d.n_out != 1) return fail(B2G_ERR_UNSUPPORTED, "layer %s: XENT output supports nOut=1 (use MCXENT for nOut>1)", d.name); }
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
      case B2G_LAYER_LOSS: l.oh = h; l.ow = w; l.oc = ch; if ((size_t)h * w * ch != 1) return fail(B2G_ERR_UNSUPPORTED, "layer %s: XENT loss needs one logit per example", d.name); break;
      case B2G_LAYER_FF_TO_CNN:
        if ((size_t)d.pre_h * d.pre_w * d.pre_c != l.in_elems) return fail(B2G_ERR_SHAPE, "layer %s: FeedForwardToCnn(%d,%d,%d) != %zu features", d.name, d.pre_h, d.pre_w, d.pre_c, l.in_elems);
        l.oh = d.pre_h; l.ow = d.pre_w; l.oc = d.pre_c; break;
      case B2G_LAYER_CNN_TO_FF: l.oh = l.ow = 1; l.oc = h * w * ch; break;
      case B2G_LAYER_DROPOUT:        // DropoutLayer.Builder(p): p = retain probability, carried in act_alpha; no parameters
        if (!(d.act_alpha > 0.f && d.act_alpha <= 1.f)) return fail(B2G_ERR_ARG, "layer %s: dropout retain probability %g outside (0, 1]", d.name, (double)d.act_alpha);
        l.oh = h; l.ow = w; l.oc = ch;
        if ((uint64_t)c.max_batch * h * w * ch > (1ull << 34))     // checked before anything is allocated
          return fail(B2G_ERR_UNSUPPORTED, "layer %s: a dropout pass of %llu elements exceeds the 2^34 the mask counter addresses", d.name, (unsigned long long)c.max_batch * h * w * ch);
        break;
      default: return fail(B2G_ERR_ARG, "layer %d: unknown type %d", i, d.type);
    }
    l.out_elems = (size_t)l.oh * l.ow * l.oc;
    if (l.has_gemm() && n->prec == PREC_BF16) { l.off_W_bf = off_bf; off_bf += l.n_W; off_bf = (off_bf + 63) / 64 * 64;
      if (n->ctx->tc_ok && tc_deconv_ps_shape(l.geom) && !getenv("B2G_NO_TC_EDGE")) { l.off_Wps_bf = off_bf; off_bf += (int64_t)k_tc_deconv_ps_weight_elems(l.geom); off_bf = (off_bf + 63) / 64 * 64; } }
    h = l.oh; w = l.ow; ch = l.oc;
    n->L.push_back(l);
  }
  // fuse BatchNormalization + ActivationLayer (north_star's BN+ReLU / BN+LeakyReLU)
  for (size_t i = 0; i + 1 < n->L.size(); ++i)
    if (n->L[i].d.type == B2G_LAYER_BATCHNORM && n->L[i + 1].d.type == B2G_LAYER_ACTIVATION) {
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
  B2(dalloc(n, &n->step_dev, sizeof(int))); B2(dalloc(n, &n->loss_dev, sizeof(float) * 8)); B2(dalloc(n, &n->l2_dev, sizeof(double)));
  B2(dalloc(n, &n->labels_dev, sizeof(float) * R * std::max<size_t>(1, n->L.back().out_elems)));
  B2(dalloc(n, (char**)&n->input, ts * R * n->in_elems));
  size_t max_act = n->in_elems, scratch = 1 << 16, max_w = 0, bn_acc_words = 0;
  for (auto& l : n->L) {
    max_act = std::max(max_act, std::max(l.in_elems, l.out_elems));
    bool alias = l.act_fused_into_prev || l.d.type == B2G_LAYER_LOSS ||
                 (l.d.type == B2G_LAYER_FF_TO_CNN && (l.oc == 1 || l.oh * l.ow == 1)) ||
                 (l.d.type == B2G_LAYER_CNN_TO_FF && (l.ic == 1 || l.ih * l.iw == 1));
    l.out_alias = alias;
    if (!alias) B2(dalloc(n, (char**)&l.out, ts * R * l.out_elems));
    if (l.d.type == B2G_LAYER_DROPOUT) { l.drop_buf = l.out; B2(dalloc(n, &l.drop_mask, sizeof(uint32_t) * (((size_t)R * l.out_elems + 31) / 32))); }
    if (l.d.type == B2G_LAYER_OUTPUT || l.d.type == B2G_LAYER_LOSS) B2(dalloc(n, (char**)&l.probs, ts * R * l.out_elems));
    if (l.d.type == B2G_LAYER_MAXPOOL) B2(dalloc(n, &l.argmax, (size_t)R * l.out_elems));
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
        l.wg_part_floats = std::max(k_tc_wgrad_scratch_floats(g), k_tc_edge_wgrad_scratch_floats(g));
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

static int updater_kind(int u) { return u == B2G_UPD_SGD ? 0 : u == B2G_UPD_RMSPROP ? 1 : u == B2G_UPD_ADAM ? 2 : 3; }

static int32_t net_init_params_and_updater(b2g_net* n) {
  cudaStream_t s = n->ctx->stream;
  std::vector<float> hp(n->n_params, 0.f), h0(n->n_params, 0.f);
  uint64_t seed = n->cfg.seed ? n->cfg.seed : 666;
  std::vector<int64_t> l2o, l2l; std::vector<float> l2c;
  std::vector<int> seg_layer;      // layer index of every segment (the norm groups of the PerLayer modes)
  for (auto& l : n->L) {
    const b2g_layer_desc& d = l.d;
    auto add_seg = [&](int64_t off, int64_t len, bool weight, bool noop) {
      if (d.frozen) return;      // FrozenLayer: no update, no l2 decay, no l2 score (calcL2() == 0)
      UpdSeg sg{}; sg.off = off; sg.len = len; sg.kind = noop ? 3 : updater_kind(d.updater);
      sg.lr = d.lr; sg.b1 = d.beta1; sg.b2 = d.beta2; sg.eps = d.eps; sg.l2 = weight ? d.l2 : 0.f; sg.clip = n->cfg.grad_clip; sg.div_mb = noop ? 0 : 1;
      sg.off_bf = (weight && l.off_W_bf >= 0) ? l.off_W_bf : -1; sg.off_ps = (weight && l.off_Wps_bf >= 0) ? l.off_Wps_bf : -1; sg.ps_O = l.geom.O; sg.ps_C = l.geom.C; n->segs.push_back(sg); seg_layer.push_back((int)(&l - n->L.data()));
      if (!noop && sg.kind == 1) for (int64_t i = 0; i < len; ++i) h0[off + i] = d.eps;     // RmsPropUpdater cache initialised to epsilon
      if (weight && d.l2 != 0.f) { l2o.push_back(off); l2l.push_back(len); l2c.push_back(0.5f * d.l2); }
    };
    if (l.has_gemm()) {
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
    }
  }
  CU(cudaMemcpyAsync(n->params, hp.data(), sizeof(float) * n->n_params, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(n->st0, h0.data(), sizeof(float) * n->n_params, cudaMemcpyHostToDevice, s));
  CU(cudaMemsetAsync(n->st1, 0, sizeof(float) * n->n_params, s)); CU(cudaMemsetAsync(n->grads, 0, sizeof(float) * n->n_params, s));
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
  n->n_l2 = (int)l2o.size();
  if (n->n_l2) {
    B2(dalloc(n, &n->l2_off_dev, sizeof(int64_t) * n->n_l2)); B2(dalloc(n, &n->l2_len_dev, sizeof(int64_t) * n->n_l2)); B2(dalloc(n, &n->l2_coef_dev, sizeof(float) * n->n_l2));
    CU(cudaMemcpyAsync(n->l2_off_dev, l2o.data(), sizeof(int64_t) * n->n_l2, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(n->l2_len_dev, l2l.data(), sizeof(int64_t) * n->n_l2, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(n->l2_coef_dev, l2c.data(), sizeof(float) * n->n_l2, cudaMemcpyHostToDevice, s));
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
struct FwdOpts { int rows; int groups; bool train; bool update_running; void* out_override; };

static const void* w_ptr(const b2g_net* n, const LayerRT& l, int* wprec) {
  if (n->prec == PREC_BF16) { *wprec = PREC_BF16; return n->shadow + l.off_W_bf; }
  *wprec = PREC_F32; return n->params + l.off_W;
}

// tensor-core versions of the <= 4-image-channel layers (B2G_NO_TC_EDGE=1 keeps the SIMT kernels of kernels_edge.cu)
static inline bool tc_on(const b2g_net* n) { return n->prec == PREC_BF16 && n->ctx->tc_ok; }
static bool tc_edge_on(const b2g_net* n) { static int on = -1; if (on < 0) on = getenv("B2G_NO_TC_EDGE") ? 0 : 1; return on && tc_on(n); }
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
  if (tc_edge_on(n) && tc_edge_conv_supported(g) && k_tc_edge_conv(g, (const __nv_bfloat16*)x, (const __nv_bfloat16*)w, bias, (__nv_bfloat16*)out, act, alpha, s) == 0) return 0;
  if (edge_conv_small_cin_supported(g)) { note_simt(n); k_edge_conv_small_cin(n->prec, wp, g, x, w, bias, out, act, alpha, s); return 0; }
  if (dense_small_o_supported(g)) { note_simt(n); k_dense_small_o_fwd(n->prec, wp, g, x, w, bias, out, act, alpha, s); return 0; }
  if (tc_on(n) && tc_fprop_supported(g)) {
    if (fuse && k_tc_fprop(g, (const __nv_bfloat16*)x, (const __nv_bfloat16*)w, bias, (__nv_bfloat16*)out, act, alpha, s, fuse) == 0) { if (fused) *fused = true; return 0; }
    if (k_tc_fprop(g, (const __nv_bfloat16*)x, (const __nv_bfloat16*)w, bias, (__nv_bfloat16*)out, act, alpha, s) == 0) return 0;
    return fail(B2G_ERR_CUDA, "tensor-core fprop launch failed");
  }
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
  if (tc_edge_on(n) && l.off_Wps_bf >= 0 && tc_deconv_ps_supported(g)) {
    const TcEpi* f = (fuse && fuse->mode == EPI_ACTBWD) ? fuse : nullptr;
    if (k_tc_deconv_ps(g, (const __nv_bfloat16*)dy, n->shadow + l.off_Wps_bf, bias, (__nv_bfloat16*)dx, act, alpha, s, f) == 0) { if (fused) *fused = f != nullptr; return 0; }
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
  note_simt(n); k_simt_dgrad(n->prec, wp, g, dy, w, bias, dx, act, alpha, s); return 0;
}
static int32_t gemm_wgrad(b2g_net* n, LayerRT& l, const ConvGeom& g, const void* x, const void* dy, float* dw, cudaStream_t s, float* scratch, float* db = nullptr, bool* bias_done = nullptr) {
  if (tc_edge_on(n) && tc_edge_wgrad_supported(g) && l.wg_part) { const int r = k_tc_edge_wgrad(g, (const __nv_bfloat16*)x, (const __nv_bfloat16*)dy, dw, db, l.wg_part, l.wg_part_floats, 0, s, &n->pending); if (r >= 0) { if (bias_done) *bias_done = r == 1; return 0; } }
  if (edge_wgrad_small_cin_supported(g)) { note_simt(n); k_edge_wgrad_small_cin(n->prec, g, x, dy, dw, scratch, 0, s); return 0; }
  if (dense_small_o_supported(g)) { note_simt(n); k_dense_small_o_wgrad(n->prec, g, x, dy, dw, scratch, 0, s); return 0; }
  if (dense_small_k_supported(g) && !(tc_on(n) && tc_wgrad_supported(g))) { note_simt(n); k_dense_small_k_wgrad(n->prec, g, x, dy, dw, s); return 0; }
  if (tc_on(n) && tc_wgrad_supported(g) && l.wg_part) {
    if (k_tc_wgrad(g, (const __nv_bfloat16*)x, (const __nv_bfloat16*)dy, dw, l.wg_part, l.wg_part_floats, 0, s, &n->pending) == 0) return 0;
    return fail(B2G_ERR_CUDA, "tensor-core wgrad launch failed");
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

// Runs layers [0, L) on `in` (T NHWC, rows examples). Returns pointer to the final activations.
static int32_t net_forward(b2g_net* n, const void* in, const FwdOpts& o, const void** result) {
  cudaStream_t s = fstream(n);
  if (o.rows > n->max_rows || o.rows < 1) return fail(B2G_ERR_SHAPE, "batch %d outside [1, max_batch=%d]", o.rows, n->max_rows);
  if (o.groups < 1 || o.rows % o.groups) return fail(B2G_ERR_SHAPE, "batch %d not divisible into %d groups", o.rows, o.groups);
  const int R = o.rows; const void* cur = in;
  n->last_rows = R;
  // every BatchNorm accumulator of the pass (forward statistics and the backward reductions that follow) starts from zero: one memset node
  if (o.train && n->bn_acc) CU(cudaMemsetAsync(n->bn_acc, 0, n->bn_acc_bytes, s));
  static int fold_bn = -1; if (fold_bn < 0) { const char* e = getenv("B2G_FOLD_BN"); fold_bn = (e && e[0] == '0') ? 0 : 1; }
  static int fuse_bn = -1; if (fuse_bn < 0) { const char* e = getenv("B2G_FUSE_BN"); fuse_bn = (e && e[0] == '0') ? 0 : 1; }
  // every masked DropoutLayer of a train-mode pass draws with the same pass counter P; the last one's kernel advances P on the device
  int last_drop = -1;
  if (o.train) for (size_t i = 0; i < n->L.size(); ++i) if (n->L[i].drop_active()) last_drop = (int)i;
  for (size_t i = 0; i < n->L.size(); ++i) {
    LayerRT& l = n->L[i]; const b2g_layer_desc& d = l.d;
    void* out = l.out;
    if (i + 1 == n->L.size() && o.out_override && !l.out_alias) out = o.out_override;
    const float* bias = l.off_b >= 0 ? n->params + l.off_b : nullptr;
    const bool gemm_then_bn = (d.type == B2G_LAYER_CONV2D || d.type == B2G_LAYER_DECONV2D || d.type == B2G_LAYER_DENSE) && i + 1 < n->L.size() && n->L[i + 1].d.type == B2G_LAYER_BATCHNORM;
    // a 1x1-input deconv is computed as the 1x1 problem with taps*C output channels: its columns are not the BatchNorm's channels
    const bool remapped = d.type == B2G_LAYER_DECONV2D && l.geom.KH == 1 && l.geom.C != l.oc;
    // inference-mode (or frozen) BatchNorm right after a linear conv / deconv / dense: fold it, and its activation, into that GEMM's epilogue
    if (fold_bn && gemm_then_bn && d.act == B2G_ACT_IDENTITY && (!o.train || n->L[i + 1].d.frozen) && !(i + 2 == n->L.size() && o.out_override) && !remapped) {
      LayerRT& bn = n->L[i + 1];
      ConvGeom g = l.geom; g.N = R;
      k_bn_fold(n->params + bn.off_mean, n->params + bn.off_var, n->params + bn.off_gamma, n->params + bn.off_beta, bias, bn.oc, bn.d.bn_eps, bn.bn_fold, bn.bn_fold + bn.oc, s);
      if (d.type == B2G_LAYER_DECONV2D) B2(gemm_dgrad(n, l, g, cur, bn.bn_fold + bn.oc, bn.out, bn.fused_act, bn.fused_alpha, bn.bn_fold));
      else B2(gemm_fprop(n, l, g, cur, bn.bn_fold + bn.oc, bn.out, bn.fused_act, bn.fused_alpha, bn.bn_fold));
      cur = bn.out; ++i; continue;
    }
    // train-mode BatchNorm right after a GEMM: its batch statistics come out of the GEMM's epilogue (kernels_tc.cu EPI_STATS)
    TcEpi st{}; const TcEpi* fuse = nullptr; bool fused = false;
    if (fuse_bn && gemm_then_bn && o.train && !n->L[i + 1].d.frozen && n->L[i + 1].bn_coef && !remapped && tc_on(n)) {
      st.mode = EPI_STATS; st.acc = n->L[i + 1].acc_fwd; st.imgs_per_group = R / o.groups; fuse = &st;
    }
    switch (d.type) {
      case B2G_LAYER_CONV2D: case B2G_LAYER_DENSE: case B2G_LAYER_OUTPUT: { ConvGeom g = l.geom; g.N = R; B2(gemm_fprop(n, l, g, cur, bias, out, d.act, d.act_alpha, nullptr, fuse, &fused)); } break;
      case B2G_LAYER_DECONV2D: { ConvGeom g = l.geom; g.N = R; B2(gemm_dgrad(n, l, g, cur, bias, out, d.act, d.act_alpha, nullptr, fuse, &fused)); } break;
      case B2G_LAYER_BATCHNORM: {
        int rows_pg = (R / o.groups) * l.oh * l.ow;
        const bool bn_train = o.train && !d.frozen;      // FrozenLayer always activates in test mode
        l.fwd_fused = false;
        if (bn_train && l.bn_coef && fuse_bn) {
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
      case B2G_LAYER_ACTIVATION: if (l.act_fused_into_prev) out = (void*)cur; else k_act_fwd(n->prec, cur, out, (size_t)R * l.out_elems, d.act, d.act_alpha, s); break;
      case B2G_LAYER_MAXPOOL: k_maxpool_fwd(n->prec, cur, out, l.argmax, R, l.ih, l.iw, l.ic, l.oh, l.ow, d.k_h, d.k_w, d.s_h, d.s_w, s); break;
      case B2G_LAYER_UPSAMPLE2D: k_upsample_fwd(n->prec, cur, out, R, l.ih, l.iw, l.ic, d.k_h, s); break;
      case B2G_LAYER_LOSS: out = (void*)cur; break;
      case B2G_LAYER_FF_TO_CNN: if (l.out_alias) out = (void*)cur; else k_permute(n->prec, cur, out, R, l.oc, l.oh * l.ow, 1, s); break;
      case B2G_LAYER_CNN_TO_FF: if (l.out_alias) out = (void*)cur; else k_permute(n->prec, cur, out, R, l.ic, l.ih * l.iw, 0, s); break;
      case B2G_LAYER_DROPOUT:
        l.drop_live = o.train && l.drop_active();
        if (l.drop_live) {
          k_dropout_fwd(n->prec, cur, l.drop_buf, l.drop_mask, (size_t)R * l.out_elems, dropout_args(n, (int)i), n->drop_pass, n->drop_ticket, (int)i == last_drop, s);
          out = l.drop_buf;
        } else out = (void*)cur;       // inference, FrozenLayer or p = 1: the identity, no launch
        l.out = out;
        break;
    }
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
  static int fork_on = -1; if (fork_on < 0) { const char* e = getenv("B2G_WGRAD_FORK"); fork_on = (e && e[0] == '0') ? 0 : 1; }
  cudaStream_t s = n->ctx->stream, s2 = fork_on ? n->ctx->side : n->ctx->stream; const int R = rows;
  void* cur = eps;
  if (input_act_done) *input_act_done = false;
  static int fuse_bn = -1; if (fuse_bn < 0) { const char* e = getenv("B2G_FUSE_BN"); fuse_bn = (e && e[0] == '0') ? 0 : 1; }
  static int fuse_act = -1; if (fuse_act < 0) { const char* e = getenv("B2G_FUSE_ACTBWD"); fuse_act = (e && e[0] == '0') ? 0 : 1; }
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
    if (k < 0) { if (input_act && fuse_act) { *e = *input_act; *target = -2; return true; } return false; }
    LayerRT& b = n->L[k];
    if (fuse_bn && b.d.type == B2G_LAYER_BATCHNORM && b.fwd_fused && !b.d.frozen && b.fwd_groups == groups) {
      e->mode = EPI_BNBWD; e->acc = b.acc_bwd; e->imgs_per_group = R / groups; e->aux = (const __nv_bfloat16*)b.out; e->aux2 = (const __nv_bfloat16*)(k == 0 ? net_in : n->L[k - 1].out);
      e->act = b.fused_act; e->alpha = b.fused_alpha; *target = k; return true;
    }
    if (fuse_act && k == i - 1 && b.has_gemm() && b.d.act != B2G_ACT_IDENTITY && b.d.type != B2G_LAYER_OUTPUT) {
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
    if (!need_in) for (int j = 0; j < i; ++j) if (!n->L[j].d.frozen && (n->L[j].has_gemm() || n->L[j].d.type == B2G_LAYER_BATCHNORM)) need_in = true;
    const bool want_wgrad_l = want_wgrad && !d.frozen;
    switch (d.type) {
      case B2G_LAYER_LOSS: break;
      case B2G_LAYER_CONV2D: case B2G_LAYER_DENSE: case B2G_LAYER_OUTPUT: {
        ConvGeom g = l.geom; g.N = R;
        if (d.act != B2G_ACT_IDENTITY && !act_done[i]) k_act_bwd_from_output(n->prec, l.out, cur, cur, (size_t)R * l.out_elems, d.act, d.act_alpha, s);
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
        int rows_pg = (R / groups) * l.oh * l.ow; void* nx = need_in ? other(cur) : nullptr;
        if (l.fwd_fused && l.fwd_groups == groups) {
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
      case B2G_LAYER_ACTIVATION: if (!l.act_fused_into_prev) k_act_bwd_from_output(n->prec, l.out, cur, cur, (size_t)R * l.out_elems, d.act, d.act_alpha, s); break;
      case B2G_LAYER_MAXPOOL: if (need_in) { void* nx = other(cur); k_maxpool_bwd(n->prec, cur, l.argmax, nx, R, l.ih, l.iw, l.ic, l.oh, l.ow, d.k_h, d.k_w, d.s_h, d.s_w, s); cur = nx; } break;
      case B2G_LAYER_UPSAMPLE2D: if (need_in) { void* nx = other(cur); k_upsample_bwd(n->prec, cur, nx, R, l.ih, l.iw, l.ic, d.k_h, s); cur = nx; } break;
      case B2G_LAYER_FF_TO_CNN: if (!l.out_alias && need_in) { void* nx = other(cur); k_permute(n->prec, cur, nx, R, l.oc, l.oh * l.ow, 0, s); cur = nx; } break;
      case B2G_LAYER_CNN_TO_FF: if (!l.out_alias && need_in) { void* nx = other(cur); k_permute(n->prec, cur, nx, R, l.ic, l.ih * l.iw, 1, s); cur = nx; } break;
      case B2G_LAYER_DROPOUT: if (need_in && l.drop_live) k_dropout_bwd(n->prec, cur, cur, l.drop_mask, (size_t)R * l.out_elems, 1.0f / d.act_alpha, s); break;   // the forward's mask
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
  // one pass: /mb -> [x multiplier] -> clip -> updater -> +l2*W -> theta -= g, the bf16 operand copies (straight and packed) and the iteration counter
  k_updater(n->params, n->grads, n->st0, n->st1, n->segs_dev, n->chunk_seg_dev, n->chunk_off_dev, n->nchunks, inv_mb, inv_world, n->step_dev, n->upd_ticket, n->shadow,
            gn ? n->gn_mult : nullptr, s);
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
extern "C" int32_t b2g_net_get_updater_state(b2g_net* n, float* host, int64_t cnt) {
  if (!n || !host) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device));
  if (cnt != 2 * n->n_params) return fail(B2G_ERR_SHAPE, "updater state has %lld elements", (long long)(2 * n->n_params));
  B2(read_flat(n, n->st0, host, n->n_params)); return read_flat(n, n->st1, host + n->n_params, n->n_params);
}
extern "C" int32_t b2g_net_set_updater_state(b2g_net* n, const float* host, int64_t cnt) {
  if (!n || !host) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(n->ctx->device));
  if (cnt != 2 * n->n_params) return fail(B2G_ERR_SHAPE, "updater state has %lld elements", (long long)(2 * n->n_params));
  B2(write_flat(n, n->st0, host, n->n_params)); return write_flat(n, n->st1, host + n->n_params, n->n_params);
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
  if (l.d.type == B2G_LAYER_OUTPUT && l.d.loss == B2G_LOSS_MCXENT) { k_softmax_xent(n->prec, res, nullptr, nullptr, l.probs, nullptr, batch, l.oc, n->ctx->stream); res = l.probs; }
  else if (l.d.type == B2G_LAYER_OUTPUT || l.d.type == B2G_LAYER_LOSS) { k_sigmoid_out(n->prec, res, l.probs, (size_t)batch * l.out_elems, n->ctx->stream); res = l.probs; }
  return download_act(n, res, batch, l.oc, l.oh * l.ow, out);
}
extern "C" int32_t b2g_net_get_activation(b2g_net* n, int32_t layer, int32_t batch, float* host) {
  if (!n || !host || layer < 0 || layer >= (int)n->L.size()) return fail(B2G_ERR_ARG, "bad layer index"); CU(cudaSetDevice(n->ctx->device));
  LayerRT& l = n->L[layer]; if (!l.out) return fail(B2G_ERR_ARG, "layer %d has not run", layer);
  return download_act(n, l.out, batch, l.oc, l.oh * l.ow, host);
}

static void net_loss(b2g_net* n, const void* logits, const float* labels, void* dz, float* loss_sums, int rows_per_group, int groups) {
  const LayerRT& l = n->L.back();
  if (l.d.type == B2G_LAYER_OUTPUT && l.d.loss == B2G_LOSS_MCXENT) k_softmax_xent(n->prec, logits, labels, dz, nullptr, loss_sums, rows_per_group * groups, l.oc, n->ctx->stream);
  else k_xent(n->prec, logits, labels, dz, loss_sums, rows_per_group, groups, n->cfg.xent_clip_eps, n->ctx->stream);
}
static int32_t train_pass(b2g_net* n, const float* x, const float* y, int batch, bool do_update, float* score) {
  cudaStream_t s = n->ctx->stream;
  if (batch < 1 || batch > n->max_rows) return fail(B2G_ERR_SHAPE, "batch %d outside [1,%d]", batch, n->max_rows);
  int lt = n->L.back().d.type;
  if (lt != B2G_LAYER_OUTPUT && lt != B2G_LAYER_LOSS) return fail(B2G_ERR_UNSUPPORTED, "fit needs a net ending in OutputLayer/LossLayer (XENT)");
  B2(upload_input(n, x, batch, n->input));
  CU(cudaMemcpyAsync(n->labels_dev, y, sizeof(float) * batch * n->L.back().out_elems, cudaMemcpyHostToDevice, s));
  CU(cudaMemsetAsync(n->grads, 0, sizeof(float) * n->n_params, s));
  const void* logits = nullptr; FwdOpts o{batch, 1, true, true, nullptr};
  B2(net_forward(n, n->input, o, &logits));
  net_loss(n, logits, n->labels_dev, n->epsA, n->loss_dev, batch, 1);
  B2(net_backward(n, n->input, n->epsA, batch, 1, true, false, /*allreduce_follows=*/do_update && !score));
  if (score) {
    double l2 = 0.0; float ls = 0.f;
    if (n->n_l2) { k_sumsq_segments(n->params, n->l2_off_dev, n->l2_len_dev, n->l2_coef_dev, n->n_l2, n->l2_dev, s); CU(cudaMemcpyAsync(&l2, n->l2_dev, sizeof(double), cudaMemcpyDeviceToHost, s)); }
    CU(cudaMemcpyAsync(&ls, n->loss_dev, sizeof(float), cudaMemcpyDeviceToHost, s)); CU(cudaStreamSynchronize(s));
    *score = ls / batch + (float)l2;
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
  float *y_d = nullptr, *y_g = nullptr;   // [2N] = y_real | y_fake ; [N]
  float* loss_dev = nullptr;              // [4]: d_real_sum, d_fake_sum, g_sum
  float* stage = nullptr; size_t stage_floats = 0;
  cudaGraph_t graph = nullptr, graph1 = nullptr; cudaGraphExec_t exec = nullptr, exec1 = nullptr; int graph_batch = 0; uint64_t graph_launches = 0, graph_simt_g = 0, graph_simt_d = 0;
  uint64_t graph_gn_g = 0, graph_gn_d = 0;   // the nets' gradient-normalization generations the captured graph was made with
  cudaEvent_t ev0 = nullptr, ev1 = nullptr; float last_ms = 0.f; int last_batch = 1; bool nccl_warm = false;
  cudaStream_t copy_stream = nullptr; cudaEvent_t ev_x = nullptr; bool ev1_valid = false;   // x_real's H2D runs under the generator's forward
  std::vector<void*> allocs;
};

// B2G_PHASES=1 (diagnostic, eager launches only -- events inside a captured graph carry no time): CUDA events on the main stream at the
// phase boundaries of the step; b2g_gan_step_resident prints the intervals to stderr.  The side streams are not marked: an interval is the
// main-stream critical path between two boundaries, including whatever it had to wait for.
static bool phases_on() { static int v = -1; if (v < 0) { const char* e = getenv("B2G_PHASES"); v = (e && atoi(e)) ? 1 : 0; } return v == 1; }
static cudaEvent_t g_ph_ev[24]; static const char* g_ph_name[24]; static int g_ph_n = 0;
static void phase_mark(cudaStream_t s, const char* name) {
  if (!phases_on()) return; cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone; cudaStreamIsCapturing(s, &st); if (st != cudaStreamCaptureStatusNone || g_ph_n >= 24) return;
  if (!g_ph_ev[g_ph_n]) cudaEventCreate(&g_ph_ev[g_ph_n]);
  cudaEventRecord(g_ph_ev[g_ph_n], s); g_ph_name[g_ph_n++] = name;
}
static void phase_report(cudaStream_t s) {
  if (!phases_on() || g_ph_n < 2) { g_ph_n = 0; return; }
  cudaStreamSynchronize(s); float tot = 0.f;
  for (int i = 1; i < g_ph_n; ++i) { float ms = 0.f; cudaEventElapsedTime(&ms, g_ph_ev[i - 1], g_ph_ev[i]); tot += ms; fprintf(stderr, "[b2g phase] %-34s %8.1f us\n", g_ph_name[i], ms * 1e3f); }
  fprintf(stderr, "[b2g phase] %-34s %8.1f us\n", "total", tot * 1e3f); g_ph_n = 0;
}
// part 1: x_fake = gen.output(z_d) -- needs nothing from the host but z_d.  part 2: everything that touches x_real.
// They are two graphs so that the copy-stream event of x_real's H2D can be waited on between them (a captured stream may not
// wait on work outside its capture).
static int32_t gan_step_part1(b2g_gan* g, int N) {
  b2g_net *G = g->G, *D = g->D;
  const size_t ts = prec_size(D->prec);
  void* fake_dst = (char*)D->input + ts * (size_t)N * D->in_elems;
  FwdOpts og{N, 1, g->cfg.fake_bn_train != 0, false, fake_dst};
  phase_mark(G->ctx->stream, "start");
  int32_t r = net_forward(G, g->z_d, og, nullptr);
  phase_mark(G->ctx->stream, "G forward (inference) on z_d");
  return r;
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
  phase_mark(s, "D forward 2N (+hoisted G fwd fork)");
  k_xent(D->prec, logits, g->y_d, D->epsA, g->loss_dev, N, 2, D->cfg.xent_clip_eps, s);
  B2(net_backward(D, D->input, D->epsA, 2 * N, 2, true, false, /*allreduce_follows=*/true));
  phase_mark(s, "D loss + backward 2N (join wgrad)");
  if (under_allreduce) B2(hoisted_g_forward());
  B2(net_allreduce_grads(D));
  B2(net_update(D, 2 * N));
  phase_mark(s, "D all-reduce + update");
  // 3. G update through D on (z_g, y_gen) (J:465-471); D's parameters / running stats / updater state untouched
  CU(cudaStreamWaitEvent(s, G->ctx->ev_b, 0));
  phase_mark(s, "wait for hoisted G train forward");
  FwdOpts od2{N, 1, true, false, nullptr};
  B2(net_forward(D, xg, od2, &logits));
  phase_mark(s, "D forward N");
  k_xent(D->prec, logits, g->y_g, D->epsA, g->loss_dev + 2, N, 1, D->cfg.xent_clip_eps, s);
  // the generator's output activation (tanh) is differentiated inside D's last input-gradient kernel when that kernel can (EPI_ACTBWD)
  TcEpi ga{}; const LayerRT& gl = G->L.back(); bool ga_done = false;
  const bool ga_can = gl.has_gemm() && gl.d.act != B2G_ACT_IDENTITY && gl.d.type != B2G_LAYER_OUTPUT;
  if (ga_can) { ga.mode = EPI_ACTBWD; ga.aux = (const __nv_bfloat16*)xg; ga.act = gl.d.act; ga.alpha = gl.d.act_alpha; }
  B2(net_backward(D, xg, D->epsA, N, 1, false, true, false, ga_can ? &ga : nullptr, &ga_done));
  phase_mark(s, "D input gradient N");
  B2(net_backward(G, g->z_g, D->input_grad, N, 1, true, false, /*allreduce_follows=*/true, nullptr, nullptr, ga_done));
  phase_mark(s, "G backward (join wgrad)");
  B2(net_allreduce_grads(G));
  B2(net_update(G, N));
  phase_mark(s, "G all-reduce + update");
  return 0;
}

extern "C" int32_t b2g_gan_create(b2g_net* gen, b2g_net* dis, const b2g_gan_config* cfg, b2g_gan** out) {
  if (!gen || !dis || !out) return fail(B2G_ERR_ARG, "null");
  if (gen->ctx != dis->ctx) return fail(B2G_ERR_ARG, "generator and discriminator live on different contexts");
  if (gen->prec != dis->prec) return fail(B2G_ERR_ARG, "generator and discriminator use different precisions");
  if (gen->L.back().out_elems != dis->in_elems) return fail(B2G_ERR_SHAPE, "generator output (%zu) != discriminator input (%zu)", gen->L.back().out_elems, dis->in_elems);
  if (gen->L.back().out_alias || gen->L.back().d.type == B2G_LAYER_DROPOUT) return fail(B2G_ERR_UNSUPPORTED, "generator must end in a layer that owns its output");
  if (dis->L.back().d.type == B2G_LAYER_OUTPUT && dis->L.back().d.loss != B2G_LOSS_XENT) return fail(B2G_ERR_UNSUPPORTED, "the adversarial step needs a binary XENT discriminator");
  if (dis->cfg.bn_groups < 2 || dis->max_rows < 2) return fail(B2G_ERR_ARG, "discriminator must be created with bn_groups>=2 and max_batch = 2*N");
  int N = std::min(gen->max_rows, dis->max_rows / 2);
  CU(cudaSetDevice(gen->ctx->device));
  b2g_gan* g = new b2g_gan(); g->G = gen; g->D = dis; if (cfg) g->cfg = *cfg; g->N = N;
  const size_t ts = prec_size(gen->prec);
  auto al = [&](void** p, size_t bytes) -> int32_t { cudaError_t e = cudaMalloc(p, bytes ? bytes : 16); if (e != cudaSuccess) return fail(B2G_ERR_OOM, "cudaMalloc: %s", cudaGetErrorString(e)); g->allocs.push_back(*p); return 0; };
  int32_t r = al(&g->z_d, ts * N * gen->in_elems); if (!r) r = al(&g->z_g, ts * N * gen->in_elems);
  if (!r) r = al((void**)&g->y_d, sizeof(float) * 2 * N); if (!r) r = al((void**)&g->y_g, sizeof(float) * N); if (!r) r = al((void**)&g->loss_dev, sizeof(float) * 4);
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
  CU(cudaMemcpyAsync(g->y_d, y_real, sizeof(float) * batch, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(g->y_d + batch, y_fake, sizeof(float) * batch, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(g->y_g, y_gen, sizeof(float) * batch, cudaMemcpyHostToDevice, s));
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
  g->last_batch = batch;
  CU(cudaEventRecord(g->ev0, s));
  if (!use_graph) { B2(gan_step_part1(g, batch)); CU(cudaStreamWaitEvent(s, g->ev_x, 0)); B2(gan_step_part2(g, batch)); phase_report(s); }
  else {
    if (!g->exec || g->graph_batch != batch || g->graph_gn_g != g->G->gn_gen || g->graph_gn_d != g->D->gn_gen) {
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
      g->graph_gn_g = g->G->gn_gen; g->graph_gn_d = g->D->gn_gen;
    }
    CU(cudaGraphLaunch(g->exec1, s));
    CU(cudaStreamWaitEvent(s, g->ev_x, 0));
    CU(cudaGraphLaunch(g->exec, s)); g_launch_count += g->graph_launches; g->G->simt_gemm_calls += g->graph_simt_g; g->D->simt_gemm_calls += g->graph_simt_d;
  }
  CU(cudaEventRecord(g->ev1, s)); g->ev1_valid = true;
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
  if (mode != n->gn_mode || threshold != n->gn_threshold) { n->gn_mode = mode; n->gn_threshold = threshold; ++n->gn_gen; }
  return 0;
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
  float* bufs[3] = {n->params, n->st0, n->st1};
  for (float* b : bufs) { NC(g_nccl.ar(b, b, (size_t)n->n_params, 7, 0, c->comm, s)); k_scale_f32(b, inv, (size_t)n->n_params, s); }
  net_refresh_shadow(n);
  CU(cudaStreamSynchronize(s)); return 0;
}
extern "C" int32_t b2g_ctx_allreduce_test(b2g_ctx* c, float* host, int64_t n) {
  if (!c || !host || n < 1) return fail(B2G_ERR_ARG, "null"); if (!c->comm) return fail(B2G_ERR_NCCL, "no communicator"); CU(cudaSetDevice(c->device));
  float* d = nullptr; CU(cudaMalloc(&d, sizeof(float) * n));
  CU(cudaMemcpyAsync(d, host, sizeof(float) * n, cudaMemcpyHostToDevice, c->stream));
  NC(g_nccl.ar(d, d, (size_t)n, 7, 0, c->comm, c->stream));
  CU(cudaMemcpyAsync(host, d, sizeof(float) * n, cudaMemcpyDeviceToHost, c->stream)); CU(cudaStreamSynchronize(c->stream)); cudaFree(d); return 0;
}

// ------------------------------------------------------------------ kernel-level test hook ----------------
// The tile-width / grid overrides of tc_conv_kernel hold for the hook's own launch loop only: reset right after it, and on every early return.
struct TcTestSchedule {
  TcTestSchedule(int bn, int max_ctas) { g_tc_test_bn = bn; g_tc_test_max_ctas = max_ctas; }
  ~TcTestSchedule() { reset(); }
  void reset() { g_tc_test_bn = 0; g_tc_test_max_ctas = 0; }
};
extern "C" int32_t b2g_test_conv_ex(b2g_ctx* c, int32_t kind, int32_t impl, int32_t precision, const b2g_conv_geom* gg, const float* a_host, const float* b_host, float* out, int32_t iters, float* ms_per_iter,
                                    b2g_test_conv_opts* opt) {
  if (!c || !gg || !a_host || !b_host || !out) return fail(B2G_ERR_ARG, "null"); CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream; int prec = precision == B2G_PREC_BF16 ? PREC_BF16 : PREC_F32; size_t ts = prec_size(prec);
  ConvGeom g{gg->n, gg->h, gg->w, gg->c, gg->oh, gg->ow, gg->o, gg->kh, gg->kw, gg->sh, gg->sw, gg->ph, gg->pw};
  size_t nx = (size_t)g.N * g.H * g.W * g.C, ny = (size_t)g.N * g.OH * g.OW * g.O, nw = (size_t)g.O * g.KH * g.KW * g.C;
  // operands: kind 0: a = x (NHWC), b = w [O][KH][KW][C] -> out y ; kind 1: a = dy, b = w -> out dx ; kind 2: a = x, b = dy -> out dw (fp32)
  size_t na = kind == 1 ? ny : nx, nb = kind == 2 ? ny : nw, no = kind == 0 ? ny : kind == 1 ? nx : nw;
  const int oc = kind == 0 ? g.O : g.C;       // channels of the result (kinds 0 / 1)
  if (impl == 1) {
    if (prec != PREC_BF16 || !c->tc_ok) return fail(B2G_ERR_UNSUPPORTED, "tensor-core kernels need BF16 precision and a working tensor-map encoder");
    bool ok = kind == 0 ? tc_fprop_supported(g) : kind == 1 ? tc_dgrad_supported(g) : tc_wgrad_supported(g);
    if (!ok) return fail(B2G_ERR_UNSUPPORTED, "no tensor-core kernel for this shape");
  }
  const bool tc_conv = impl == 1 && kind != 2, ps = impl == 3 && kind == 1;     // the launches of tc_conv_kernel (ps: its pixel-shuffle form)
  if (opt && !tc_conv && !ps && (opt->epi || opt->bias || opt->scale || opt->act))
    return fail(B2G_ERR_UNSUPPORTED, "epilogue options apply to the tensor-core fprop / dgrad kernels (impl 1, kind 0 / 1) and the pixel-shuffle deconv (impl 3, kind 1)");
  if (opt && ps && (opt->scale || (opt->epi != EPI_PLAIN && opt->epi != EPI_ACTBWD)))
    return fail(B2G_ERR_UNSUPPORTED, "the pixel-shuffle deconv has bias, activation and the activation-backward epilogue only");
  const int force_bn = opt ? opt->bn : 0, max_ctas = opt ? opt->max_ctas : 0;
  const bool poison = opt && opt->poison, w_mn = opt && opt->w_mn;
  if (force_bn && (!tc_conv || (force_bn != 64 && force_bn != 128) || oc % force_bn))
    return fail(B2G_ERR_UNSUPPORTED, "bn %d: the tensor-core fprop / dgrad tile is 64 or 128 columns and must divide the %d output channels", force_bn, oc);
  if (max_ctas < 0 || (max_ctas && !tc_conv && !ps)) return fail(B2G_ERR_UNSUPPORTED, "max_ctas %d: a grid cap applies to tc_conv_kernel launches only", max_ctas);
  if (poison && kind == 2) return fail(B2G_ERR_UNSUPPORTED, "poison applies to the bf16 outputs of kinds 0 / 1");
  if (w_mn && (impl != 1 || kind != 0 || g.KH != 1 || g.KW != 1)) return fail(B2G_ERR_UNSUPPORTED, "w_mn: the [C][O] weight operand exists for the 1x1 tensor-core fprop only");
  // impl 2 = the SIMT skinny-layer kernels (kernels_edge.cu), impl 3 = their tensor-core counterparts; both need <= 4 image channels (g.C)
  if (impl == 2 || impl == 3) {
    bool ok = kind == 0 ? edge_conv_small_cin_supported(g) : kind == 1 ? edge_deconv_small_c_supported(g) : edge_wgrad_small_cin_supported(g);
    if (impl == 3) ok = ok && prec == PREC_BF16 && c->tc_ok && (kind == 0 ? tc_edge_conv_supported(g) : kind == 1 ? tc_deconv_ps_supported(g) : tc_edge_wgrad_supported(g));
    // the training step runs the pixel-shuffle deconv wherever tc_deconv_ps_supported holds, also where the SIMT kernel has no variant (O > 128)
    if (ps) ok = prec == PREC_BF16 && c->tc_ok && tc_deconv_ps_supported(g);
    if (!ok) return fail(B2G_ERR_UNSUPPORTED, "no skinny-layer kernel (impl %d) for this shape", impl);
  }
  // impl 4 = the dense (1x1 geometry) SIMT kernels: <= 4 output units (D-last) or a short reduction (G-first in its dgrad form)
  if (impl == 4 && !(dense_small_o_supported(g) || (dense_small_k_supported(g) && kind != 0))) return fail(B2G_ERR_UNSUPPORTED, "no dense kernel for this shape");
  float *fa = nullptr, *fb = nullptr, *fo = nullptr, *scratch = nullptr; void *ta = nullptr, *tb = nullptr, *to = nullptr; __nv_bfloat16* wps = nullptr;
  float *d_bias = nullptr, *d_scale = nullptr, *d_coef = nullptr, *d_auxf = nullptr; __nv_bfloat16 *d_aux = nullptr, *d_aux2 = nullptr; unsigned long long* d_acc = nullptr;
  size_t sc = std::max(std::max(std::max(k_simt_wgrad_scratch_floats(g), k_tc_wgrad_scratch_floats(g)), std::max(k_edge_wgrad_scratch_floats(g), k_tc_edge_wgrad_scratch_floats(g))), k_dense_small_o_wgrad_scratch_floats(g)) + 16;
  CU(cudaMalloc(&fa, 4 * na)); CU(cudaMalloc(&fb, 4 * nb)); CU(cudaMalloc(&fo, 4 * no)); CU(cudaMalloc(&scratch, 4 * sc));
  CU(cudaMalloc(&ta, ts * na)); CU(cudaMalloc(&tb, ts * nb)); CU(cudaMalloc(&to, ts * no));
  CU(cudaMemcpyAsync(fa, a_host, 4 * na, cudaMemcpyHostToDevice, s)); CU(cudaMemcpyAsync(fb, b_host, 4 * nb, cudaMemcpyHostToDevice, s));
  if (prec == PREC_BF16) { k_cast_f32_to_bf16(fa, (__nv_bfloat16*)ta, na, s); k_cast_f32_to_bf16(fb, (__nv_bfloat16*)tb, nb, s); }
  else { CU(cudaMemcpyAsync(ta, fa, 4 * na, cudaMemcpyDeviceToDevice, s)); CU(cudaMemcpyAsync(tb, fb, 4 * nb, cudaMemcpyDeviceToDevice, s)); }
  if (impl == 3 && kind == 1) { CU(cudaMalloc(&wps, 2 * k_tc_deconv_ps_weight_elems(g))); k_pack_deconv_ps(fb, wps, g.O, g.C, s); }
  TcEpi epi{}; const TcEpi* pe = nullptr; const float* bias = nullptr; int act = 0; float alpha = 0.f; int groups = 1;
  if (opt && (tc_conv || ps)) {
    groups = opt->groups > 0 ? opt->groups : 1; act = opt->act; alpha = opt->alpha;
    if (opt->bias) { CU(cudaMalloc(&d_bias, 4 * oc)); CU(cudaMemcpyAsync(d_bias, opt->bias, 4 * oc, cudaMemcpyHostToDevice, s)); bias = d_bias; }
    if (opt->scale) { CU(cudaMalloc(&d_scale, 4 * oc)); CU(cudaMemcpyAsync(d_scale, opt->scale, 4 * oc, cudaMemcpyHostToDevice, s)); }
    epi.mode = opt->epi; epi.scale = d_scale; epi.imgs_per_group = g.N / groups; epi.act = opt->act; epi.alpha = opt->alpha;
    if (opt->epi == EPI_STATS || opt->epi == EPI_BNBWD) { CU(cudaMalloc(&d_acc, 8 * k_bn_acc_elems(oc, groups))); epi.acc = d_acc; }
    if (opt->epi == EPI_BNBWD || opt->epi == EPI_ACTBWD) {
      if (!opt->aux) return fail(B2G_ERR_ARG, "epilogue %d needs aux", opt->epi);
      CU(cudaMalloc(&d_auxf, 4 * no)); CU(cudaMalloc(&d_aux, 2 * no)); CU(cudaMemcpyAsync(d_auxf, opt->aux, 4 * no, cudaMemcpyHostToDevice, s)); k_cast_f32_to_bf16(d_auxf, d_aux, no, s); epi.aux = d_aux;
    }
    if (opt->epi == EPI_BNBWD) {      // aux = the BatchNorm(+activation) output y, aux2 = its input z
      if (!opt->aux2) return fail(B2G_ERR_ARG, "epilogue 2 needs aux2 (the BatchNorm input z)");
      CU(cudaMalloc(&d_coef, 4 * no)); CU(cudaMalloc(&d_aux2, 2 * no)); CU(cudaMemcpyAsync(d_coef, opt->aux2, 4 * no, cudaMemcpyHostToDevice, s)); k_cast_f32_to_bf16(d_coef, d_aux2, no, s); epi.aux2 = d_aux2;
    }
    if (opt->epi || opt->scale) pe = &epi;
  }
  cudaEvent_t e0, e1; CU(cudaEventCreate(&e0)); CU(cudaEventCreate(&e1));
  int reps = iters < 1 ? 1 : iters; int rc = 0;
  g_tc_last_kernel = "";
  TcTestSchedule schedule(force_bn, max_ctas);
  for (int it = -1; it < reps; ++it) {       // it = -1: warm-up
    if (it == 0) CU(cudaEventRecord(e0, s));
    if (d_acc) CU(cudaMemsetAsync(d_acc, 0, 8 * k_bn_acc_elems(oc, groups), s));
    if (poison) CU(cudaMemsetAsync(to, 0xFF, ts * no, s));       // a tile this launch does not write reads back as NaN, not as the warm-up's values
    if (impl == 4) {
      const bool so = dense_small_o_supported(g);
      if (kind == 0) k_dense_small_o_fwd(prec, prec, g, ta, tb, nullptr, to, 0, 0.f, s);
      else if (kind == 1) { if (so) k_dense_small_o_dgrad(prec, prec, g, ta, tb, to, s); else k_dense_small_k_dgrad(prec, prec, g, ta, tb, nullptr, to, 0, 0.f, s); }
      else { if (so) k_dense_small_o_wgrad(prec, g, ta, tb, fo, scratch, 0, s); else k_dense_small_k_wgrad(prec, g, ta, tb, fo, s); }
    }
    else if (impl >= 2) {
      if (kind == 0) { if (impl == 3) rc = k_tc_edge_conv(g, (const __nv_bfloat16*)ta, (const __nv_bfloat16*)tb, nullptr, (__nv_bfloat16*)to, 0, 0.f, s); else k_edge_conv_small_cin(prec, prec, g, ta, tb, nullptr, to, 0, 0.f, s); }
      else if (kind == 1) { if (impl == 3) rc = k_tc_deconv_ps(g, (const __nv_bfloat16*)ta, wps, bias, (__nv_bfloat16*)to, act, alpha, s, pe); else k_edge_deconv_small_c(prec, prec, g, ta, tb, nullptr, to, 0, 0.f, s); }
      else { if (impl == 3) rc = k_tc_edge_wgrad(g, (const __nv_bfloat16*)ta, (const __nv_bfloat16*)tb, fo, nullptr, scratch, sc, 0, s); else k_edge_wgrad_small_cin(prec, g, ta, tb, fo, scratch, 0, s); }
    }
    else if (kind == 0) { if (impl) rc = k_tc_fprop(g, (const __nv_bfloat16*)ta, (const __nv_bfloat16*)tb, bias, (__nv_bfloat16*)to, act, alpha, s, pe, w_mn ? 1 : 0); else k_simt_fprop(prec, prec, g, ta, tb, nullptr, to, 0, 0.f, s); }
    else if (kind == 1) { if (impl) rc = k_tc_dgrad(g, (const __nv_bfloat16*)ta, (const __nv_bfloat16*)tb, bias, (__nv_bfloat16*)to, act, alpha, s, pe); else k_simt_dgrad(prec, prec, g, ta, tb, nullptr, to, 0, 0.f, s); }
    else { if (impl) rc = k_tc_wgrad(g, (const __nv_bfloat16*)ta, (const __nv_bfloat16*)tb, fo, scratch, sc, 0, s); else k_simt_wgrad(prec, g, ta, tb, fo, scratch, sc, 0, s); }
    if (rc) break;
  }
  schedule.reset();
  CU(cudaEventRecord(e1, s));
  if (rc) return fail(B2G_ERR_CUDA, "tensor-core kernel launch failed (%d)", rc);
  if (opt) { strncpy(opt->kernel, g_tc_last_kernel, sizeof(opt->kernel) - 1); opt->kernel[sizeof(opt->kernel) - 1] = 0; }
  if (kind != 2) { if (prec == PREC_BF16) { /* widen */ k_nhwc_to_nchw_f32(prec, to, fo, 1, 1, (int)no, s); } else CU(cudaMemcpyAsync(fo, to, 4 * no, cudaMemcpyDeviceToDevice, s)); }
  CU(cudaMemcpyAsync(out, fo, 4 * no, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s)); CHECK_KERNELS();
  if (d_acc && opt && opt->stats) {      // [groups][2][C] doubles from the [groups][2][2][C] hi | lo words
    std::vector<long long> h(k_bn_acc_elems(oc, groups)); CU(cudaMemcpy(h.data(), d_acc, 8 * h.size(), cudaMemcpyDeviceToHost));
    for (int gi = 0; gi < groups; ++gi) for (int st = 0; st < 2; ++st) for (int ch = 0; ch < oc; ++ch)
      opt->stats[((size_t)gi * 2 + st) * oc + ch] = (double)h[((size_t)(gi * 2 + st) * 2 + 0) * oc + ch] / 1024.0 + (double)h[((size_t)(gi * 2 + st) * 2 + 1) * oc + ch] / 1152921504606846976.0;
  }
  float ms = 0.f; CU(cudaEventElapsedTime(&ms, e0, e1)); if (ms_per_iter) *ms_per_iter = ms / reps;
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  cudaFree(fa); cudaFree(fb); cudaFree(fo); cudaFree(scratch); cudaFree(ta); cudaFree(tb); cudaFree(to); if (wps) cudaFree(wps);
  if (d_bias) cudaFree(d_bias); if (d_scale) cudaFree(d_scale); if (d_coef) cudaFree(d_coef); if (d_auxf) cudaFree(d_auxf); if (d_aux) cudaFree(d_aux); if (d_aux2) cudaFree(d_aux2); if (d_acc) cudaFree(d_acc);
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
  const size_t n = (size_t)groups * rows * C, gc = (size_t)groups * C, ts = prec_size(prec);
  std::vector<void*> mem;
  auto alloc = [&](void** p, size_t bytes) -> int32_t { *p = nullptr; CU(cudaMalloc(p, bytes)); mem.push_back(*p); return 0; };
  auto release = [&]() { for (void* p : mem) cudaFree(p); mem.clear(); };
  float *fx, *fe, *fo, *d_par, *d_grad, *d_stat, *scratch, *coef, *unit; void *tx, *te, *ty, *tei; unsigned long long* acc;
  int32_t r = 0;
  if ((r = alloc((void**)&fx, 4 * n)) || (r = alloc((void**)&fe, 4 * n)) || (r = alloc((void**)&fo, 4 * n)) || (r = alloc(&tx, ts * n)) || (r = alloc(&te, ts * n)) ||
      (r = alloc(&ty, ts * n)) || (r = alloc(&tei, ts * n)) || (r = alloc((void**)&d_par, 4 * 4 * (size_t)C)) || (r = alloc((void**)&d_grad, 4 * 4 * (size_t)C)) ||
      (r = alloc((void**)&d_stat, 4 * 2 * gc)) || (r = alloc((void**)&scratch, 4 * k_bn_scratch_floats(C, groups))) || (r = alloc((void**)&coef, 4 * 4 * gc)) ||
      (r = alloc((void**)&unit, 4 * 4 * gc)) || (r = alloc((void**)&acc, 8 * 2 * k_bn_acc_elems(C, groups)))) { release(); return r; }
  float *d_gamma = d_par, *d_beta = d_par + C, *d_rm = d_par + 2 * C, *d_rv = d_par + 3 * C;
  float *d_gg = d_grad, *d_gb = d_grad + C, *d_gm = d_grad + 2 * C, *d_gv = d_grad + 3 * C, *d_mean = d_stat, *d_is = d_stat + gc;
  unsigned long long *acc_f = acc, *acc_b = acc + k_bn_acc_elems(C, groups);
  auto up = [&](float* d, const float* h, size_t k) { return cudaMemcpyAsync(d, h, 4 * k, cudaMemcpyHostToDevice, s); };
  if (up(fx, x, n) || up(fe, eps_out, n) || up(d_gamma, gamma, C) || up(d_beta, beta, C) || up(d_rm, run_mean, C) || up(d_rv, run_var, C) ||
      up(d_gg, g_gamma, C) || up(d_gb, g_beta, C) || cudaMemsetAsync(acc, 0, 8 * 2 * k_bn_acc_elems(C, groups), s)) { release(); return fail(B2G_ERR_CUDA, "BatchNorm test upload failed"); }
  if (prec == PREC_BF16) { k_cast_f32_to_bf16(fx, (__nv_bfloat16*)tx, n, s); k_cast_f32_to_bf16(fe, (__nv_bfloat16*)te, n, s); }
  else { cudaMemcpyAsync(tx, fx, 4 * n, cudaMemcpyDeviceToDevice, s); cudaMemcpyAsync(te, fe, 4 * n, cudaMemcpyDeviceToDevice, s); }
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
  auto down = [&](float* h, const void* t) -> int32_t {     // widen a T tensor to fp32 and copy it out
    k_nhwc_to_nchw_f32(prec, t, fo, 1, 1, (int)n, s); CU(cudaMemcpyAsync(h, fo, 4 * n, cudaMemcpyDeviceToHost, s)); CU(cudaStreamSynchronize(s)); return 0;
  };
  if ((r = down(y, ty)) || (r = down(eps_in, tei))) { release(); return r; }
  cudaError_t e = cudaSuccess;
  float* hs[6] = {g_gamma, g_beta, g_mean, g_var, mean, invstd}; const float* ds[6] = {d_gg, d_gb, d_gm, d_gv, d_mean, d_is}; const size_t ks[6] = {(size_t)C, (size_t)C, (size_t)C, (size_t)C, gc, gc};
  for (int k = 0; k < 6 && e == cudaSuccess; ++k) e = cudaMemcpyAsync(hs[k], ds[k], 4 * ks[k], cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e == cudaSuccess) e = cudaGetLastError();
  release();
  if (e != cudaSuccess) return fail(B2G_ERR_CUDA, "BatchNorm test: %s", cudaGetErrorString(e));
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
  std::vector<void*> mem;
  auto alloc = [&](void** q, size_t bytes) -> int32_t { *q = nullptr; CU(cudaMalloc(q, bytes)); mem.push_back(*q); return 0; };
  auto release = [&]() { for (void* q : mem) cudaFree(q); mem.clear(); };
  float *fx, *fe; void *tx, *te, *ty; uint32_t* mask; unsigned long long* dpass; unsigned* ticket; int32_t r = 0;
  if ((r = alloc((void**)&fx, 4 * n)) || (r = alloc((void**)&fe, 4 * n)) || (r = alloc(&tx, ts * n)) || (r = alloc(&te, ts * n)) || (r = alloc(&ty, ts * n)) ||
      (r = alloc((void**)&mask, 4 * ((n + 31) / 32))) || (r = alloc((void**)&dpass, sizeof(unsigned long long))) || (r = alloc((void**)&ticket, sizeof(unsigned)))) { release(); return r; }
  const unsigned long long p0 = (unsigned long long)pass;
  cudaError_t e = cudaMemcpyAsync(fx, x, 4 * n, cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(fe, dy, 4 * n, cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(dpass, &p0, sizeof(p0), cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaMemsetAsync(ticket, 0, sizeof(unsigned), s);
  if (e != cudaSuccess) { release(); return fail(B2G_ERR_CUDA, "dropout test upload: %s", cudaGetErrorString(e)); }
  if (prec == PREC_BF16) { k_cast_f32_to_bf16(fx, (__nv_bfloat16*)tx, n, s); k_cast_f32_to_bf16(fe, (__nv_bfloat16*)te, n, s); }
  else { cudaMemcpyAsync(tx, fx, 4 * n, cudaMemcpyDeviceToDevice, s); cudaMemcpyAsync(te, fe, 4 * n, cudaMemcpyDeviceToDevice, s); }
  const DropoutArgs a = make_dropout_args(seed, layer, rank, p);
  k_dropout_fwd(prec, tx, ty, mask, n, a, dpass, ticket, 1, s);
  k_dropout_bwd(prec, te, te, mask, n, a.scale, s);
  unsigned long long p1 = 0;
  k_nhwc_to_nchw_f32(prec, ty, fx, 1, 1, (int)n, s);
  k_nhwc_to_nchw_f32(prec, te, fe, 1, 1, (int)n, s);
  e = cudaMemcpyAsync(y, fx, 4 * n, cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(dx, fe, 4 * n, cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(&p1, dpass, sizeof(p1), cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e == cudaSuccess) e = cudaGetLastError();
  release();
  if (e != cudaSuccess) return fail(B2G_ERR_CUDA, "dropout test: %s", cudaGetErrorString(e));
  if (p1 != p0 + 1) return fail(B2G_ERR_CUDA, "dropout test: the forward left the pass counter at %llu, expected %llu", p1, p0 + 1);
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

// Times the HBM-bound kernels of the step in isolation (bench.py's `hbm` roofline entries): every launch is bracketed by its own CUDA events
// on the library stream and preceded by an L2 flush (a 256 MiB memset), so the operands really come from HBM as they do inside a step.
// ms[0] = one updater pass over `net` (Adam: 28 B/param + 2 B bf16 operand copy; the net's parameters are perturbed -- bench only),
// ms[1] = BatchNorm apply (read + write a [groups*rows x C] bf16 tensor), ms[2] = BatchNorm backward apply (two reads + one write).
extern "C" int32_t b2g_test_hbm_kernels(b2g_net* n, int32_t rows, int32_t channels, int32_t iters, float* ms3) {
  if (!n || !ms3 || rows < 8 || iters < 1) return fail(B2G_ERR_ARG, "bad arguments"); b2g_ctx* c = n->ctx; CU(cudaSetDevice(c->device)); cudaStream_t s = c->stream;
  if (!k_bn_vec_ok(PREC_BF16, channels)) return fail(B2G_ERR_UNSUPPORTED, "channels %d not supported by the vector BatchNorm kernels", channels);
  const size_t ne = (size_t)rows * channels; __nv_bfloat16 *x = nullptr, *e = nullptr, *y = nullptr; float *coef = nullptr, *gb = nullptr; unsigned long long* acc = nullptr;
  CU(cudaMalloc(&x, 2 * ne)); CU(cudaMalloc(&e, 2 * ne)); CU(cudaMalloc(&y, 2 * ne)); CU(cudaMalloc(&coef, 4 * 4 * channels)); CU(cudaMalloc(&gb, 4 * 4 * channels)); CU(cudaMalloc(&acc, 8 * k_bn_acc_elems(channels, 1)));
  CU(cudaMemsetAsync(x, 0x3c, 2 * ne, s)); CU(cudaMemsetAsync(e, 0x3c, 2 * ne, s)); CU(cudaMemsetAsync(acc, 0, 8 * k_bn_acc_elems(channels, 1), s)); k_fill_f32(coef, 1.0f, 4 * channels, s); k_fill_f32(gb, 1.0f, 4 * channels, s);
  cudaEvent_t e0, e1; CU(cudaEventCreate(&e0)); CU(cudaEventCreate(&e1));
  ms3[0] = ms3[1] = ms3[2] = 0.f;
  for (int which = 0; which < 3; ++which) for (int it = -1; it < iters; ++it) {
    B2(b2g_flush_l2(c));
    CU(cudaEventRecord(e0, s));
    if (which == 0) k_updater(n->params, n->grads, n->st0, n->st1, n->segs_dev, n->chunk_seg_dev, n->chunk_off_dev, n->nchunks, 1.0f, 1.0f, n->step_dev, n->upd_ticket, n->shadow, nullptr, s);
    else if (which == 1) k_bn_apply_acc(x, y, rows, channels, 1, acc, gb, gb + channels, ACT_LRELU, 0.2f, 1e-5f, coef, gb + 2 * channels, gb + 3 * channels, nullptr, nullptr, 0.9f, s);
    else k_bn_bwd_apply_acc(x, e, y, rows, channels, 1, coef, ACT_LRELU, 0.2f, 1, acc, gb, gb + channels, 0, s);
    CU(cudaEventRecord(e1, s)); CU(cudaEventSynchronize(e1));
    float ms = 0.f; CU(cudaEventElapsedTime(&ms, e0, e1)); if (it >= 0) ms3[which] += ms / iters;
  }
  CHECK_KERNELS();
  cudaEventDestroy(e0); cudaEventDestroy(e1); cudaFree(x); cudaFree(e); cudaFree(y); cudaFree(coef); cudaFree(gb); cudaFree(acc);
  return 0;
}
