/*
 * b200gan.h -- C-ABI of libb200gan.so: the H100-native (sm_90a) execution engine behind the DL4J
 * ComputationGraph / Layer API used by hamaadshah/gan_deeplearning4j.
 *
 * This is the drop-in boundary (SURVEY.md section 8b): plain pointers and sizes, no C++/torch types.
 * The Java facade (java/, same package/class/method names the reference driver imports, J:21-58) reaches
 * it through the primitive-only JNI shim (jni/b200gan_jni.cpp); the Python host mirror
 * (gan_deeplearning4j_b200/) and every test reach the SAME functions through ctypes.
 *
 * J = Java/src/main/java/org/deeplearning4j/dl4jGANComputerVision.java of the reference repository
 *
 * Conventions
 *   - every function returns int32: 0 = OK, <0 = b2g_status error; text via b2g_last_error().
 *     Nothing throws or aborts across the boundary (DL4J helpers throw; the facade maps !=0 to
 *     IllegalStateException like DL4J does).
 *   - the library owns all device memory (one arena per net, sized at b2g_net_create); host buffers
 *     are only read/written during the call (like INDArray.assign / setParam copying into the
 *     flattened parameter view).
 *   - host tensors cross in DL4J layouts: activations NCHW (or [N,F]) fp32, conv W [nOut,nIn,kH,kW] 'c',
 *     deconv W [nIn,nOut,kH,kW] 'c', dense W [nIn,nOut] 'f', i.e. exactly the element order of DL4J's
 *     flattened parameter vector (ConvolutionParamInitializer [b|W], DefaultParamInitializer [W|b],
 *     BatchNormalizationParamInitializer [gamma|beta|mean|var]).  Internally everything is NHWC.
 *   - a b2g_ctx is single-threaded (the caller serialises), one CUDA device, one compute stream.
 */
#ifndef B200GAN_H
#define B200GAN_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2G_VERSION 101
#define B2G_NAME_LEN 64

typedef struct b2g_ctx b2g_ctx;
typedef struct b2g_net b2g_net;
typedef struct b2g_gan b2g_gan;

typedef enum {
  B2G_OK = 0,
  B2G_ERR_ARG = -1,        /* bad argument / unknown layer or parameter name */
  B2G_ERR_SHAPE = -2,      /* shape mismatch (DL4J: DL4JInvalidInputException) */
  B2G_ERR_CUDA = -3,       /* CUDA runtime / driver error (text in b2g_last_error) */
  B2G_ERR_NCCL = -4,
  B2G_ERR_OOM = -5,
  B2G_ERR_UNSUPPORTED = -6,
  B2G_ERR_NO_DEVICE = -7   /* no sm_90 device: there is NO CPU fallback */
} b2g_status;

/* Layer vocabulary = {what the reference file builds} U {what north_star names}. */
typedef enum {
  B2G_LAYER_CONV2D = 0,      /* ConvolutionLayer.Builder(kH,kW).stride().padding().nIn().nOut()   J:135-140,203-219 */
  B2G_LAYER_DECONV2D = 1,    /* Deconvolution2D (north_star's ConvolutionTranspose2D)                              */
  B2G_LAYER_BATCHNORM = 2,   /* BatchNormalization.Builder()                                      J:132-134,186-199 */
  B2G_LAYER_DENSE = 3,       /* DenseLayer.Builder().nOut()                                       J:155-158,189-196 */
  B2G_LAYER_ACTIVATION = 4,  /* ActivationLayer (ReLU / LeakyReLU after BatchNormalization)                        */
  B2G_LAYER_MAXPOOL = 5,     /* SubsamplingLayer.Builder(PoolingType.MAX).kernelSize().stride()   J:141-144,151-154 */
  B2G_LAYER_UPSAMPLE2D = 6,  /* Upsampling2D.Builder(size)                                        J:201-202,210-211 */
  B2G_LAYER_OUTPUT = 7,      /* OutputLayer.Builder(LossFunction.XENT).activation(SIGMOID).nOut() J:159-163,303-308 */
  B2G_LAYER_LOSS = 8,        /* LossLayer(XENT, sigmoid): loss on incoming logits (DCGAN D-last conv)              */
  B2G_LAYER_FF_TO_CNN = 9,   /* FeedForwardToCnnPreProcessor(h,w,c)                               J:200,255         */
  B2G_LAYER_CNN_TO_FF = 10,  /* CnnToFeedForwardPreProcessor (auto-inserted by setInputTypes, SURVEY.md 3.1)       */
  B2G_LAYER_DROPOUT = 11     /* DropoutLayer.Builder(p): p = RETAIN probability in (0, 1], carried in act_alpha; no parameters */
} b2g_layer_type;

/* DropoutLayer (inverted dropout, DL4J 1.0.0-beta3).  Train-mode forward y = x * m, m = 1/p (fp32 1.0f / p) with probability p, else 0;
 * y = x * (1/p) is formed in fp32 and rounded once to the activation type, dropped elements are +0.  Backward dx = dy * m with the forward's
 * mask (kept as one bit per element).  Inference (train = 0) and a frozen DropoutLayer (FrozenLayer = test mode) are the identity, launch
 * nothing and b2g_net_get_activation returns the layer's input.
 * The mask is a pure function of (S, r, L, P, e), so the same on every run and in both precisions:
 *   S = b2g_net_config.seed (0 -> 666), r = the context's rank (0 without a communicator), L = the layer's index in the b2g_layer_desc array,
 *   P = the net's dropout pass counter, e = ((row*H + h)*W + w)*C + c the element's NHWC index in the pass (row = position in the pass batch);
 *   (x0,x1,x2,x3) = Philox4x32-10(ctr = {e >> 2, lo32(P), hi32(P), L | (r << 16)}, key = {lo32(S), hi32(S)})
 *   keep(e) = p >= 1  ||  x[e & 3] < (uint32)floor(p * 2^32)
 * P is a 64-bit word in device memory, 0 at b2g_net_create.  Every train-mode forward of a net with at least one masking DropoutLayer
 * (train, not frozen, p < 1) uses the current P for all of them and then advances P by 1 on the device (so a replayed CUDA graph draws new
 * masks); other forwards leave it unchanged.  In the GAN step D's real|fake pass (2N rows) uses P and the generator step's D pass P + 1.
 * A pass may hold at most 2^34 elements (max_batch * layer size; B2G_ERR_UNSUPPORTED at b2g_net_create). */

typedef enum {               /* org.nd4j.linalg.activations.Activation  J:126,162,215 */
  B2G_ACT_IDENTITY = 0, B2G_ACT_TANH = 1, B2G_ACT_SIGMOID = 2, B2G_ACT_RELU = 3, B2G_ACT_LRELU = 4
} b2g_activation;

typedef enum {               /* org.nd4j.linalg.learning.config.*  J:133 (RmsProp), north_star (Adam) */
  B2G_UPD_SGD = 0, B2G_UPD_RMSPROP = 1, B2G_UPD_ADAM = 2, B2G_UPD_NOOP = 3
} b2g_updater;

typedef enum { B2G_PREC_FP32 = 0, B2G_PREC_BF16 = 1 } b2g_precision;
typedef enum { B2G_LOSS_XENT = 0, B2G_LOSS_MCXENT = 1 } b2g_loss;

/* One layer of a chain-shaped ComputationGraph (every graph in the reference is a chain, J:118-310). */
typedef struct {
  int32_t type;                 /* b2g_layer_type */
  char name[B2G_NAME_LEN];      /* DL4J vertex name, e.g. "dis_conv2d_layer_2" */
  int32_t n_in, n_out;          /* channels / features (n_in may be 0 = infer, like setInputTypes) */
  int32_t k_h, k_w, s_h, s_w, p_h, p_w;   /* conv / deconv / pool geometry; upsample factor in k_h */
  int32_t has_bias;             /* hasBias(true) default */
  int32_t act;                  /* b2g_activation */
  float act_alpha;              /* ActivationLReLU alpha: DL4J default 0.01, DCGAN passes 0.2; DropoutLayer retain probability p */
  int32_t updater;              /* b2g_updater; "frozen" in the reference = RMSPROP with lr 0 (J:84) */
  float lr, beta1, beta2, eps;  /* RmsProp: beta1 = rmsDecay (ctor order lr, rmsDecay, epsilon; J:133 passes 1e-8, 1e-8) */
  float l2;                     /* .l2(1e-4) (J:125): weights only, applied AFTER the updater, not lr-scaled */
  float bn_decay, bn_eps;       /* BatchNormalization defaults 0.9 / 1e-5 */
  int32_t pre_h, pre_w, pre_c;  /* FF_TO_CNN target shape */
  int32_t loss;                 /* OUTPUT layer: 0 = LossFunction.XENT + sigmoid (J:159-163), 1 = MCXENT + softmax (J:357-362) */
  int32_t frozen;               /* TransferLearning.setFeatureExtractor (J:350): FrozenLayer = test-mode forward, no gradient, no update */
} b2g_layer_desc;

typedef struct {
  int32_t in_h, in_w, in_c;     /* InputType.convolutionalFlat(h,w,c) / convolutional; feedForward(n): h=w=1,c=n */
  int32_t max_batch;            /* largest minibatch any call will present */
  int32_t precision;            /* b2g_precision: FP32 = DL4J-parity mode; BF16 = tensor-core mode */
  float grad_clip;              /* GradientNormalization.ClipElementWiseAbsoluteValue threshold (J:123-124); 0 = off */
  float xent_clip_eps;          /* LossBinaryXENT clipEps: 1e-5 = DL4J-exact, 0 = BCE-with-logits (north_star) */
  int32_t bn_groups;            /* >1: statistics per contiguous batch group (the GAN step runs real|fake as 2 groups) */
  uint64_t seed;                /* .seed(666) (J:121): Xavier-normal init from a counter-based generator */
} b2g_net_config;

/* ---------------------------------------------------------------- context ------------------------- */
int32_t b2g_version(void);
/* Replaces Nd4j backend selection + CudaEnvironment.getInstance().getConfiguration()... (J:103-115). */
int32_t b2g_ctx_create(int32_t device, b2g_ctx** out);
int32_t b2g_ctx_destroy(b2g_ctx* ctx);
const char* b2g_last_error(void);                 /* thread-local message of the last failing call */
int32_t b2g_sync(b2g_ctx* ctx);                    /* the only host<->device sync point besides get_* */
/* kernels launched by this library on ctx since creation (bench.py's gpu_launches evidence) */
int32_t b2g_launch_count(b2g_ctx* ctx, uint64_t* out);
/* CUDA-event stopwatch on the ctx stream: start records an event; stop records, synchronises and returns ms. */
int32_t b2g_timer_start(b2g_ctx* ctx);
int32_t b2g_timer_stop_ms(b2g_ctx* ctx, float* ms);
/* write a buffer larger than L2 (measurement hygiene between timed iterations) */
int32_t b2g_flush_l2(b2g_ctx* ctx);
int32_t b2g_device_info(b2g_ctx* ctx, int32_t* sm_count, int32_t* cc_major, int32_t* cc_minor, uint64_t* mem_bytes);

/* ---------------------------------------------------------------- nets ---------------------------- */
/* new ComputationGraph(conf).init() (J:118-166): infers nIn, allocates the flattened params/grads/
 * updater-state arena and every activation buffer; Xavier-normal weights, BN gamma=1 beta=0 mean=0 var=1. */
int32_t b2g_net_create(b2g_ctx* ctx, const b2g_net_config* cfg, const b2g_layer_desc* layers, int32_t n_layers, b2g_net** out);
int32_t b2g_net_destroy(b2g_net* net);
int32_t b2g_net_num_params(b2g_net* net, int64_t* out);                       /* ComputationGraph.numParams() */
int32_t b2g_net_output_size(b2g_net* net, int64_t* per_example);              /* elements per example of output() */
int32_t b2g_net_layer_output_size(b2g_net* net, int32_t layer, int64_t* per_example);
/* Layer.getParam / setParam (J:429-510): name in {"W","b","gamma","beta","mean","var"}; host fp32 in
 * DL4J flattened-view order; n = element count (checked). */
int32_t b2g_net_set_param(b2g_net* net, const char* layer, const char* param, const float* host, int64_t n);
int32_t b2g_net_get_param(b2g_net* net, const char* layer, const char* param, float* host, int64_t n);
/* ComputationGraph.params() / setParams(): the whole flattened vector in DL4J order (== coefficients.bin payload). */
int32_t b2g_net_get_params(b2g_net* net, float* host, int64_t n);
int32_t b2g_net_set_params(b2g_net* net, const float* host, int64_t n);
/* ComputationGraph.gradient(): summed (not minibatch-divided) gradients of the last backward, DL4J order. */
int32_t b2g_net_get_gradients(b2g_net* net, float* host, int64_t n);
/* updater state (ModelSerializer updaterState.bin payload): [state0 | state1] each in params order. */
int32_t b2g_net_get_updater_state(b2g_net* net, float* host, int64_t n);
int32_t b2g_net_set_updater_state(b2g_net* net, const float* host, int64_t n);
/* ComputationGraph.output(x)[0] (J:170,420): inference mode (BN uses mean/var). x: [batch, in] NCHW fp32 host;
 * out: [batch, out] NCHW fp32 host.  train!=0 gives the train-mode forward (batch statistics). */
int32_t b2g_net_output(b2g_net* net, const float* x, int32_t batch, int32_t train, float* out);
/* Activations of one layer from the most recent forward (parity tests): NCHW fp32. */
int32_t b2g_net_get_activation(b2g_net* net, int32_t layer, int32_t batch, float* host);
/* computeGradientAndScore(): train-mode forward, XENT loss vs labels y [batch,1], backprop.
 * score = sum(loss)/batch + 0.5*l2*||W||^2 ; gradients stay on device (b2g_net_get_gradients).
 * Labels y are [batch, nOut] (nOut = 1 for XENT; one-hot rows for MCXENT). */
int32_t b2g_net_compute_gradient_and_score(b2g_net* net, const float* x, const float* y, int32_t batch, float* score);
/* epsilon w.r.t. the network input from the last backward (NCHW fp32; what the stacked gan graph feeds the generator). */
int32_t b2g_net_get_input_gradient(b2g_net* net, int32_t batch, float* host);
/* ComputationGraph.fit(DataSet) (J:426,471 via SparkComputationGraph): one minibatch =
 * computeGradientAndScore + [gradient all-reduce if a communicator is attached] + updater + params.subi. */
int32_t b2g_net_fit(b2g_net* net, const float* x, const float* y, int32_t batch, float* score);
/* The updater's iteration counter (BaseMultiLayerUpdater's iteration; Adam's t = iteration + 1).  ModelSerializer keeps it in
 * configuration.json ("iterationCount"); a restore that drops it restarts Adam's bias correction with warm moments (J:606-618). */
int32_t b2g_net_get_iteration(b2g_net* net, int64_t* out);
int32_t b2g_net_set_iteration(b2g_net* net, int64_t iteration);
/* The dropout pass counter P (see B2G_LAYER_DROPOUT); a checkpoint carries it so that a resumed run draws the masks of an uninterrupted one.
 * Both are sync points, like get_iteration. */
int32_t b2g_net_get_dropout_pass(b2g_net* net, int64_t* out);
int32_t b2g_net_set_dropout_pass(b2g_net* net, int64_t pass);
/* GradientNormalization (DL4J 1.0.0-beta3 BaseMultiLayerUpdater.preApply; the values are DL4J's ordinals).  Set per net; it applies wherever the
 * net's updater runs (b2g_net_fit, the D and G updates of b2g_gan_step, parameter-averaging mode) and takes effect at the next update.
 * The order of one update is  g /= mb  ->  normalization  ->  updater  ->  + l2*W  ->  theta -= g,  where g /= mb is the division the updater
 * already does (BatchNorm running-stat pseudo-gradients are not divided by mb; under a gradient all-reduce they are averaged over ranks).
 *   RENORM_L2_LAYER (1):  g <- g / ||g_layer||_2, dividing by 1e-5 instead when the norm is exactly 0; the threshold is ignored.
 *   RENORM_L2_PARAM (2):  the same per parameter tensor (W, b, gamma, beta, mean, var).
 *   CLIP_ELEMENTWISE (3): not accepted here: it is b2g_net_config.grad_clip.
 *   CLIP_L2_LAYER (4):    g <- g * threshold / ||g_layer||_2 when ||g_layer||_2 > threshold (a norm equal to the threshold is not scaled).
 *   CLIP_L2_PARAM (5):    the same per parameter tensor.
 * A layer is one b2g_layer_desc entry with parameters that is not frozen; its gradient is its whole contiguous range of the flattened vector,
 * so a BatchNorm layer's mean/var pseudo-gradients count in its norm and are scaled with it (as grad_clip clips them).  The norm is summed in
 * double over the fp32 values of g after the division, the multiplier is rounded to fp32 once and multiplied into g.  Under a gradient
 * all-reduce the norm is that of the all-reduced gradient, so every rank derives the same multipliers.  b2g_net_get_gradients still returns
 * the raw summed gradients.  An L2 mode adds one kernel launch per update; B2G_GN_NONE launches what a net without normalization launches. */
typedef enum {
  B2G_GN_NONE = 0, B2G_GN_RENORM_L2_LAYER = 1, B2G_GN_RENORM_L2_PARAM = 2, B2G_GN_CLIP_ELEMENTWISE = 3, B2G_GN_CLIP_L2_LAYER = 4, B2G_GN_CLIP_L2_PARAM = 5
} b2g_gradient_normalization;
/* mode in {0, 1, 2, 4, 5}; the clip modes need a finite threshold > 0.  B2G_ERR_ARG for mode 3 (use grad_clip), an unknown mode, a bad
 * threshold, or an L2 mode on a net created with grad_clip > 0 (DL4J allows one mode per layer). */
int32_t b2g_net_set_gradient_normalization(b2g_net* net, int32_t mode, float threshold);
/* BF16 nets: how many GEMM-shaped operations ran on the SIMT kernels instead of the tensor-core kernels since creation (skinny layers by design, or a
 * shape the tensor-core kernels do not tile).  north_star: no silent fallback -- bench.py prints it per step. */
int32_t b2g_net_simt_gemm_calls(b2g_net* net, uint64_t* out);

/* ---------------------------------------------------------------- the fused GAN step -------------- */
/* The adversarial iteration J:408-471 with dis / gan / gen sharing storage (the 28 setParam copies J:429-510
 * become aliasing): x_fake = G.output(z_d); D update on (x_real,y_real)+(x_fake,y_fake); G update through D on
 * (z_g, y_gen).  See oracle/dl4j_oracle.py::gan_step for the exact arithmetic. */
typedef struct {
  int32_t fake_bn_train;   /* 0: x_fake from inference-mode BN (gen.output, J:420); 1: batch statistics */
  int32_t use_cuda_graph;  /* capture the whole step once and replay it */
} b2g_gan_config;
int32_t b2g_gan_create(b2g_net* gen, b2g_net* dis, const b2g_gan_config* cfg, b2g_gan** out);
int32_t b2g_gan_destroy(b2g_gan* gan);
/* Host-buffer entry point (what the Java driver calls): x_real [N,C,H,W] fp32, z_d/z_g [N,z], labels [N,1].
 * losses[3] = {mean D loss on real, mean D loss on fake, mean G loss}. Copies are part of the call. */
int32_t b2g_gan_step(b2g_gan* gan, const float* x_real, const float* z_d, const float* z_g,
                     const float* y_real, const float* y_fake, const float* y_gen, int32_t batch, float* losses);
/* Device-resident variant: inputs already uploaded with b2g_gan_upload (or a previous step); nothing crosses PCIe. */
int32_t b2g_gan_upload(b2g_gan* gan, const float* x_real, const float* z_d, const float* z_g,
                       const float* y_real, const float* y_fake, const float* y_gen, int32_t batch);
int32_t b2g_gan_step_resident(b2g_gan* gan, int32_t batch);
int32_t b2g_gan_read_losses(b2g_gan* gan, float* losses);   /* syncs */
/* CUDA-event time of the last b2g_gan_step_resident call, in ms (measured on the launching stream). */
int32_t b2g_gan_last_step_ms(b2g_gan* gan, float* ms);

/* ---------------------------------------------------------------- data parallel -------------------- */
/* Replaces SparkComputationGraph + ParameterAveragingTrainingMaster (J:325-333): one process per GPU, one
 * ncclAllReduce(sum) of the gradient vector per D / G update.  The unique id is created on rank 0 and
 * distributed by the host (torch.distributed store / any side channel). */
#define B2G_NCCL_ID_BYTES 128
int32_t b2g_comm_unique_id(void* id128);
int32_t b2g_ctx_comm_init(b2g_ctx* ctx, int32_t world, int32_t rank, const void* id128);
int32_t b2g_ctx_comm_destroy(b2g_ctx* ctx);
/* ParameterAveragingTrainingMaster semantics (J:325-330; Python/gan.ipynb:182-186): Theta <- mean over ranks of theta_i, and
 * likewise the updater state.  The host calls it every `averagingFrequency` local b2g_net_fit minibatches on nets whose gradient
 * all-reduce is switched off (b2g_net_set_grad_allreduce(net, 0)) -- the reference's own data-parallel rule, kept as an option
 * next to the per-update gradient all-reduce north_star mandates. */
int32_t b2g_net_set_grad_allreduce(b2g_net* net, int32_t enabled);
int32_t b2g_net_average_parameters(b2g_net* net);
/* SURVEY.md 8e options.  sync_bn: BatchNorm statistics (forward sums and the two backward reductions) are pooled over all ranks -- the 64-bit
 * integer accumulators are all-reduced, so every rank derives bit-identical statistics and "W ranks x N/W == 1 rank x N" holds; default off
 * (= local statistics per replica, what the reference's Spark workers do).  BF16 nets only.
 * grad_payload_bf16: the gradient all-reduce travels as bf16 (half the bytes); default fp32 (data parallel == single GPU, bit for bit). */
int32_t b2g_net_set_sync_bn(b2g_net* net, int32_t enabled);
int32_t b2g_net_set_grad_payload_bf16(b2g_net* net, int32_t enabled);
/* COLLECTIVE over the communicator (every rank, nets in the same order): map every rank's gradient vector into this process (CUDA IPC over
 * NVLink) and run the gradient all-reduce as ONE peer-memory kernel (reduce-scatter + all-gather, fixed summation order: replicas stay
 * bit-identical) instead of ncclAllReduce.  *enabled = 1 if every rank could map, else all ranks keep NCCL.  Replaces the network transport of
 * ParameterAveragingTrainingMaster's aggregation (reference J:325-333) on one NVSwitch node. */
int32_t b2g_net_enable_p2p_allreduce(b2g_net* net, int32_t* enabled);
/* all-reduce an arbitrary device float buffer on the ctx stream (tests) */
int32_t b2g_ctx_allreduce_test(b2g_ctx* ctx, float* host_inout, int64_t n);

/* ---------------------------------------------------------------- kernel-level test hooks --------- */
/* Run ONE hot-path kernel on caller-provided host tensors (NHWC, fp32 on host, rounded to bf16 on the
 * device when precision is BF16) and return the fp32 result; used by tests/ and the roofline bench.
 * kind: 0 = conv fprop, 1 = conv dgrad (= deconv fprop), 2 = conv wgrad.
 * impl: 0 = SIMT reference kernel, 1 = tensor-core kernel, 2 / 3 = skinny-layer (<= 4 image channels) SIMT / tensor-core kernels,
 * 4 = dense 1x1-geometry kernels (B2G_ERR_UNSUPPORTED if the shape has none). */
typedef struct {
  int32_t n, h, w, c;          /* conv input  (NHWC) */
  int32_t oh, ow, o;           /* conv output (NHWC) */
  int32_t kh, kw, sh, sw, ph, pw;
} b2g_conv_geom;
int32_t b2g_test_conv(b2g_ctx* ctx, int32_t kind, int32_t impl, int32_t precision, const b2g_conv_geom* g,
                      const float* x_or_dy, const float* w_or_x, float* out, int32_t iters, float* ms_per_iter);
/* The same with the epilogue the training step actually uses (impl 1, kind 0 / 1): bias, folded inference-BatchNorm scale, activation,
 * and the fused BatchNorm epilogues of kernels_tc.cu; for the pixel-shuffle deconv (impl 3, kind 1) bias, activation and the
 * activation-backward epilogue.  `kernel` returns the name of the tensor-core kernel that was dispatched, so a parity test can assert
 * that it exercised the variant the benchmark runs.  bn / max_ctas / poison / w_mn let a test pin the tile width and the grid of the
 * persistent kernel, see every element the measured launch left unwritten, and reach the dense input-gradient operand layout. */
typedef struct {
  int32_t epi;            /* 0 plain; 1 + statistics (sum, sum of squares per group and channel) of the stored outputs;
                             2 BatchNorm-backward epilogue: out = acc * act'(aux) (aux = the BatchNorm+activation output y), statistics sum out, sum out*aux2
                               (aux2 = the BatchNorm input z);
                             3 activation-backward epilogue: out = acc * act'(aux) with aux the forward output */
  int32_t act; float alpha;
  const float* bias;      /* [C_out] or NULL */
  const float* scale;     /* [C_out] or NULL: out = act(acc*scale + bias) */
  int32_t groups;         /* statistics groups (the batch split evenly, like real | fake in the D step) */
  const float* aux;       /* epi 2 / 3: the forward output whose activation derivative multiplies the result (NHWC, shape of the result) */
  const float* aux2;      /* epi 2: the BatchNorm input z (same shape) */
  double* stats;          /* out (epi 1 / 2): [groups][2][C_out] */
  char kernel[64];        /* out */
  /* Schedule controls of the persistent tensor-core conv kernel (impl 1 kind 0 / 1, and impl 3 kind 1 where noted); 0 = production. */
  int32_t bn;             /* impl 1: force the 64- or 128-column tile (B2G_ERR_UNSUPPORTED unless C_out is a multiple of it) */
  int32_t max_ctas;       /* impl 1 / impl 3 kind 1: grid = min(work items, max_ctas) instead of min(work items, SMs); may exceed the SM count */
  int32_t poison;         /* kinds 0 / 1: fill the output with 0xFF bytes (bf16 NaN) before every launch, warm-up included */
  int32_t w_mn;           /* impl 1 kind 0, 1x1 geometry: the weight operand is [C][O] (the dense input gradient's own [nOut][nIn] weight) */
} b2g_test_conv_opts;
int32_t b2g_test_conv_ex(b2g_ctx* ctx, int32_t kind, int32_t impl, int32_t precision, const b2g_conv_geom* g,
                         const float* x_or_dy, const float* w_or_x, float* out, int32_t iters, float* ms_per_iter, b2g_test_conv_opts* opts);

/* Times the HBM-bound kernels in isolation, each launch after an L2 flush (bench.py's `hbm` roofline entries): ms[0] one updater pass over
 * `net` (perturbs its parameters: bench only), ms[1] BatchNorm apply and ms[2] BatchNorm backward apply on a [rows x channels] bf16 tensor. */
int32_t b2g_test_hbm_kernels(b2g_net* net, int32_t rows, int32_t channels, int32_t iters, float* ms3);

/* One train-mode BatchNorm(+activation act) forward and backward on host tensors x, eps_out [groups*rows][C] (fp32; rounded to bf16 on the
 * device when precision is BF16), through the kernels of the training step.  path 0: the two-stage kernels (fp32 or bf16, any C);
 * 1: the 128-bit accumulator kernels (bf16, C % 8 == 0, 256 % (C/8) == 0, else B2G_ERR_UNSUPPORTED); 2: the accumulator kernels in the
 * state the fused BatchNorm-backward GEMM epilogue leaves: eps_out must already be multiplied by act'.
 * Out: y, eps_in [groups*rows][C]; g_gamma / g_beta [C] are accumulated into (untouched when want_param_grads = 0); g_mean / g_var [C] =
 * the running-statistic pseudo-gradients averaged over groups; mean / invstd [groups][C]. */
int32_t b2g_test_bn(b2g_ctx* ctx, int32_t precision, int32_t path, int32_t groups, int32_t rows, int32_t C, const float* x, const float* eps_out,
                    const float* gamma, const float* beta, const float* run_mean, const float* run_var, int32_t act, float alpha, float eps, float decay,
                    int32_t want_param_grads, float* y, float* eps_in, float* g_gamma, float* g_beta, float* g_mean, float* g_var, float* mean, float* invstd);
/* BF16 nets: the bf16 weight operand the next forward reads instead of the fp32 master, widened to fp32 (n = its element count).
 * which = 0: the straight copy of W in the internal [A][taps][B] order; 1: the packed [(py,px,c)][(dyr,dxc)][O] operand of the
 * pixel-shuffle transposed conv onto <= 4 channels (B2G_ERR_UNSUPPORTED if the layer has none). */
int32_t b2g_test_net_shadow(b2g_net* net, int32_t layer, int32_t which, float* out, int64_t n);
/* One DropoutLayer forward and backward on host tensors x, dy of rows*h*w*c elements in NHWC element order (fp32; rounded to bf16 on the
 * device when precision is BF16), through the kernels of the training step, with the mask of (seed, layer, rank, pass) as defined at
 * B2G_LAYER_DROPOUT.  Out: y, dx (same order).  Fails unless the forward advanced its pass counter from pass to pass + 1. */
int32_t b2g_test_dropout(b2g_ctx* ctx, int32_t precision, uint64_t seed, int32_t layer, int32_t rank, int64_t pass, int32_t rows, int32_t h, int32_t w,
                         int32_t c, float p, const float* x, const float* dy, float* y, float* dx);

#ifdef __cplusplus
}
#endif
#endif /* B200GAN_H */
