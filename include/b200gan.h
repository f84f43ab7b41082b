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
  B2G_LAYER_LOSS = 8,        /* LossLayer(loss): loss (b2g_loss) on the incoming pre-activations (DCGAN D-last conv) */
  B2G_LAYER_FF_TO_CNN = 9,   /* FeedForwardToCnnPreProcessor(h,w,c)                               J:200,255         */
  B2G_LAYER_CNN_TO_FF = 10,  /* CnnToFeedForwardPreProcessor (auto-inserted by setInputTypes, SURVEY.md 3.1)       */
  B2G_LAYER_DROPOUT = 11,    /* DropoutLayer.Builder(p): p = RETAIN probability in (0, 1], carried in act_alpha; no parameters */
  B2G_LAYER_SUBSAMPLING = 12,    /* SubsamplingLayer.Builder(PoolingType.AVG / SUM / PNORM).kernelSize().stride().padding().pnorm(): b2g_pooling */
  B2G_LAYER_GLOBAL_POOLING = 13, /* GlobalPoolingLayer.Builder(PoolingType).pnorm(): b2g_pooling, output [mb, C] (H = W = 1)                 */
  B2G_LAYER_CNN_LOSS = 14,       /* CnnLossLayer.Builder(LossFunction).activation(..): the loss per pixel of a [mb, C, H, W] map; no parameters  */
  B2G_LAYER_ELEMENTWISE = 15,    /* ElementWiseVertex(Op) of the spine and an earlier entry's output: b2g_elementwise_op; no parameters       */
  B2G_LAYER_MERGE = 16,          /* MergeVertex: concatenation of the two inputs along dimension 1 (channels / features); no parameters        */
  B2G_LAYER_PRELU = 17           /* PReLULayer.Builder().inputShape(..).sharedAxes(..): learned negative slopes "W" (alpha), shared-axes mask in act */
} b2g_layer_type;

/* PReLULayer (DL4J 1.0.0-beta3 org.deeplearning4j.nn.conf.layers.PReLULayer with libnd4j prelu / prelu_bp, recalled; parity unpinned like the
 * rest of the DL4J semantics).  Output shape = input shape.
 *   Parameter "W" = alpha, DL4J's weight shape: the input shape [C, H, W] ([F] for a feed-forward input, H = W = 1) with every shared axis of
 *   extent 1, flattened in 'c' order at the layer's place in the parameter vector, so get_param / set_param / get_params and a checkpoint are
 *   plain copies.  sharedAxes (DL4J's 1-based axes 1 = C, 2 = H, 3 = W) travel as a bit mask in b2g_layer_desc.act: bit 0 = C (or F), bit 1 = H,
 *   bit 2 = W; 0 = one slope per element, 6 = sharedAxes(2, 3) = one slope per channel.  inputShape, when given, in pre_c, pre_h, pre_w (a
 *   feed-forward input: pre_c = F, pre_h = pre_w = 0; all 0 = not given).  A 1 x 1 map is a feed-forward input unless inputShape is [C, 1, 1];
 *   then it is a [C, 1, 1] map, whose H and W bits are accepted and change nothing.
 *   B2G_ERR_ARG at b2g_net_create for a mask bit outside the input's rank (bit 0 only on a feed-forward input); B2G_ERR_SHAPE for an inputShape
 *   other than the inferred input.
 *   Arithmetic, in fp32 from the stored activations, each result rounded once to the activation type:
 *     y = x < 0 ? alpha*x : x;    dx = x < 0 ? alpha*dy : dy;    dalpha[k] = sum over the examples and the positions of slope k of (x < 0 ? x*dy : 0)
 *   x = +-0 is not negative (dy passes, no slope term); NaN passes.  dalpha is summed, not divided by the minibatch (the updater's division is
 *   the only one, as for W and b).
 *   Summation order of dalpha, fixed by the shape: a pass of R rows of M = H*W*C elements is cut into G row groups of rpg consecutive rows
 *   (bx = ceil(M / 2048), G0 = max(1, min(R, 64, 1024 / bx)) with integer division, rpg = ceil(R / G0), G = ceil(R / rpg); G is not monotone
 *   in R, and the partials of a net are sized for min(max_batch, 64, 1024 / bx) groups, which bounds G for every batch up to max_batch).  The partial of
 *   group g at row element j is the fp32 sum over the group's rows, ascending, from +0, of the products x*dy (rounded, no fused multiply-add) with
 *   x < 0.  Element j = (h*W + w)*C + c belongs to slope k = ((c')*aH + h')*aW + w' and position s = ((c")*sH + h")*sW + w" among the S = M / K
 *   positions sharing it, where a primed coordinate is 0 on a shared axis, a double-primed one 0 on a kept axis, aX = 1 on a shared axis (else X)
 *   and sX = X on a shared axis (else 1).  dalpha[k] is then the sum over t < G*S of partial[t] (t = g*S + s) as a reduce-list job does it: from
 *   +0 in ascending t, or, when G*S >= 64 and K <= 65536, as 32 lane sums (lane l takes t = l, l + 32, ... ascending) folded by a butterfly
 *   (xor 16, 8, 4, 2, 1).
 *   Launches: one forward and one backward per PReLU layer and pass; a trainable layer's slope gradient is one job of the backward pass's
 *   reduce-list launch (kernels_ew.cu reduce_multi_kernel), which a pass that queues no other job launches for it alone.  A FrozenLayer (or the
 *   generator step's pass through D) computes dx only.  Never fused into a BatchNorm or GEMM epilogue.
 *   Training: alpha takes the layer's updater, learning rate, schedule and gradient normalization like any parameter; l1 / l2 of
 *   b2g_regularization apply to it (the desc's l2 included; l1_bias / l2_bias have no tensor); it starts at 0 (a new PReLU is a ReLU) and
 *   b2g_net_init_weights on the named layer takes ZERO, ONES and DISTRIBUTION (the global form leaves it alone).  Not supported (documented
 *   deviations): constraints and weight noise on alpha -- the named setters return B2G_ERR_ARG. */

/* Spine-plus-skip graphs (DL4J 1.0.0-beta3 ElementWiseVertex / MergeVertex, recalled; parity unpinned like the rest of the DL4J semantics).
 * Entry i of the b2g_layer_desc array takes entry i-1's output as its input (entry 0 the net input): the spine.  ELEMENTWISE and MERGE
 * entries take a second input, the output of an earlier entry j (0 <= j < i), carried in fields these types do not otherwise use:
 *   act    ELEMENTWISE: the b2g_elementwise_op
 *   pre_h  j, the skip source
 *   pre_w  the input order: 0 = (spine, j), 1 = (j, spine) -- DL4J's addVertex("m", v, "enc2", "dec3") in either order.  Only SUBTRACT and MAX's
 *          tie rule depend on it for ELEMENTWISE; for MERGE it is the channel order of the concatenation.
 * Every entry still depends on its predecessor, so the array order is the graph's only topological order: DL4J's flattened parameter vector
 * (topological order) is the array order as for a chain, and the vertices have no parameters.
 *   ELEMENTWISE: both inputs have the same shape.  y = a + b | a - b | a * b | (a + b) * 0.5 | (a >= b ? a : b) on the inputs (a, b) in input
 *     order, in fp32, rounded once to the activation type.  Backward with e = the epsilon w.r.t. y:  ADD da = db = e;  SUBTRACT da = e,
 *     db = -e;  PRODUCT da = e*b, db = e*a;  AVERAGE da = db = e*0.5;  MAX e to the larger input, a tie to the first input (a), 0 to the other.
 *   MERGE: the inputs have the same H and W; the output has C_a + C_b channels, a's first ([N, F] vectors: the features, in DL4J's order after
 *     CNN_TO_FF).  In the NHWC layout this is a per-pixel channel concat; its backward splits the epsilon into the two channel slices.
 *   Gradient at a skip source j: each source has an fp32 buffer [max_batch][its output elements].  The backward visits entries in descending
 *   order; a vertex writes the skip input's share of its epsilon into the buffer if it is the first (highest) consumer of j and adds it (fp32)
 *   otherwise, so the order is fixed.  At the top of entry j's backward the buffer is added to the spine epsilon (fp32 sum, rounded once to
 *   the activation type) before j's own backward runs.
 *   Launches: one per vertex in the forward; one per vertex plus one per skip source in the backward.  A net without vertices launches what a
 *   chain always launched.  The fusions that assume one consumer are not taken where the consumer set is larger: a BatchNorm that is a skip
 *   source is not fused with the ActivationLayer after it, an inference-mode BatchNorm is not folded into a GEMM that is a skip source, and a
 *   GEMM's input gradient does not premultiply a BatchNorm / activation derivative of a layer that still waits for a skip share.
 *   B2G_ERR_ARG at b2g_net_create for j outside [0, i), an unknown op or an order outside {0, 1}; B2G_ERR_SHAPE for mismatched shapes;
 *   B2G_ERR_UNSUPPORTED for a skip source of type LOSS, CNN_LOSS or OUTPUT.
 *   Not provided: layers on the skip branch (projection shortcuts), vertices of more than two inputs, the net input as a vertex input, and the
 *   Subset / Scale / Shift / L2 / Stack / Preprocessor vertices. */
typedef enum {
  B2G_EW_OP_ADD = 0, B2G_EW_OP_SUBTRACT = 1, B2G_EW_OP_PRODUCT = 2, B2G_EW_OP_AVERAGE = 3, B2G_EW_OP_MAX = 4   /* ElementWiseVertex.Op order */
} b2g_elementwise_op;

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
 * A pass may hold at most 2^34 elements (max_batch * layer size; B2G_ERR_UNSUPPORTED at b2g_net_create).
 * The rest of this comment is b2g_dropout_kind: the other IDropout kinds of a DropoutLayer. */

/* The IDropout of a B2G_LAYER_DROPOUT layer (DL4J 1.0.0-beta3, recalled; parity unpinned like the rest of the DL4J semantics).  The kind is
 * carried in b2g_layer_desc.act (a DropoutLayer has no activation), its value in act_alpha:
 *   DROPOUT           retain probability p in (0, 1]      as above (B2G_LAYER_DROPOUT)
 *   GAUSSIAN_DROPOUT  rate in [0, 1)                      y = x * m, m = fmaf(s, z, 1.0f), s = sqrt(rate / (1 - rate)) in double, then fp32;
 *                                                         dx = dy * m, m drawn again from the forward's (S, r, L, P, e): no noise buffer
 *   GAUSSIAN_NOISE    stddev s >= 0, finite               y = fmaf(s, z, x);  dx = dy (no launch)
 *   ALPHA_DROPOUT     retain probability p in (0, 1]      y = fmaf(a, keep ? x : a', b);  dx = keep ? dy * a : 0;  a' = -lambda * alpha
 *                                                         (SELU's alpha = 1.6732632423543772, lambda = 1.0507009873554805), a = 1 / sqrt(p +
 *                                                         a'^2 p (1 - p)), b = -a (1 - p) a', each computed in double and rounded to fp32 once
 *   SPATIAL_DROPOUT   retain probability p in (0, 1]      Dropout's x * (1/p) or +0 with one keep bit per (row, channel) of a [rows][H][W][C] map
 * Another kind or a value outside its range is B2G_ERR_ARG at b2g_net_create; SPATIAL_DROPOUT on a 1 x 1 map (a feed-forward input) is
 * B2G_ERR_SHAPE.  Train mode only, in fp32 from the stored activation, each result rounded once to the activation type.
 * Draws: the Philox4x32-10 words of B2G_LAYER_DROPOUT with the counter word j >> 2, where j = e (the element's NHWC index in the pass) for
 * every kind except SPATIAL_DROPOUT, and j = row * C + c for it.  The Bernoulli kinds keep where x[j & 3] < floor(p * 2^32), p >= 1 keeps all.
 * The Gaussian kinds turn the four words of one counter into four normals, pair (x0, x1) into z0, z1 and pair (x2, x3) into z2, z3; element e
 * takes z[e & 3].  In fp32, with IEEE sqrtf and the library's logf / sincospif (no fast-math):
 *   u = ((x_even >> 9) + 0.5f) * 2^-23 (exact, in [2^-24, 1)),  v = (x_odd >> 8) * 2^-24 (exact),  r = sqrtf(-2 logf(u)),
 *   sincospif(2v, &s, &c),  z_even = r * c,  z_odd = r * s.
 * So |z| <= sqrt(-2 ln 2^-24), about 5.8: a truncated normal, a documented deviation (DL4J draws from its own generator).
 * Identity cases launch nothing, report their input as their activation and do not count as a masking pass for P: inference, a FrozenLayer,
 * p = 1, rate = 0 and stddev = 0.  Every other train-mode DropoutLayer of any kind is stochastic: the pass uses one P for all of them and the
 * last one's forward advances it.  Buffers: DROPOUT and ALPHA_DROPOUT keep one bit per element, SPATIAL_DROPOUT one per (row, channel),
 * GAUSSIAN_DROPOUT the P of its latest forward (one device word, written by the forward, read by the backward), GAUSSIAN_NOISE nothing.
 * Any kind, Dropout included, may take a schedule in place of its value: b2g_net_set_dropout_schedule. */
typedef enum {
  B2G_DROPOUT = 0, B2G_DROPOUT_GAUSSIAN_DROPOUT = 1, B2G_DROPOUT_GAUSSIAN_NOISE = 2, B2G_DROPOUT_ALPHA = 3, B2G_DROPOUT_SPATIAL = 4
} b2g_dropout_kind;

/* org.deeplearning4j.nn.conf.layers.PoolingType of SUBSAMPLING and GLOBAL_POOLING layers (DL4J 1.0.0-beta3, recalled; parity unpinned like the
 * rest of the DL4J semantics).  The kind is carried in b2g_layer_desc.act (pooling layers have no activation), PNORM's p in act_alpha: a whole
 * number >= 1 (DL4J's int pnorm; at most 1024).  SUBSAMPLING takes AVG, SUM and PNORM (MAX stays B2G_LAYER_MAXPOOL, unpadded); GLOBAL_POOLING
 * takes all four.  B2G_ERR_ARG at b2g_net_create for another kind or a p that is not such a number; B2G_ERR_SHAPE for a SUBSAMPLING kernel or
 * stride below 1, a padding below 0 or not smaller than the kernel, or an empty output.
 *   SUBSAMPLING (Truncate): OH = (H + 2 ph - kh) / sh + 1, likewise OW; the window of output row oy is input rows oy*sh - ph ... + kh - 1, the
 *   positions outside the input are zeros.  Per (example, output pixel, channel) the window's in-range elements are summed in fp32 in row-major
 *   window order, then
 *     AVG    y = sum / (kh*kw)       (the padding counts in the divisor)      dx += eps / (kh*kw)
 *     SUM    y = sum                                                           dx += eps
 *     PNORM  y = (sum |x|^p)^(1/p)                                             dx += eps * sign(x)|x|^(p-1) / max(y^(p-1), 1e-8)
 *   The backward gathers: each input element sums, in fixed order (filter row, then column, ascending), eps (AVG / SUM) or eps / max(y^(p-1),
 *   1e-8) (PNORM) of the windows that cover it, then divides by kh*kw (AVG) or multiplies by sign(x)|x|^(p-1) (PNORM), in fp32.
 *   GLOBAL_POOLING: per (example, channel) over the H*W pixels to [mb, C] (collapseDimensions; [mb, C, 1, 1] is the same bytes):
 *     MAX    y = the first maximum in row-major pixel order; dx = eps at that pixel, 0 elsewhere
 *     AVG    y = sum / (H*W);  dx = eps / (H*W)        SUM  y = sum;  dx = eps
 *     PNORM  y = (sum |x|^p)^(1/p);  dx = eps * sign(x)|x|^(p-1) / max(y^(p-1), 1e-8)
 *   The pixel sum is in fp32 in an order fixed by the shape: lane t of a block takes pixels t, t + r, t + 2r, ... of its pixel range, the lanes
 *   fold in lane order and, where a large map is split over blocks, the splits fold in split order (kernels_pool.cu gp_plan).
 * Powers: |x|^p and y^(p-1) are exact products for p = 1, 2 and powf otherwise; the root is sqrtf for p = 2 and powf(s, 1.0f / p) for p >= 3.
 * Every result is rounded once to the activation type.  The 1e-8 floor (SubsamplingLayer's default eps) keeps an all-zero window (after a
 * ReLU) at 0 instead of 0/0; DL4J's GlobalPoolingLayer has no floor, so its NaN on a zero map is a deliberate deviation here. */
typedef enum { B2G_POOL_MAX = 0, B2G_POOL_AVG = 1, B2G_POOL_SUM = 2, B2G_POOL_PNORM = 3 } b2g_pooling;

/* org.nd4j.linalg.activations.Activation  J:126,162,215.  Codes 0-4 as DL4J; LRELU's alpha = b2g_layer_desc.act_alpha.
 * Codes 5-16 (DL4J 1.0.0-beta3 org.nd4j.linalg.activations.impl.*, recalled; parity unpinned like the rest of the DL4J semantics).  f and f' are
 * computed in fp32 from the pre-activation z as stored (bf16 in a BF16 net: the GEMM's z is rounded once before f) with expf / expm1f / log1pf /
 * tanhf, and the result is rounded once to the activation type.  The derivative is taken from z, as IActivation.backprop(in, epsilon) takes it:
 *   ELU (5)             z >= 0 ? z : a*expm1(z)                           f' = z >= 0 ? 1 : a*e^z                    a = act_alpha (DL4J 1.0)
 *   SELU (6)            l*(z > 0 ? z : s*expm1(z))                        f' = z > 0 ? l : l*s*e^z       l = 1.0507009873554805, s = 1.6732632423543772
 *   SOFTPLUS (7)        max(z, 0) + log1p(e^-|z|)                         f' = sigmoid(z)
 *   SOFTSIGN (8)        z / (1 + |z|)                                     f' = 1 / (1 + |z|)^2
 *   HARDTANH (9)        min(1, max(-1, z))                                f' = 1 on -1 <= z <= 1, else 0
 *   HARDSIGMOID (10)    min(1, max(0, 0.2z + 0.5))                        f' = 0.2 on -2.5 <= z <= 2.5, else 0
 *   RELU6 (11)          min(max(z, 0), 6)                                 f' = 1 on 0 < z < 6, else 0
 *   SWISH (12)          z*sigmoid(z)                                      f' = s*(1 + z*(1 - s)), s = sigmoid(z)
 *   CUBE (13)           z^3                                               f' = 3z^2
 *   RATIONALTANH (14)   y = 2z/3, A = 1 + |y| + y^2 + 1.41645*y^4:  1.7159*sgn(y)*(1 - 1/A)
 *                                                                         f' = 1.7159*(2/3)*(1 + sgn(y)*(2y + 4*1.41645*y^3)) / A^2
 *   RECTIFIEDTANH (15)  max(0, tanh z)                                    f' = z > 0 ? 1 - tanh^2 z : 0
 *   THRESHOLDEDRELU (16) z > t ? z : 0                                    f' = z > t ? 1 : 0                         t = act_alpha (DL4J 1.0)
 * Softplus and Swish use the overflow-safe forms above: DL4J's literal log(1 + e^z) and e^z(z + e^z + 1)/(e^z + 1)^2 overflow to inf / NaN in
 * fp32 for large z; where those are finite the forms agree to rounding.  The Python and Java builders fill act_alpha = 1.0 for ELU and
 * ThresholdedReLU when none is given; the C-ABI takes it as given and a non-finite act_alpha with codes 5-16 is B2G_ERR_ARG.
 * Codes 0-16 are valid on CONV2D, DECONV2D, DENSE and ACTIVATION layers and on OUTPUT / LOSS layers with loss codes 2-8 (XENT / MCXENT ignore
 * act); any other code there is B2G_ERR_ARG at b2g_net_create.  A GEMM layer with a code of 5-16 keeps its pre-activation z in a buffer of its own
 * and applies f in a separate element-wise kernel; it is never fused into a GEMM or BatchNorm epilogue.
 * Not provided: RRELU (random slopes per element in train mode), SOFTMAX as a hidden activation (implied by MCXENT), GELU / MISH (later DL4J
 * versions), and PReLU as an activation code (it is a layer with parameters: B2G_LAYER_PRELU). */
typedef enum {
  B2G_ACT_IDENTITY = 0, B2G_ACT_TANH = 1, B2G_ACT_SIGMOID = 2, B2G_ACT_RELU = 3, B2G_ACT_LRELU = 4,
  B2G_ACT_ELU = 5, B2G_ACT_SELU = 6, B2G_ACT_SOFTPLUS = 7, B2G_ACT_SOFTSIGN = 8, B2G_ACT_HARDTANH = 9, B2G_ACT_HARDSIGMOID = 10,
  B2G_ACT_RELU6 = 11, B2G_ACT_SWISH = 12, B2G_ACT_CUBE = 13, B2G_ACT_RATIONALTANH = 14, B2G_ACT_RECTIFIEDTANH = 15, B2G_ACT_THRESHOLDEDRELU = 16
} b2g_activation;

/* org.nd4j.linalg.learning.config.*  J:133 (RmsProp), north_star (Adam); the others as in DL4J 1.0.0-beta3 (recalled, parity unpinned like
 * the rest of the DL4J semantics).  One update is  g /= mb -> [normalization] -> [clip] -> u = updater(g) -> u += l2*W [+ l1*sign(W)] -> theta -= u,
 * in fp32 (the regularization terms: b2g_regularization).
 * t = iteration + 1 (b2g_net_get_iteration before the update's increment); lr = b2g_layer_desc.lr or the layer's schedule value (b2g_lr_schedule);
 * the bias-correction factors are computed once per updater block in fp32.  Desc fields: beta1, beta2, eps as named, except where noted.
 *   SGD (0)        u = lr*g
 *   RMSPROP (1)    beta1 = rmsDecay.  s0 (init eps): s0 = b1*s0 + (1-b1)*g^2;  u = lr*g / (sqrt(s0) + eps)
 *   ADAM (2)       s0 = m, s1 = v: m = b1*m + (1-b1)*g;  v = b2*v + (1-b2)*g^2;  u = alpha_t*m / (sqrt(v) + eps),  alpha_t = lr*sqrt(1-b2^t)/(1-b1^t)
 *   NOOP (3)       u = g
 *   NESTEROVS (4)  new Nesterovs(lr = 0.1, momentum = 0.9); beta1 = momentum.  s0 = v (init 0):  vPrev = v;  v = mu*v - lr*g;
 *                  u = mu*vPrev - (1+mu)*v
 *   ADAGRAD (5)    new AdaGrad(lr = 0.1, eps = 1e-6).  s0 = h (init eps):  h = h + g^2;  u = lr*g / (sqrt(h) + eps)
 *   ADAMAX (6)     new AdaMax(lr = 1e-3, b1 = 0.9, b2 = 0.999, eps = 1e-8).  s0 = m, s1 = u_inf:  m = b1*m + (1-b1)*g;
 *                  u_inf = max(b2*u_inf, |g|) + 1e-32 (stored back);  u = lr/(1-b1^t) * m / u_inf  (eps is not used)
 *   NADAM (7)      new Nadam(lr = 1e-3, b1 = 0.9, b2 = 0.999, eps = 1e-8).  s0 = m, s1 = v:  m, v as Adam;
 *                  u = lr/(1-b1^t) * (b1*m + (1-b1)*g) / (sqrt(v) + eps)  (v is not bias-corrected)
 *   AMSGRAD (8)    new AMSGrad(lr = 1e-3, b1 = 0.9, b2 = 0.999, eps = 1e-8).  s0 = m, s1 = v, s2 = vhat:  m, v as Adam;  vhat = max(vhat, v);
 *                  u = alpha_t*m / (sqrt(vhat) + eps), alpha_t as Adam
 *   ADADELTA (9)   new AdaDelta(rho = 0.95, eps = 1e-6); beta1 = rho, lr is ignored (the layer has no learning rate).  s0 = msg, s1 = msdx:
 *                  msg = rho*msg + (1-rho)*g^2;  u = sqrt(msdx + eps) / sqrt(msg + eps) * g;  msdx = rho*msdx + (1-rho)*u^2
 * A layer with lr 0 takes a zero updater step (DL4J's fallback from alpha_t == 0 to eps is not restated).  BatchNorm mean/var always update
 * through NOOP.  Any other value is B2G_ERR_ARG at b2g_net_create. */
typedef enum {
  B2G_UPD_SGD = 0, B2G_UPD_RMSPROP = 1, B2G_UPD_ADAM = 2, B2G_UPD_NOOP = 3, B2G_UPD_NESTEROVS = 4, B2G_UPD_ADAGRAD = 5, B2G_UPD_ADAMAX = 6,
  B2G_UPD_NADAM = 7, B2G_UPD_AMSGRAD = 8, B2G_UPD_ADADELTA = 9
} b2g_updater;

typedef enum { B2G_PREC_FP32 = 0, B2G_PREC_BF16 = 1 } b2g_precision;
/* org.nd4j.linalg.lossfunctions.LossFunctions.LossFunction (DL4J 1.0.0-beta3 org.nd4j.linalg.lossfunctions.impl.*, recalled; parity unpinned like
 * the rest of the DL4J semantics).  The loss of OUTPUT and LOSS layers (b2g_layer_desc.loss); any other value is B2G_ERR_ARG at b2g_net_create.
 *   XENT (0)    LossBinaryXENT with the implied sigmoid, nOut = 1 (clipEps = b2g_net_config.xent_clip_eps); b2g_layer_desc.act is ignored
 *   MCXENT (1)  LossMCXENT with the implied softmax, OUTPUT layers only (B2G_ERR_UNSUPPORTED on a LOSS layer); act is ignored
 * Codes 2-8 act like ILossFunction.computeGradient(labels, preOutput, activationFn): the layer's pre-activation z, a = act(z) in fp32 with the
 * layer's b2g_activation act (act_alpha = LeakyReLU's alpha), and dL/dz = dL/da * act'(a), the derivative taken from the output a.  Per example,
 * over the outputs j < nOut (y = labels):
 *   MSE (2)             score sum (a-y)^2 / nOut              dL/da = 2(a-y) / nOut
 *   L1 (3)              score sum |a-y|                       dL/da = sign(a-y), sign(0) = 0
 *   L2 (4)              score sum (a-y)^2                     dL/da = 2(a-y)
 *   MAE (5)             score sum |a-y| / nOut                dL/da = sign(a-y) / nOut       (LossMAE = LossFunction.MEAN_ABSOLUTE_ERROR)
 *   HINGE (6)           score sum max(0, 1 - y a)             dL/da = -y where 1 - y a > 0 (strictly), else 0     (labels +-1)
 *   SQUARED_HINGE (7)   score sum max(0, 1 - y a)^2           dL/da = -2y max(0, 1 - y a)
 *   WASSERSTEIN (8)     score sum y a / nOut                  dL/da = y / nOut
 * The loss of a pass (or of a group of the GAN step) is the sum of its examples' scores, summed in double in an order fixed by the shape (the same
 * bits on every run) and rounded to fp32 once; score = that sum / minibatch + the l2 term.  OUTPUT layers take any nOut; a LOSS layer needs a
 * feed-forward input (H = W = 1) or one element per example (else B2G_ERR_UNSUPPORTED).  b2g_net_output returns a = act(z).
 * With an activation of codes 5-16 (b2g_activation) a = f(z) is formed by its own kernel and rounded to the activation type, the loss takes a
 * with the identity, and dL/dz = dL/da * f'(z) with the derivative taken from z.
 *
 * Per-output weights and label masks (b2g_net_set_loss_weights, b2g_net_fit_masked, b2g_gan_set_label_masks; DL4J 1.0.0-beta3 ILossFunction
 * weights and DataSet labels masks, recalled).  Row r is an example (a pixel of a CnnLossLayer), column j an output (a channel of a
 * CnnLossLayer), w_j the weight (1 without weights), m_rj the mask (1 without one; a [rows, 1] mask gives every column of its row one value):
 *   XENT, codes 2-8   the row's score terms become w_j m_rj l(a_rj, y_rj) and dz_rj = w_j m_rj (dz_rj unweighted)
 *   MCXENT            score -m_r sum_j w_j y_rj log clamp(p_rj);  dz_rj = m_r (p_rj sum_k w_k y_rk - w_j y_rj) with weights (LossMCXENT's
 *                     weighted softmax gradient), m_r (p_rj - y_rj) without
 *   The score stays the sum divided by the minibatch (not by the mask count); MSE, MAE and WASSERSTEIN still divide by nOut / C.  Masks are
 *   multiplicative fp32 values taken as given, like labels: [N, 1] or [N, nOut] on OUTPUT / LOSS layers, NCHW [N, 1, H, W] or [N, C, H, W] on a
 *   CnnLossLayer.  Weights are nOut (C) finite floats.  b2g_net_output ignores both.
 *   Refused: weights on HINGE, SQUARED_HINGE or WASSERSTEIN (DL4J has no weights constructor for them) and a per-output mask with MCXENT
 *   (LossMCXENT: "Per output masking for MCXENT + softmax: not supported"): B2G_ERR_UNSUPPORTED; a weight count or mask width other than
 *   those above: B2G_ERR_SHAPE; a non-finite weight, or weights on a net whose last layer is not OUTPUT / LOSS / CNN_LOSS: B2G_ERR_ARG.
 *   Arithmetic (no product below is fused into an add): s = w_j * m_rj in fp32 (w first; what is absent is 1); the score term enters the
 *   loss's double sum as (double)l * (double)s (the loss kernel's double l times (double)s) and dz is the unweighted fp32 dz times s, in the
 *   unweighted kernels' slicing and summation order.  MCXENT forms sy = sum_k w_k y_rk in fp32 in class order (each product rounded, then
 *   added); dz = m_r * (p * sy - w_j y_j) with p * sy rounded before the subtraction; its term is (double)(m_r * w_j y_rj) *
 *   log((double)clamp(p)), subtracted from the double sum.  A net with neither
 *   weights nor a mask launches the unweighted instantiations; a weighted or masked loss is the same single launch.  All-ones weights and
 *   mask give the unweighted bits (for MCXENT with one-hot labels).
 *
 * B2G_LAYER_CNN_LOSS (DL4J 1.0.0-beta3 CnnLossLayer, recalled; parity unpinned like the rest of the DL4J semantics).  No parameters.
 *   Rows and columns: the input is the layer below's [N, C, H, W]; the rows are its N*H*W pixels and the columns its C channels (DL4J's
 *   reshape4dTo2d, which in the engine's NHWC layout is the buffer as it is).  A 1x1 map is accepted and then equals a LOSS layer on the same
 *   values.
 *   XENT (0): a sigmoid on every element, any C; the per-element formulas and xent_clip_eps are those of XENT above; act is ignored.
 *   MCXENT (1): a softmax over the C channels of each pixel; score -sum_c y log(clamp(p, 1e-10, 1 - 1e-10)) (the log in double), dz = p - y;
 *   act is ignored.
 *   Codes 2-8: on a = act(z) with activation codes 0-16, exactly as on LOSS layers, with nOut = C (MSE, MAE and WASSERSTEIN divide by the
 *   channel count, not by C*H*W).
 *   Score = (sum of the row scores over all N*H*W rows) / N + the l2 term: CnnLossLayer.computeScore divides by the minibatch, not by the
 *   pixel count.  dz is not divided; the updater's division by the minibatch is the only one.  The sums are taken in double in an order
 *   fixed by the shape (kernels_cnnloss.cu for XENT / MCXENT, loss_kernel for codes 2-8) and rounded to fp32 once.
 *   Labels: [N, C, H, W] fp32 in DL4J's NCHW order, b2g_net_output_size elements per example (fit, computeGradientAndScore and the GAN step).
 *   b2g_net_output returns the activated map in NCHW: the sigmoid (XENT), the per-pixel softmax (MCXENT) or act(z).
 *   Not supported: the NHWC CNN2DFormat of later DL4J versions.
 *   The adversarial step (b2g_gan_create) takes a discriminator ending in CNN_LOSS with XENT or codes 2-8 (a PatchGAN critic: one logit and
 *   one label per patch); MCXENT there is B2G_ERR_UNSUPPORTED. */
typedef enum {
  B2G_LOSS_XENT = 0, B2G_LOSS_MCXENT = 1, B2G_LOSS_MSE = 2, B2G_LOSS_L1 = 3, B2G_LOSS_L2 = 4, B2G_LOSS_MAE = 5, B2G_LOSS_HINGE = 6,
  B2G_LOSS_SQUARED_HINGE = 7, B2G_LOSS_WASSERSTEIN = 8
} b2g_loss;

/* One layer of a spine-plus-skip ComputationGraph (every graph in the reference is a chain, J:118-310; vertices: B2G_LAYER_ELEMENTWISE). */
typedef struct {
  int32_t type;                 /* b2g_layer_type */
  char name[B2G_NAME_LEN];      /* DL4J vertex name, e.g. "dis_conv2d_layer_2" */
  int32_t n_in, n_out;          /* channels / features (n_in may be 0 = infer, like setInputTypes) */
  int32_t k_h, k_w, s_h, s_w, p_h, p_w;   /* conv / deconv / pool geometry; upsample factor in k_h */
  int32_t has_bias;             /* hasBias(true) default */
  int32_t act;                  /* b2g_activation; b2g_pooling on SUBSAMPLING / GLOBAL_POOLING layers; b2g_dropout_kind on DROPOUT layers */
  float act_alpha;              /* ActivationLReLU alpha: DL4J default 0.01, DCGAN passes 0.2; ELU alpha / ThresholdedReLU theta (DL4J 1.0);
                                   DropoutLayer value (b2g_dropout_kind); PNORM pooling's p */
  int32_t updater;              /* b2g_updater; "frozen" in the reference = RMSPROP with lr 0 (J:84) */
  float lr, beta1, beta2, eps;  /* RmsProp: beta1 = rmsDecay (ctor order lr, rmsDecay, epsilon; J:133 passes 1e-8, 1e-8) */
  float l2;                     /* .l2(1e-4) (J:125): weights only, applied AFTER the updater, not lr-scaled (b2g_net_set_regularization) */
  float bn_decay, bn_eps;       /* BatchNormalization defaults 0.9 / 1e-5 */
  int32_t pre_h, pre_w, pre_c;  /* FF_TO_CNN target shape */
  int32_t loss;                 /* OUTPUT / LOSS layer: b2g_loss (0 = LossFunction.XENT + sigmoid J:159-163, 1 = MCXENT + softmax J:357-362, 2-8 on act) */
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
 * updater-state arena and every activation buffer; Xavier-normal weights, BN gamma=1 beta=0 mean=0 var=1 (b2g_net_init_weights redraws
 * W and b with any other WeightInit). */
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
/* updater state (ModelSerializer updaterState.bin payload): [state0 | state1] each in params order, plus | state2 (AMSGrad's vhat) on a net
 * with an AMSGrad layer; b2g_net_updater_state_size gives the element count (2 or 3 x numParams).  Slots per kind: b2g_updater. */
int32_t b2g_net_updater_state_size(b2g_net* net, int64_t* out);
int32_t b2g_net_get_updater_state(b2g_net* net, float* host, int64_t n);
int32_t b2g_net_set_updater_state(b2g_net* net, const float* host, int64_t n);
/* ComputationGraph.output(x)[0] (J:170,420): inference mode (BN uses mean/var). x: [batch, in] NCHW fp32 host;
 * out: [batch, out] NCHW fp32 host.  train!=0 gives the train-mode forward (batch statistics). */
int32_t b2g_net_output(b2g_net* net, const float* x, int32_t batch, int32_t train, float* out);
/* Activations of one layer from the most recent forward (parity tests): NCHW fp32. */
int32_t b2g_net_get_activation(b2g_net* net, int32_t layer, int32_t batch, float* host);
/* computeGradientAndScore(): train-mode forward, the last layer's loss (b2g_loss) vs labels y, backprop.
 * score = sum(loss)/batch + 0.5*l2*||W||^2 (+ the other terms of b2g_regularization); gradients stay on device (b2g_net_get_gradients).
 * Labels y are [batch, nOut] (nOut = 1 for XENT; one-hot rows for MCXENT; targets for codes 2-8). */
int32_t b2g_net_compute_gradient_and_score(b2g_net* net, const float* x, const float* y, int32_t batch, float* score);
/* epsilon w.r.t. the network input from the last backward (NCHW fp32; what the stacked gan graph feeds the generator). */
int32_t b2g_net_get_input_gradient(b2g_net* net, int32_t batch, float* host);
/* ComputationGraph.fit(DataSet) (J:426,471 via SparkComputationGraph): one minibatch =
 * computeGradientAndScore + [gradient all-reduce if a communicator is attached] + updater + params.subi. */
int32_t b2g_net_fit(b2g_net* net, const float* x, const float* y, int32_t batch, float* score);
/* fit / computeGradientAndScore of a DataSet with a labels mask (DataSet(features, labels, null, labelsMask)); semantics at b2g_loss.
 * mask: fp32 host, [batch, mask_width] on OUTPUT / LOSS layers (mask_width 1 = per example, nOut = per output), NCHW [batch, mask_width, H, W]
 * on a CnnLossLayer (mask_width 1 = per pixel, C = per output); null = no mask (mask_width ignored). */
int32_t b2g_net_fit_masked(b2g_net* net, const float* x, const float* y, int32_t batch, float* score, const float* mask, int32_t mask_width);
int32_t b2g_net_compute_gradient_and_score_masked(b2g_net* net, const float* x, const float* y, int32_t batch, float* score, const float* mask,
                                                  int32_t mask_width);
/* new LossMCXENT(weights), new LossBinaryXENT(weights), new LossMSE(weights), ...: the per-output weights of the net's loss layer (semantics at
 * b2g_loss), kept in device memory and used by every later fit, computeGradientAndScore and GAN step.  layer: null = the net's loss layer, or
 * its name; w: n = nOut (C on a CnnLossLayer) finite floats, null = clear (with layer null a no-op on a net that has none, whatever its last
 * layer).  Setting or clearing re-captures a captured GAN step. */
int32_t b2g_net_set_loss_weights(b2g_net* net, const char* layer, const float* w, int32_t n);
/* The columns of the net's loss: nOut (the outputs per example), or the channels C of a CnnLossLayer.  A mask of width 1 holds
 * b2g_net_output_size / columns values per example, one of width = columns b2g_net_output_size. */
int32_t b2g_net_loss_columns(b2g_net* net, int32_t* cols);
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
/* Weight constraints (DL4J 1.0.0-beta3 org.deeplearning4j.nn.conf.constraint.*, Layer.Builder.constrainWeights / constrainBias /
 * constrainAllParameters, recalled; parity unpinned like the rest of the DL4J semantics; the Keras constraints of the same names agree).
 * A constraint acts on one parameter tensor in DL4J's shape: conv W [nOut, nIn, kH, kW], deconv W [nIn, nOut, kH, kW], dense / output W
 * [nIn, nOut], and b, gamma, beta, mean, var [1, n].  Bit d of dims_mask is dimension d of that shape (conv / deconv W: d < 4, others d < 2).
 * The L2 norm is taken over the set dimensions once per index of the remaining ones (a group); dims_mask 0 reduces over everything, as
 * norm2() does.  norm = sqrt of the sum of squares in double over the fp32 values, in an order fixed by the shape (kernels_constraint.cu);
 * the multiplier m is computed in double, rounded to fp32 once, and each element of the group becomes the fp32 product w * m.  eps = 1e-6
 * (BaseConstraint.DEFAULT_EPSILON):
 *   MAX_NORM (0)       m = clip(norm, 0, max_norm) / (norm + eps)     (a group under the bound still shrinks by norm / (norm + eps))
 *   MIN_MAX_NORM (1)   m = (rate * clip(norm, min_norm, max_norm) + (1 - rate) * norm) / (norm + eps)
 *   UNIT_NORM (2)      m = 1 / norm; an all-zero group is left as it is (DL4J divides by 0 and gives NaN: a deliberate deviation, as the
 *                      PNORM floor at b2g_pooling)
 *   NON_NEGATIVE (3)   w = w < 0 ? +0 : w, element-wise; -0.0 and NaN stay (replaceWhere(.., 0, lessThan(0))); dims_mask is not used
 * Fields a kind does not use are ignored (rate is read by MIN_MAX_NORM only).
 * When: after theta -= u of every update the net's updater runs (b2g_net_fit, the D update and the G update of b2g_gan_step, local fits in
 * parameter-averaging mode) -- DL4J's applyConstraints after the step -- and in b2g_net_apply_constraints (Model.applyConstraints).  Never after
 * b2g_net_average_parameters, set_param(s) or compute_gradient_and_score.  The G step leaves D untouched, constraints included.  A FrozenLayer
 * (b2g_layer_desc.frozen) is never constrained; a layer with lr 0 is.  The bf16 weight operands of a BF16 net are rewritten with the fp32
 * result, so they stay bf16(master).
 * Order: a tensor's constraints run in list order; the callers put a layer's constrainAllParameters list first, then constrainWeights (W of
 * CONV2D, DECONV2D, DENSE, OUTPUT; nothing on BATCHNORM), then constrainBias (b where the layer has one), each in the order given.  A layer
 * whose own lists reach none of its parameters (none given, or only constrainBias on a BatchNorm) takes the global builder's lists, as DL4J's
 * NeuralNetConfiguration.Builder fills them in.
 * Launches per update: round r is the r-th constraint of every constrained tensor.  A tensor whose innermost stored axis (conv W: nIn and
 * deconv W: nOut, both DL4J dimension 1; dense W: nIn, dimension 0; a vector: n, dimension 1) is reduced and whose groups hold at most 4096
 * elements is one-pass, as is NonNegative; every other tensor (larger groups, or the innermost axis kept:
 * strided groups such as a deconv W per output unit, dims {0, 2, 3}) takes two launches.  A round launches 1 kernel if it has a one-pass
 * tensor, plus 2 if it has a two-launch tensor.  A net without constraints launches what it always launched. */
typedef enum {
  B2G_CONSTRAINT_MAX_NORM = 0, B2G_CONSTRAINT_MIN_MAX_NORM = 1, B2G_CONSTRAINT_UNIT_NORM = 2, B2G_CONSTRAINT_NON_NEGATIVE = 3
} b2g_constraint_kind;
typedef struct {
  int32_t kind;                   /* b2g_constraint_kind */
  int32_t dims_mask;              /* bit d = DL4J dimension d of the parameter */
  double max_norm, min_norm, rate;
} b2g_constraint;
/* Replaces the constraint list of one tensor (param in {"W","b","gamma","beta","mean","var"}); n = 0 clears it.  Takes effect at the next update
 * (a captured GAN step is re-captured).  B2G_ERR_ARG for an unknown kind, layer or parameter, a dims bit outside the parameter's rank, a bound
 * that is not finite and >= 0, min_norm > max_norm, a rate outside [0, 1], or more than 4 constraints. */
int32_t b2g_net_set_constraints(b2g_net* net, const char* layer, const char* param, const b2g_constraint* list, int32_t n);
/* Model.applyConstraints(iteration, epoch): every constraint once, now, as after an update.  Sync point. */
int32_t b2g_net_apply_constraints(b2g_net* net);
/* Learning-rate schedules (DL4J 1.0.0-beta3 org.nd4j.linalg.schedule.ISchedule; new Adam(ISchedule), ComputationGraph.setLearningRate(ISchedule)).
 * A layer with a schedule updates with lr_i = (float)value(i) in place of b2g_layer_desc.lr; l2 is unchanged (applied after the updater, not
 * lr-scaled).  value(i) is computed in double and rounded to fp32 once:
 *   EXPONENTIAL (1): initial * pow(gamma, i)
 *   INVERSE     (2): initial / pow(1 + gamma * i, power)
 *   SIGMOID     (3): initial / (1 + exp(-gamma * (i - step)))                       (step = DL4J's stepSize)
 *   STEP        (4): initial * pow(decay_rate, floor(i / step))                     (step a double > 0)
 *   MAP         (5): map_values[j] for the largest map_keys[j] <= i                  (the keys strictly increase and contain 0)
 * i is the net's iteration counter before this update's increment (b2g_net_get_iteration: 0 on the first update, Adam's t - 1) for
 * type ITERATION, or the net's epoch word (b2g_net_get_epoch) for type EPOCH.  Both are read from device memory by the updater kernel, so a
 * replayed CUDA graph uses the current values.  Sgd: u = lr_i * g.  RmsProp: u = lr_i * g / (sqrt(s) + eps).  Adam:
 * alpha_t = lr_i * sqrt(1 - b2^t) / (1 - b1^t) in fp32 as without a schedule; likewise lr_i replaces lr in every b2g_updater formula (AdaDelta
 * has none and takes no schedule).  A schedule applies wherever the net's updater runs
 * (b2g_net_fit, the D and G updates of b2g_gan_step, parameter-averaging mode) and adds no kernel launch.  PolySchedule is not supported. */
typedef enum {
  B2G_SCHED_NONE = 0, B2G_SCHED_EXPONENTIAL = 1, B2G_SCHED_INVERSE = 2, B2G_SCHED_SIGMOID = 3, B2G_SCHED_STEP = 4, B2G_SCHED_MAP = 5
} b2g_schedule_kind;
typedef enum { B2G_SCHED_ITERATION = 0, B2G_SCHED_EPOCH = 1 } b2g_schedule_type;   /* org.nd4j.linalg.schedule.ScheduleType */
typedef struct {
  int32_t kind, type;               /* b2g_schedule_kind, b2g_schedule_type */
  double initial, gamma, power, step, decay_rate;   /* the fields a kind does not use are ignored but must be finite */
  int32_t n_map;                    /* MAP: entries of map_keys / map_values (copied during the call) */
  const int32_t* map_keys;
  const double* map_values;
} b2g_lr_schedule;
/* ComputationGraph.setLearningRate(ISchedule) (layer NULL: every non-frozen layer whose updater has a learning rate, others are skipped) and
 * setLearningRate(String, ISchedule) (layer named).  s NULL or kind NONE: back to the layer's constant lr.  Takes effect at the next update.
 * B2G_ERR_ARG for an unknown kind or type, a non-finite parameter or map value, step <= 0 (STEP), gamma < 0 (INVERSE), a map that is empty,
 * whose keys do not strictly increase or that has no key 0, and a named layer that does not exist, is frozen or has no learning rate (no
 * parameters, NoOp or AdaDelta). */
int32_t b2g_net_set_lr_schedule(b2g_net* net, const char* layer, const b2g_lr_schedule* s);
/* ComputationGraph.getLearningRate(String): the fp32 learning rate the layer's next update will use (before Adam's bias correction), computed
 * on the device by the function the updater kernel calls.  Sync point. */
int32_t b2g_net_get_learning_rate(b2g_net* net, const char* layer, float* out);
/* IDropout with an ISchedule in place of its constant (b2g_dropout_kind): layer NULL = every non-frozen DropoutLayer, else the named one
 * (B2G_ERR_ARG if it is not a DropoutLayer); s NULL or kind NONE: back to the constant from b2g_net_create.  The schedule checks of
 * b2g_net_set_lr_schedule apply.  Each train-mode forward evaluates it on the device, by the function the updater calls, at the owning net's
 * iteration counter (before the update's increment) or epoch word -- in b2g_gan_step the generator step's pass through D at the generator's --
 * and clamps the value into its kind's range (p to [2^-32, 1], rate to [0, 1 - 2^-24], stddev to >= 0; a documented deviation), then derives
 * the kernels' constants from it; its backward uses the forward's value.  A scheduled layer is stochastic whatever its value.  Bumps the
 * settings generation (a captured GAN step is re-captured); a replay reads the counters from device memory. */
int32_t b2g_net_set_dropout_schedule(b2g_net* net, const char* layer, const b2g_lr_schedule* s);
/* The value (p, rate or stddev) the named DropoutLayer's next train-mode forward uses, clamped, computed on the device.  Sync point. */
int32_t b2g_net_get_dropout_value(b2g_net* net, const char* layer, float* out);

/* Weight noise (DL4J 1.0.0-beta3 org.deeplearning4j.nn.conf.weightnoise: Layer.Builder.weightNoise / NeuralNetConfiguration.Builder.weightNoise
 * with DropConnect or WeightNoise, recalled; parity unpinned like the rest of the DL4J semantics).
 * Which layers: CONV2D, DECONV2D, DENSE and OUTPUT; W always, b only with apply_to_bias.  BatchNorm parameters are never perturbed.
 * When: in the train-mode passes of a non-frozen layer, exactly the passes in which the net's DropoutLayers draw (b2g_net_fit,
 * b2g_net_compute_gradient_and_score, b2g_net_output with train = 1, the GAN step's real|fake pass of D and its generator pass through D, the
 * generator's train-mode pass).  A FrozenLayer draws nothing; a layer with lr 0 does draw.  Inference passes use the clean parameters (DL4J's
 * `train && isWeight || (applyToBias && isBias)` would also perturb biases at inference: a documented deviation).
 * One pass, one draw: the forward and the input gradient of a pass use the same W' and b'.  The weight and bias gradients are computed from x
 * and dy as without noise and applied to the clean W and b (straight through; DL4J does not multiply dW by the mask).  The l2 score, the
 * updater, the constraints and b2g_net_get_param see the clean parameters.
 * Draws: element j of a noisy tensor takes word x[j & 3] of Philox4x32-10(ctr = {j >> 2, lo32(P), hi32(P), L | r << 16}, key = {lo32(S), hi32(S)})
 * with S, r and P of B2G_LAYER_DROPOUT and L the GEMM layer's own index (no DropoutLayer mask uses a GEMM layer's index).  For W, j is the
 * element's index in the fp32 master as stored (the internal [A][taps][B] order of b2g_test_net_shadow); bias element k takes
 * j = 4 * ceil(n_W / 4) + k.  Each result is computed in fp32 and rounded once to the operand type (fp32, or bf16 in BF16 nets):
 *   DROPCONNECT(p)   keep = p >= 1 || x[j & 3] < floor(p * 2^32);  W' = keep ? w : +0.  Not rescaled by 1/p (DL4J applies the DropOut op, not
 *                    DropOutInverted).  p in (0, 1]; p_schedule (may be NULL) replaces it with an ISchedule evaluated on the device at each
 *                    train-mode pass, at the owning net's iteration counter or epoch word (in b2g_gan_step's generator pass through D at the
 *                    generator's, as for DropoutLayer schedules), clamped to [2^-32, 1].
 *   WEIGHTNOISE      n = fmaf(b, z, a) for NORMAL(mean a, std b >= 0), z = z[j & 3] of the Box-Muller normals of b2g_dropout_kind (truncated
 *                    at |z| <= 5.8); n = fmaf(b - a, u, a) for UNIFORM(lower a, upper b >= a), u = (x[j & 3] >> 8) * 2^-24.
 *                    W' = additive ? w + n : w * n.
 * Pass counter: a train-mode pass with at least one noisy layer issues one launch at its top, before any layer, for every noisy tensor of the
 * net.  It reads P; when the pass has no stochastic DropoutLayer its last block advances P, otherwise the last DropoutLayer does as before, so
 * adding weight noise changes no DropoutLayer mask.  DROPCONNECT with a constant p = 1 is the identity: no launch, no pass counted; a scheduled
 * DROPCONNECT draws whatever its value.  One GPU runs the reference's two worker minibatches of the D step (real | fake) as one pass: they share
 * one W', as they share DropoutLayer masks.  Buffers: the noisy operands of a layer are allocated when it first gets weight noise. */
typedef enum { B2G_WEIGHT_NOISE_NONE = 0, B2G_WEIGHT_NOISE_DROPCONNECT = 1, B2G_WEIGHT_NOISE_WEIGHTNOISE = 2 } b2g_weight_noise_kind;
typedef enum { B2G_DIST_NORMAL = 0, B2G_DIST_UNIFORM = 1 } b2g_distribution_kind;    /* NormalDistribution(mean, std), UniformDistribution(lower, upper) */
/* The further b2g_distribution_kind values, for weight initialization (b2g_weight_init; weight noise takes NORMAL and UNIFORM only):
 * TruncatedNormalDistribution(mean, std), LogNormalDistribution(mean, std), BinomialDistribution(nTrials, p), ConstantDistribution(value),
 * OrthogonalDistribution(gain) (refused).  GaussianDistribution is NORMAL under another name. */
enum { B2G_DIST_TRUNCATED_NORMAL = 2, B2G_DIST_LOG_NORMAL = 3, B2G_DIST_BINOMIAL = 4, B2G_DIST_CONSTANT = 5, B2G_DIST_ORTHOGONAL = 6 };
typedef struct {
  int32_t kind;                     /* b2g_weight_noise_kind */
  int32_t apply_to_bias;            /* DropConnect's applyToBiases / WeightNoise's applyToBias */
  float p;                          /* DROPCONNECT: retain probability in (0, 1] */
  const b2g_lr_schedule* p_schedule;   /* DROPCONNECT: an ISchedule in place of p (NULL: none; copied during the call) */
  int32_t dist;                     /* WEIGHTNOISE: b2g_distribution_kind */
  float a, b;                       /* WEIGHTNOISE: NORMAL mean, std; UNIFORM lower, upper */
  int32_t additive;                 /* WEIGHTNOISE: W' = w + n (1) or w * n (0) */
} b2g_weight_noise;
/* Layer.Builder.weightNoise (layer named) or NeuralNetConfiguration.Builder.weightNoise (layer NULL: every non-frozen CONV2D, DECONV2D, DENSE
 * and OUTPUT layer).  wn NULL or kind NONE clears it.  Bumps the settings generation (a captured GAN step is re-captured).  B2G_ERR_ARG for an
 * unknown kind or distribution, p outside (0, 1], std < 0, upper < lower, a non-finite value, a schedule b2g_net_set_dropout_schedule refuses,
 * or a named layer that does not exist or has no W. */
int32_t b2g_net_set_weight_noise(b2g_net* net, const char* layer, const b2g_weight_noise* wn);

/* Weight initialization (DL4J 1.0.0-beta3 WeightInitUtil.initWeights with Layer.Builder / NeuralNetConfiguration.Builder .weightInit, .dist and
 * .biasInit, recalled; parity unpinned like the rest of the DL4J semantics).  A named PRELU layer takes ZERO, ONES and DISTRIBUTION for its slopes,
 * element j = the slope's index in DL4J's order (the other schemes need fans: B2G_ERR_ARG); the global form leaves PReLU layers alone.  The
 * scheme numbers are DL4J's WeightInit ordinals.  Each scheme
 * draws W from a distribution of the layer's fans:
 *    0 DISTRIBUTION     the b2g_weight_init's own dist(a, b)          11 RELU                  N(0, sqrt(2 / fanIn))
 *    1 ZERO             0                                            12 RELU_UNIFORM          U(+-sqrt(6 / fanIn))
 *    2 ONES             1                                            13 IDENTITY              the identity (square DENSE / OUTPUT only)
 *    3 SIGMOID_UNIFORM  U(+-4 sqrt(6 / (fanIn + fanOut)))             14 LECUN_UNIFORM         U(+-3 / sqrt(fanIn))
 *    4 NORMAL           N(0, 1 / sqrt(fanIn))                         15 VAR_SCALING_NORMAL_FAN_IN    T(0, sqrt(1 / fanIn))
 *    5 LECUN_NORMAL     N(0, 1 / sqrt(fanIn))                         16 VAR_SCALING_NORMAL_FAN_OUT   T(0, sqrt(1 / fanOut))
 *    6 UNIFORM          U(+-1 / sqrt(fanIn))                          17 VAR_SCALING_NORMAL_FAN_AVG   T(0, sqrt(2 / (fanIn + fanOut)))
 *    7 XAVIER           N(0, sqrt(2 / (fanIn + fanOut)))              18 VAR_SCALING_UNIFORM_FAN_IN   U(+-3 / sqrt(fanIn))
 *    8 XAVIER_UNIFORM   U(+-sqrt(6) / sqrt(fanIn + fanOut))           19 VAR_SCALING_UNIFORM_FAN_OUT  U(+-3 / sqrt(fanOut))
 *    9 XAVIER_FAN_IN    N(0, 1 / sqrt(fanIn))                         20 VAR_SCALING_UNIFORM_FAN_AVG  U(+-3 / sqrt((fanIn + fanOut) / 2))
 *   10 XAVIER_LEGACY    N(0, 1 / sqrt(nIn + nOut))
 * N(mean, std) is NORMAL, U(+-r) UNIFORM(-r, r), T(mean, std) TRUNCATED_NORMAL below.  Fans come from the layer desc, whatever geometry the
 * engine computes the layer with (the 1x1-map deconv, the whole-input conv): CONV2D and DECONV2D fanIn = nIn kH kW, fanOut = nOut kH kW /
 * (sH sW); DENSE and OUTPUT fanIn = nIn, fanOut = nOut.  Each std or bound is computed in double and rounded to fp32 once.
 * Draws: S = b2g_net_config.seed (0: 666), L = the layer's index in the desc array, j = the element's index in DL4J's view order of W (what
 * b2g_net_get_param(layer, "W") returns, so the draw does not depend on the internal layout).  Round k of element j uses word x[j & 3] of
 * Philox4x32-10(ctr = {j >> 2, k, 0, L | 0x80000000}, key = {lo32(S), hi32(S)}); the top bit keeps these streams apart from every
 * DropoutLayer and weight-noise draw.  No rank input: every data-parallel replica draws the same W.  Values are fp32:
 *   NORMAL(mean a, std b >= 0)            fmaf(b, z, a), z = z[j & 3] of round 0's Box-Muller normals of b2g_dropout_kind (|z| <= 5.8)
 *   UNIFORM(lower a, upper b >= a)        fmaf(b - a, u, a) (b - a in fp32), u = (x >> 8) 2^-24 of round 0
 *   TRUNCATED_NORMAL(mean a, std b >= 0)  fmaf(b, z, a) with z of the first round k < 16 whose |z| <= 2; none: round 15's z clamped to +-2
 *   LOG_NORMAL(mean a, std b >= 0)        expf(fmaf(b, z, a)), z as for NORMAL
 *   BINOMIAL(nTrials a, p b)              the count over rounds t < nTrials of x_t < floor(p 2^32) (p = 1: nTrials); nTrials a whole number
 *                                         in [0, 65536], p in [0, 1]
 *   CONSTANT(value a)                     a, no draw (ZERO, ONES and IDENTITY draw nothing either)
 *   ORTHOGONAL                            refused with B2G_ERR_UNSUPPORTED: it needs an SVD, and DL4J's bits could not be matched anyway.
 * b2g_net_create's own draw is unchanged: Xavier-normal weights from a host generator and zero biases.  An explicit XAVIER through
 * b2g_net_init_weights draws the same distribution from the stream above, so it gives other bits. */
typedef enum {
  B2G_WI_DISTRIBUTION = 0, B2G_WI_ZERO = 1, B2G_WI_ONES = 2, B2G_WI_SIGMOID_UNIFORM = 3, B2G_WI_NORMAL = 4, B2G_WI_LECUN_NORMAL = 5,
  B2G_WI_UNIFORM = 6, B2G_WI_XAVIER = 7, B2G_WI_XAVIER_UNIFORM = 8, B2G_WI_XAVIER_FAN_IN = 9, B2G_WI_XAVIER_LEGACY = 10, B2G_WI_RELU = 11,
  B2G_WI_RELU_UNIFORM = 12, B2G_WI_IDENTITY = 13, B2G_WI_LECUN_UNIFORM = 14, B2G_WI_VAR_SCALING_NORMAL_FAN_IN = 15,
  B2G_WI_VAR_SCALING_NORMAL_FAN_OUT = 16, B2G_WI_VAR_SCALING_NORMAL_FAN_AVG = 17, B2G_WI_VAR_SCALING_UNIFORM_FAN_IN = 18,
  B2G_WI_VAR_SCALING_UNIFORM_FAN_OUT = 19, B2G_WI_VAR_SCALING_UNIFORM_FAN_AVG = 20
} b2g_weight_init_scheme;
typedef struct {
  int32_t scheme;       /* b2g_weight_init_scheme */
  int32_t dist;         /* DISTRIBUTION: a b2g_distribution_kind, B2G_DIST_NORMAL .. B2G_DIST_ORTHOGONAL (the typedef's two and the enum after it) */
  float a, b;           /* DISTRIBUTION: NORMAL / TRUNCATED_NORMAL / LOG_NORMAL mean, std; UNIFORM lower, upper; BINOMIAL nTrials, p; CONSTANT value */
  float bias_init;      /* biasInit: every element of b */
} b2g_weight_init;
/* DL4J's per-layer initialization at init(): redraws W as above and sets b = bias_init, now.  layer named: Layer.Builder's weightInit / dist /
 * biasInit; layer NULL: every CONV2D, DECONV2D, DENSE and OUTPUT layer (the global builder's).  Nothing else changes: BatchNorm parameters,
 * other layers, the updater state, the iteration counter, the dropout pass counter and the epoch word stay as they are.  BF16 nets get the
 * layer's bf16 operand copy (and its packed pixel-shuffle operand) refreshed.  Call it right after b2g_net_create, as DL4J initializes at
 * init(); a captured GAN step reads the new weights at its next replay.  Every target is checked before anything is written: a failed call
 * leaves the net unchanged.  Sync point.
 * B2G_ERR_ARG: an unknown scheme or distribution; DISTRIBUTION with a non-finite or out-of-range parameter (std < 0, upper < lower, p outside
 * [0, 1], nTrials not a whole number in [0, 65536]); a non-finite bias_init; a named layer that does not exist or has no W.
 * B2G_ERR_SHAPE: IDENTITY on a CONV2D or DECONV2D layer, or on a DENSE / OUTPUT layer with nIn != nOut (DL4J throws).
 * B2G_ERR_UNSUPPORTED: DISTRIBUTION with ORTHOGONAL. */
int32_t b2g_net_init_weights(b2g_net* net, const char* layer, const b2g_weight_init* wi);

/* Regularization (DL4J 1.0.0-beta3 Layer.Builder / NeuralNetConfiguration.Builder .l1, .l2, .l1Bias, .l2Bias, resolved per parameter by
 * getL1ByParam / getL2ByParam, recalled; parity unpinned like the rest of the DL4J semantics).
 * Which tensors: on CONV2D, DECONV2D, DENSE and OUTPUT layers l1 and l2 apply to W, l1_bias and l2_bias to b; on PRELU layers l1 and l2 apply to
 * the slopes W.  BatchNorm parameters are never
 * regularized (beta3's BatchNormalization returns 0 for every parameter).  A FrozenLayer takes no term, in the update or in the score; a layer
 * with lr 0 still decays.
 * Update (UpdaterBlock.postApply): after the updater, with the coefficients as set (no schedule, not lr-scaled; the normalization of
 * b2g_net_set_gradient_normalization and grad_clip never see the term):
 *   u = fmaf(l2, theta, u);  then  u = u + l1 * sign(theta),  sign(+0) = sign(-0) = 0;  theta -= u
 * (l2_bias / l1_bias on b), in the updater's one pass, wherever the net's updater runs (b2g_net_fit, the D and G updates of b2g_gan_step,
 * local fits in parameter-averaging mode).  BF16 nets get the bf16 weight operands from the same pass, as always.
 * Score (calcL2 / calcL1): score = sum(loss) / minibatch + (float)(L2 + L1), where over the layers
 *   L2 = sum of 0.5 * l2 * ||W||^2 + 0.5 * l2_bias * ||b||^2        L1 = sum of l1 * ||W||_1 + l1_bias * ||b||_1
 * each norm summed in double over the fp32 master values (never the weight-noise operands) in an order fixed by the shape, and multiplied by
 * the fp32 coefficient (0.5f * l2 for the squares).  A term whose coefficients are all 0 launches nothing: a net with l2 only launches what it
 * launched before and scores the same bits.
 * b2g_layer_desc.l2 is the initial l2 of W; every other coefficient starts at 0. */
typedef struct { float l1, l2, l1_bias, l2_bias; } b2g_regularization;
/* Layer.Builder.l1 / l2 / l1Bias / l2Bias (layer named) or NeuralNetConfiguration.Builder's (layer NULL: every non-frozen CONV2D, DECONV2D,
 * DENSE, OUTPUT and PRELU layer).  Replaces all four coefficients of the layer (the desc's l2 too).  Takes effect at the next update, also in a replayed
 * CUDA graph of the GAN step (the updater reads the coefficients from device memory).  B2G_ERR_ARG for a value that is not finite and >= 0
 * (DL4J silently ignores a value <= 0: refusing negatives is a deliberate deviation), or a named layer that does not exist or has no W. */
int32_t b2g_net_set_regularization(b2g_net* net, const char* layer, const b2g_regularization* r);
/* The four coefficients of a named CONV2D, DECONV2D, DENSE, OUTPUT or PRELU layer (B2G_ERR_ARG for any other name). */
int32_t b2g_net_get_regularization(b2g_net* net, const char* layer, b2g_regularization* out);
/* ComputationGraph.calcL1(true) and calcL2(true): L1 and L2 of the score above, now, in double.  Either pointer may be NULL.  Sync point. */
int32_t b2g_net_calc_regularization(b2g_net* net, double* l1, double* l2);
/* ComputationGraph.getEpochCount / setEpochCount: the 64-bit device word EPOCH schedules read, 0 at b2g_net_create.  The host sets it, nothing
 * increments it; a new value takes effect at the next update, also in a replayed CUDA graph.  Sync points.  B2G_ERR_ARG for epoch < 0. */
int32_t b2g_net_get_epoch(b2g_net* net, int64_t* out);
int32_t b2g_net_set_epoch(b2g_net* net, int64_t epoch);
/* BF16 nets: how many GEMM-shaped operations ran on the SIMT kernels instead of the tensor-core kernels since creation (skinny layers by design, or a
 * shape the tensor-core kernels do not tile).  north_star: no silent fallback -- bench.py prints it per step. */
int32_t b2g_net_simt_gemm_calls(b2g_net* net, uint64_t* out);

/* ---------------------------------------------------------------- the fused GAN step -------------- */
/* The adversarial iteration J:408-471 with dis / gan / gen sharing storage (the 28 setParam copies J:429-510
 * become aliasing): x_fake = G.output(z_d); D update on (x_real,y_real)+(x_fake,y_fake); G update through D on
 * (z_g, y_gen).  See oracle/dl4j_oracle.py::gan_step for the exact arithmetic.
 * The discriminator ends in one output per example with loss XENT or one of codes 2-8 (b2g_loss; MCXENT is B2G_ERR_UNSUPPORTED); the caller's
 * labels pick the objective: least-squares GAN 1 / 0 / 1 with MSE, hinge +1 / -1 / +1, Wasserstein the caller's sign convention. */
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
/* Label masks of the discriminator's loss for every later b2g_gan_step / b2g_gan_step_resident (semantics at b2g_loss): m_real / m_fake for the
 * D update's two halves, m_gen for the G update through D, each [batch, mask_width(, H, W)] fp32 host laid out like b2g_net_fit_masked's mask,
 * copied to the device here.  A step with another batch is B2G_ERR_SHAPE.  All three null clears.  New contents reach a replayed graph
 * without re-capture; turning masks on or off, or changing the width, re-captures. */
int32_t b2g_gan_set_label_masks(b2g_gan* gan, const float* m_real, const float* m_fake, const float* m_gen, int32_t mask_width, int32_t batch);
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
 * activation-backward epilogue; for the skinny-layer conv forward (impl 3, kind 0) bias and activation.  `kernel` returns the name of the tensor-core kernel that was dispatched, so a parity test can assert
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
  /* Schedule controls of the persistent tensor-core conv kernel (impl 1 kind 0 / 1, and impl 3 kind 0 / 1 where noted); 0 = production. */
  int32_t bn;             /* impl 1: force the 64- or 128-column tile (B2G_ERR_UNSUPPORTED unless C_out is a multiple of it) */
  int32_t max_ctas;       /* impl 1 / impl 3 kind 1: grid = min(work items, max_ctas) instead of min(work items, SMs); may exceed the SM count.
                             impl 3 kind 0: the CTA target of the skinny-layer conv, tiles_per_cta = ceil(tiles / max_ctas) instead of
                             ceil(tiles / (8 x SMs)) */
  int32_t poison;         /* kinds 0 / 1: fill the output with 0xFF bytes (bf16 NaN) before every launch, warm-up included; kind 2 impl 1 / 3:
                             dw, db and the split-K partials with fp32 NaN */
  int32_t w_mn;           /* impl 1 kind 0, 1x1 geometry: the weight operand is [C][O] (the dense input gradient's own [nOut][nIn] weight) */
  int32_t per_tap;        /* impl 1: load the activations one box per tap also where the 4x4 s2 p1 slab path applies */
  int32_t slab;           /* out: 1 when the launch loaded its activations as slabs shared by two taps */
  /* kind 2, impl 1 / impl 3: queue the split-K reduction into a list and sum it with ONE reduce-list launch afterwards, as a backward pass
   * does, instead of reducing right after the wgrad kernel */
  int32_t defer;
  float* db;              /* kind 2, impl 3, C < 4: out [O], the bias gradient (column sums of dy) the edge wgrad kernel produces beside dw; NULL: not asked */
  /* The SIMT (impl 0), skinny-layer (impl 2) and dense (impl 4) kernels take bias / act / alpha wherever their production wrapper does:
   * impl 0 kind 0 / 1 (also scale), impl 2 kind 0 / 1, impl 4 kind 0 and kind 1 on the short-reduction kernel; never epi != 0.  poison
   * applies to them for kinds 0 / 1 / 2 (kind 2: the fp32 dw is filled with 0xFF bytes, fp32 NaN).  `kernel` names the kernel they ran. */
  int32_t param_offset;   /* impl 0 / 2 / 4: the fp32 weight operand (kinds 0 / 1; FP32 only -- the bf16 operand is a 64-element aligned copy) and the
                             fp32 weight gradient (kind 2) start this many elements past a 256-byte aligned address, as a layer's W and dW do in the
                             flattened parameter and gradient vectors.  Kind 2 impl 1 / 3: dw and db, in the immediate and the deferred reduction */
  int32_t splits;         /* out, impl 0 / 2 / 4: the number of split-K partial sums the kernel reduced (1 where it has no split).
                             in / out, kind 2 impl 1 / 3: in, force the split count (0 = production): tc_wgrad_kernel's grid.x, any value >= 1
                             (splits past the last K-block are empty), or tc_edge_wgrad_kernel's CTA target (tiles_per_cta = ceil(tiles / splits));
                             out, the count launched */
} b2g_test_conv_opts;
/* impl 5: the few-output conv kernels of BF16 nets (a k x k conv, KH*KW > 1, KH, KW <= 7, stride 1-2, 0 <= pad < kernel, from C % 8 == 0
 * channels onto O <= 4 on a map wider than one pixel; B2G_ERR_UNSUPPORTED otherwise): bias / act / poison as impl 2 takes them; kind 2 runs the
 * weight gradient's split sums as one reduce-list launch, takes splits (forced count, splits past the last pixel are empty), param_offset and
 * db (the column sums of dy, as the training step forms the bias gradient). */
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
/* Cross-replica (sync) BatchNorm on one device: what `replicas` ranks of a data-parallel step run on the 128-bit accumulator kernels (path 1
 * or 2 of b2g_test_bn, bf16, the same channel rule).  x, eps_out are [replicas][groups][rows][C]: replica r's rows, as rank r holds them.
 * Each replica fills its own zeroed accumulators from its own rows (k_bn_stats_acc); the replicas' words are summed as uint64 modulo 2^64,
 * as an ncclUint64 sum all-reduce leaves them; every replica then applies the sum with replicas = R (k_bn_apply_acc), and the backward runs
 * the same way (k_bn_bwd_stats_acc, the word sum, k_bn_bwd_apply_acc).  Out, per replica: y, eps_in [R][groups][rows][C]; g_gamma / g_beta
 * [R][C], each replica's row accumulated into from the shared initial value [C] (the (global sum) / R the gradient all-reduce sums back);
 * g_mean / g_var [R][C]; mean / invstd [R][groups][C].  replicas = 1 runs exactly b2g_test_bn's launches. */
typedef struct {
  int32_t path;           /* 1: backward statistics from k_bn_bwd_stats_acc; 2: as the fused BatchNorm-backward epilogue leaves them */
  int32_t replicas;       /* R >= 1 */
  int32_t groups, rows, C;                /* rows per replica and group */
  int32_t act; float alpha, eps, decay;
  int32_t want_param_grads;
} b2g_test_bn_opts;
int32_t b2g_test_bn_ex(b2g_ctx* ctx, const b2g_test_bn_opts* opts, const float* x, const float* eps_out, const float* gamma, const float* beta,
                       const float* run_mean, const float* run_var, const float* g_gamma0, const float* g_beta0, float* y, float* eps_in,
                       float* g_gamma, float* g_beta, float* g_mean, float* g_var, float* mean, float* invstd);
/* BF16 nets: the bf16 weight operand the next forward reads instead of the fp32 master, widened to fp32 (n = its element count).
 * which = 0: the straight copy of W in the internal [A][taps][B] order; 1: the packed [(py,px,c)][(dyr,dxc)][O] operand of the
 * pixel-shuffle transposed conv onto <= 4 channels (B2G_ERR_UNSUPPORTED if the layer has none). */
int32_t b2g_test_net_shadow(b2g_net* net, int32_t layer, int32_t which, float* out, int64_t n);
/* The noisy operands the latest train-mode pass of a weight-noise layer drew (b2g_weight_noise), widened to fp32 (n = the element count).
 * which = 0: W' in the internal [A][taps][B] order (the fp32 copy in FP32 nets, the bf16 straight copy in BF16 nets); 1: the packed
 * pixel-shuffle W' (BF16 nets, layers that have that operand); 2: b' (apply_to_bias).  B2G_ERR_UNSUPPORTED if the layer drew nothing. */
int32_t b2g_test_net_noisy_operand(b2g_net* net, int32_t layer, int32_t which, float* out, int64_t n);
/* One DropoutLayer forward and backward on host tensors x, dy of rows*h*w*c elements in NHWC element order (fp32; rounded to bf16 on the
 * device when precision is BF16), through the kernels of the training step, with the mask of (seed, layer, rank, pass) as defined at
 * B2G_LAYER_DROPOUT.  Out: y, dx (same order).  Fails unless the forward advanced its pass counter from pass to pass + 1. */
int32_t b2g_test_dropout(b2g_ctx* ctx, int32_t precision, uint64_t seed, int32_t layer, int32_t rank, int64_t pass, int32_t rows, int32_t h, int32_t w,
                         int32_t c, float p, const float* x, const float* dy, float* y, float* dx);
/* The same for a DropoutLayer of any b2g_dropout_kind with its value (p, rate or stddev; the ranges of b2g_dropout_kind, else B2G_ERR_ARG).
 * An identity case (p = 1, rate = 0, stddev = 0) launches nothing and leaves the pass counter alone: y = x, dx = dy.  Otherwise it fails unless
 * the forward advanced the pass counter from pass to pass + 1. */
int32_t b2g_test_dropout_kind(b2g_ctx* ctx, int32_t precision, int32_t kind, uint64_t seed, int32_t layer, int32_t rank, int64_t pass, int32_t rows,
                              int32_t h, int32_t w, int32_t c, float value, const float* x, const float* dy, float* y, float* dx);

/* One reduction, loss or element-wise kernel of the training step on host tensors, through its production launch wrapper (tests).
 * T tensors are fp32 on the host, rounded to bf16 on the device when precision is BF16 and widened back on the way out; the others are fp32.
 *   REDUCE_SPLITS  in0 src [splits*stride] fp32, in1 dst's initial value [n]          -> out0 dst [n]            (n, splits, stride, accumulate)
 *   REDUCE_MULTI   in0 one fp32 buffer [n]; the jobs index into it                    -> out0 the buffer [n]     (jobs, n_jobs)
 *   COLSUM         in0 x [rows][cols] T, in1 out's initial value [cols]               -> out0 [cols]             (rows, cols, accumulate)
 *   XENT           in0 logits [groups][rows] T, in1 labels fp32                       -> out0 dz T, out1 loss per group [groups]   (clip_eps)
 *   SOFTMAX_XENT   in0 logits [rows][cols] T, in1 labels fp32 or NULL (inference: no labels, dz or loss passed to the kernel)
 *                                                                                     -> out0 dz T, out1 loss [1], out2 probabilities T
 *   ACT_FWD        in0 x [n] T                                                        -> out0 act(x) T           (act, alpha)
 *   ACT_BWD        in0 a = the forward output [n] T, in1 eps_out [n] T                -> out0 eps_in T           (act, alpha, in_place)
 *   MAXPOOL        in0 x [N][H][W][C] T, in1 eps_out [N][OH][OW][C] T (OH = (H-KH)/SH + 1, OW likewise)
 *                                                                                     -> out0 y T, out1 eps_in T, out2 argmax (as float)
 *   UPSAMPLE       in0 x [N][H][W][C] T, in1 eps_out [N][H*KH][W*KH][C] T (factor KH) -> out0 y T, out1 eps_in T
 *   SUMSQ          in0 p [n] fp32, segments seg_off / seg_len / seg_coef              -> sumsq
 *   LOSS           in0 logits [groups][rows][cols] T, in1 labels fp32                 -> out0 dz T, out1 loss per group [groups]
 *                                                                                        (loss = b2g_loss 2-8, cols = nOut, act, alpha)
 *   ACT_EXT_FWD    in0 z [n] T                                                        -> out0 f(z) T             (act = b2g_activation 5-16, alpha)
 *   ACT_EXT_BWD    in0 z [n] T, in1 eps_out [n] T                                     -> out0 eps_out * f'(z) T, computed in place in eps_out's
 *                                                                                        buffer as the backward pass calls it (act 5-16, alpha)
 *   CNN_XENT       in0 logits [groups][rows][cols] T (NHWC pixels x channels), in1 labels fp32
 *                                                                                     -> out0 dz T, out1 loss per group [groups]   (clip_eps)
 *   CNN_SOFTMAX_XENT  in0 logits [groups][rows][cols] T, in1 labels fp32 or NULL (inference: probabilities only)
 *                                                                                     -> out0 dz T, out1 loss per group [groups], out2 probabilities T
 * The skip-connection vertices (B2G_LAYER_ELEMENTWISE; act = b2g_elementwise_op, groups = the input order 0 / 1, accumulate = add to the
 * accumulator instead of writing it):
 *   VERTEX_FWD     in0 spine [n] T, in1 skip [n] T                                    -> out0 y [n] T
 *   VERTEX_BWD     in0 [spine | skip] [2n] T (the forward inputs), in1 [eps [n] T | acc [n] fp32] (acc: the accumulator's initial value, read
 *                  when accumulate)                                                   -> out0 the spine's epsilon T (eps's buffer, in place),
 *                                                                                        out1 acc [n] fp32
 *   MERGE_FWD      in0 spine [rows][cols] T, in1 skip [rows][C] T                     -> out0 y [rows][cols + C] T (input order: groups)
 *   MERGE_BWD      in0 eps [rows][cols + C] T, in1 acc's initial value [rows][C] fp32 (when accumulate)
 *                                                                                     -> out0 the spine's slice [rows][cols] T, out1 acc [rows][C]
 *   SKIP_ADD       in0 eps [n] T, in1 acc [n] fp32                                    -> out0 eps + acc T (in place)
 * PReLU (B2G_LAYER_PRELU; act = the shared-axes mask, the map N x H x W x C, K = the slope count):
 *   PRELU_FWD      in0 [x [n] T | alpha [K] fp32]                                     -> out0 y T
 *   PRELU_BWD      in0 [x [n] T | alpha [K] fp32], in1 dy [n] T                       -> out0 dx T (dy's buffer, in place; NULL: not written),
 *                                                                                        out1 dalpha [K] (NULL: no slope gradient), summed by
 *                                                                                        one reduce-list launch
 * Layout conversion and casts (the map N x C x HW, HW = H * W):
 *   NCHW_TO_NHWC   in0 x [N][C][HW] fp32                                              -> out0 [N][HW][C] T
 *   NHWC_TO_NCHW   in0 x [N][HW][C] T                                                 -> out0 [N][C][HW] fp32
 *   PERMUTE        in0 x T, groups = 1: [N][C][HW] -> [N][HW][C], 0: the reverse      -> out0 T
 *   CAST_BF16      in0 x [n] fp32 (any precision)                                     -> out0 the bf16 result, widened on the host, out1 the
 *                                                                                        same widened on the device (nhwc_to_nchw_f32 at
 *                                                                                        1 x 1 x n, the bf16 gradient payload's round trip)
 * Every output buffer not asked for may be NULL. */
typedef enum {
  B2G_EW_REDUCE_SPLITS = 0, B2G_EW_REDUCE_MULTI = 1, B2G_EW_COLSUM = 2, B2G_EW_XENT = 3, B2G_EW_SOFTMAX_XENT = 4,
  B2G_EW_ACT_FWD = 5, B2G_EW_ACT_BWD = 6, B2G_EW_MAXPOOL = 7, B2G_EW_UPSAMPLE = 8, B2G_EW_SUMSQ = 9, B2G_EW_LOSS = 10,
  B2G_EW_ACT_EXT_FWD = 11, B2G_EW_ACT_EXT_BWD = 12, B2G_EW_CNN_XENT = 13, B2G_EW_CNN_SOFTMAX_XENT = 14,
  B2G_EW_VERTEX_FWD = 15, B2G_EW_VERTEX_BWD = 16, B2G_EW_MERGE_FWD = 17, B2G_EW_MERGE_BWD = 18, B2G_EW_SKIP_ADD = 19,
  B2G_EW_PRELU_FWD = 20, B2G_EW_PRELU_BWD = 21,
  B2G_EW_NCHW_TO_NHWC = 22, B2G_EW_NHWC_TO_NCHW = 23, B2G_EW_PERMUTE = 24, B2G_EW_CAST_BF16 = 25
} b2g_ew_op;
typedef struct {          /* one split-K sum of a reduce list: dst[i] = sum_s src[s*stride + i], i < n, all offsets in elements of in0 */
  int64_t n, stride, src_off, dst_off;
  int32_t splits;
  int32_t wide;           /* out: 1 when the list runs this job one warp per output, 0 when one thread per 4 outputs */
} b2g_ew_reduce_job;
typedef struct {
  int32_t op;             /* b2g_ew_op */
  int64_t n;              /* REDUCE_SPLITS outputs, REDUCE_MULTI buffer length, ACT_* / SUMSQ / CAST_BF16 elements */
  int32_t rows, cols;     /* COLSUM rows x channels; XENT rows per group; SOFTMAX_XENT rows x classes; CNN_* pixels per group x channels */
  int32_t groups;         /* XENT, LOSS, CNN_*; PERMUTE: 1 = to NHWC */
  int32_t splits; int64_t stride;       /* REDUCE_SPLITS */
  int32_t N, H, W, C, KH, KW, SH, SW;  /* MAXPOOL input and window; UPSAMPLE input and factor KH; layout ops: the map */
  int32_t act; float alpha;             /* ACT_*: b2g activation */
  float clip_eps;                       /* XENT: 0 = BCE with logits */
  int32_t offset;         /* every device operand starts this many elements past a 256-byte aligned address (reaches the misaligned fallbacks) */
  int32_t in_place;       /* ACT_BWD: eps_in is eps_out's buffer, as the backward pass calls it */
  int32_t accumulate;     /* REDUCE_SPLITS / COLSUM: add to the initial destination in1 */
  int32_t poison;         /* fill every output with NaN before the launch: an element the kernel leaves unwritten reads back as NaN */
  int32_t n_jobs; b2g_ew_reduce_job* jobs;                              /* REDUCE_MULTI: at most 24 */
  int32_t n_seg; const int64_t* seg_off; const int64_t* seg_len; const float* seg_coef;   /* SUMSQ */
  double sumsq;           /* out: SUMSQ's result */
  char kernel[64];        /* out: the kernel each wrapper call dispatched, comma-separated in call order (MAXPOOL / UPSAMPLE: forward, backward);
                             COLSUM names its first stage, the final stage is the same kernel on every path */
  int32_t loss;           /* LOSS: b2g_loss 2-8 */
} b2g_test_ew_opts;
int32_t b2g_test_ew(b2g_ctx* ctx, int32_t precision, b2g_test_ew_opts* opts, const float* in0, const float* in1, float* out0, float* out1, float* out2);

/* One pooling layer's forward and backward kernels (kernels_pool.cu) through their production wrappers on host tensors, as b2g_test_ew runs the
 * other element-wise kernels (T tensors fp32 on the host, rounded to bf16 on the device when precision is BF16; offset and poison as there):
 *   POOL2D       in0 x [N][H][W][C] T, in1 eps_out [N][OH][OW][C] T (b2g_pooling geometry with KH, KW, SH, SW, PH, PW; pool = AVG / SUM / PNORM)
 *                                                                          -> out0 y T, out1 eps_in T (the backward reads the forward's y)
 *   GLOBAL_POOL  in0 x [N][H][W][C] T, in1 eps_out [N][C] T (pool = any)  -> out0 y [N][C] T, out1 eps_in T, out2 MAX's pixel index (as float;
 *                                                                             -1 for the other kinds)
 * Every output buffer not asked for may be NULL. */
typedef enum { B2G_TEST_POOL2D = 0, B2G_TEST_GLOBAL_POOL = 1 } b2g_test_pool_op;
typedef struct {
  int32_t op;             /* b2g_test_pool_op */
  int32_t pool;           /* b2g_pooling */
  float pnorm;            /* PNORM: p */
  int32_t N, H, W, C, KH, KW, SH, SW, PH, PW;
  int32_t offset;         /* every device operand starts this many elements past a 256-byte aligned address (reaches the per-element path) */
  int32_t poison;         /* fill every output with NaN before the launch: an element the kernel leaves unwritten reads back as NaN */
  char kernel[64];        /* out: forward, backward kernel */
  int32_t splits;         /* out, GLOBAL_POOL: the number of blocks each example's pixel range was split over (1: no split) */
} b2g_test_pool_opts;
int32_t b2g_test_pool(b2g_ctx* ctx, int32_t precision, b2g_test_pool_opts* opts, const float* in0, const float* in1, float* out0, float* out1, float* out2);

/* The weighted / masked instantiations of the five loss kernels (semantics and order at b2g_loss) through their production wrappers on host
 * tensors (z rounded to bf16 on the device when precision is BF16; offset and poison as b2g_test_ew's):
 *   XENT               xent_kernel: z, y, dz [groups][rows] (cols = 1)
 *   SOFTMAX_XENT       softmax_xent_kernel: z, y, dz [rows][cols] (groups = 1)
 *   CODES              loss_kernel: z, y, dz [groups][rows][cols], loss b2g_loss 2-8 on act (b2g_activation 0-4, alpha)
 *   CNN_XENT           cnn_xent_kernel: z, y, dz [groups][rows][cols] (NHWC pixels x channels)
 *   CNN_SOFTMAX_XENT   cnn_softmax_xent_kernel: as CNN_XENT
 * w: [cols] or NULL; mask: [groups * rows][mask_width] or NULL (mask_width 1 or cols); out dz (T, widened to fp32) and loss_sums [groups].
 * The weighted / masked instantiation runs even with neither. */
typedef enum { B2G_TEST_LOSS_XENT = 0, B2G_TEST_LOSS_SOFTMAX_XENT = 1, B2G_TEST_LOSS_CODES = 2, B2G_TEST_LOSS_CNN_XENT = 3,
               B2G_TEST_LOSS_CNN_SOFTMAX_XENT = 4 } b2g_test_loss_kernel;
typedef struct {
  int32_t kernel;         /* b2g_test_loss_kernel */
  int32_t rows, cols, groups;
  int32_t loss, act; float alpha;       /* CODES */
  float clip_eps;                       /* XENT, CNN_XENT: 0 = BCE with logits */
  int32_t mask_width;     /* with a mask: 1 or cols */
  int32_t offset;         /* every device operand starts this many elements past a 256-byte aligned address (reaches the misaligned paths) */
  int32_t poison;         /* fill dz and the loss sums with NaN before the launch */
  char kernel_name[64];   /* out: the kernel the wrapper dispatched */
} b2g_test_loss_opts;
int32_t b2g_test_loss(b2g_ctx* ctx, int32_t precision, b2g_test_loss_opts* opts, const float* z, const float* y, const float* w, const float* mask,
                      float* dz, float* loss_sums);

#ifdef __cplusplus
}
#endif
#endif /* B200GAN_H */
