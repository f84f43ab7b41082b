"""CPU oracle: a NumPy restatement of the DL4J 1.0.0-beta3 arithmetic on the GAN training-step path.

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only ``tests/``, ``__graft_entry__.smoke()`` and the
``cpu_baseline`` / ``--impl reference`` legs of ``bench.py`` may import it.  The shipped path
(``gan_deeplearning4j_b200``) never routes through this module and fails loudly without its CUDA
library.

PARITY UNPINNED.  The reference repository (hamaadshah/gan_deeplearning4j @ 1fc05d6) holds no tests,
golden vectors or saved numeric outputs, and its arithmetic lives in un-vendored Maven dependencies
(``org.deeplearning4j:deeplearning4j-core:1.0.0-beta3``, ``org.nd4j:nd4j-native-platform:1.0.0-beta3``,
``org.deeplearning4j:dl4j-spark_2.11:1.0.0-beta3_spark_1`` -- Java/pom.xml:13-14,99-113) that cannot
run here (no JVM).  This file restates the *published* DL4J-beta3 algorithms, anchored on the reference's
own call sites; it is pinned only by self-consistency checks (finite differences with DL4J's own
GradientCheckUtil tolerances, an independent torch.autograd cross-check, hand-computed known-answer
cases) in ``tests/``.  Points of medium confidence are isolated behind flags (see ``Quirks``).

Reference call sites restated here (J = Java/src/main/java/org/deeplearning4j/dl4jGANComputerVision.java):
  * ConvolutionLayer      J:135-140,145-150,203-209,212-219   -> ``Conv2D``  (im2col + GEMM, as nd4j-native)
  * Deconvolution2D       (north_star; DL4J ``Deconvolution2DLayer``)         -> ``Deconv2D``
  * Upsampling2D          J:201-202,210-211                     -> ``Upsample2D``
  * BatchNormalization    J:132-134,186-188,197-199             -> ``BatchNorm``
  * SubsamplingLayer MAX  J:141-144,151-154                     -> ``MaxPool``
  * DenseLayer            J:155-158,189-196                     -> ``Dense``
  * OutputLayer XENT      J:159-163,303-308                     -> ``Output`` / ``LossLayer``
  * Activation.*          J:126,162,215                         -> ``act_forward`` / ``act_backward``
  * RmsProp/Adam, clip, l2  J:123-125,133...                    -> ``Net.apply_update``
  * fit / output loop     J:408-471                             -> ``Net.fit``, ``Net.output``, ``gan_iteration_reference``,
                                                                   ``gan_step`` (the aliased G+D step the CUDA path runs)
  * parameter averaging   J:325-333, Python/gan.ipynb:177-187   -> ``parameter_average``

DL4J features the library offers beyond the reference's call sites, restated here from DL4J 1.0.0-beta3 (formulas at the named enum in
include/b200gan.h):
  * activations of b2g_activation codes 5-16       -> ``forward`` / ``derivative`` (reached through ``act_forward`` / ``act_backward``)
  * losses of b2g_loss codes 2-8                   -> ``score_and_grad`` (``Output`` / ``LossLayer`` with a loss other than XENT)
  * SubsamplingLayer AVG / SUM / PNORM, GlobalPoolingLayer (b2g_pooling)  -> ``Subsampling`` / ``GlobalPooling``
  * DropoutLayer (B2G_LAYER_DROPOUT; b2g_dropout_kind: Dropout, GaussianDropout, GaussianNoise, AlphaDropout, SpatialDropout; scheduled
    values; the draws are the library's Philox draws)  -> ``Dropout``, ``dropout_mask``, ``dropout_normals``, ``spatial_mask``,
                                                          ``Net.set_dropout_schedule``
  * weight noise (b2g_weight_noise: DropConnect, WeightNoise)  -> ``noisy_operands``, ``Net.set_weight_noise``
  * weight initialization (b2g_weight_init)        -> ``resolve``, ``weights``, ``init_layer``
  * l1, l2, l1Bias, l2Bias (b2g_regularization)    -> ``Net.layer_regularization``, ``Net.reg_coefs``, ``Net.calc_l1`` / ``calc_l2``
  * PReLULayer (B2G_LAYER_PRELU)                   -> ``PReLU``
  * per-output loss weights and labels masks (b2g_loss)  -> ``rows_score_and_grad``, ``Net.set_loss_weights``, the ``mask`` of
                                                            ``Net.fit`` / ``compute_gradient_and_score`` and ``gan_step``'s three
  * the updaters of b2g_updater                    -> ``UpdaterCfg``, ``init_state``, ``update``
  * L2 gradient normalization                      -> ``Net.set_gradient_normalization``, ``normalize``
  * learning-rate schedules (ISchedule)            -> ``Net.set_lr_schedule``, ``value``, ``lr_at``
  * CnnLossLayer (B2G_LAYER_CNN_LOSS)              -> ``CnnLossLayer``
  * ElementWiseVertex / MergeVertex (b2g_elementwise_op) -> ``ElementWiseVertex`` / ``MergeVertex``, the skip edges of ``Net``
  * weight constraints (b2g_constraint)            -> ``constraint_multiplier``, ``apply_constraint``, ``constraints_by_param``,
                                                      ``Net.set_constraints`` / ``apply_constraints``
``net_from_specs`` builds a Net from the layer specs the CUDA engine consumes.

Layouts follow DL4J: activations NCHW, conv W [nOut,nIn,kH,kW] 'c' order flattened as [b | W],
deconv W [nIn,nOut,kH,kW] flattened [b | W], dense W [nIn,nOut] 'f' order flattened [W | b],
BN [gamma | beta | mean | var].
"""
from __future__ import annotations

import dataclasses
import math
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np


# --------------------------------------------------------------------------------------------------
# Quirk flags: each is a point where recall of DL4J-beta3 is "medium confidence" (SURVEY.md section 8a).
# --------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Quirks:
    xent_clip_eps: float = 1e-5          # LossBinaryXENT default clipEps; 0 -> BCE-with-logits (north_star)
    bn_stats_minibatch_exempt: bool = True   # BN mean/var pseudo-gradients are not divided by minibatch
    bn_stats_clipped: bool = True        # ...but do pass through the layer-wise elementwise clip
    l2_after_updater: bool = True        # pre-beta4: g <- updater(g) ; g += l2*W   (not lr-scaled)
    rmsprop_cache_init_eps: bool = True  # RmsPropUpdater state initialised to epsilon
    adam_eps_outside: bool = True        # alpha_t*m/(sqrt(v)+eps), alpha_t = lr*sqrt(1-b2^t)/(1-b1^t)
    # activations of codes 5-16
    hardtanh_closed: bool = True             # HardTanh' = 1 on the CLOSED interval [-1, 1]
    hardsigmoid_closed: bool = True          # HardSigmoid' = 0.2 on the CLOSED interval [-2.5, 2.5]
    relu6_open: bool = True                  # ReLU6' = 1 on the OPEN interval (0, 6)
    thresholded_relu_in_beta3: bool = True   # ActivationThresholdedReLU exists in 1.0.0-beta3 (False: the name is refused)
    # losses of codes 2-8
    wasserstein_per_output: bool = True      # LossWasserstein divides score and gradient by nOut (moot at nOut = 1)
    # pooling
    avg_include_pad_in_divisor: bool = True  # AVG divides by kh*kw, padding included (beta4 added the switch)
    pnorm_denominator_floor: bool = True     # y^(p-1) floored at 1e-8 (SubsamplingLayer); global pooling: deliberate deviation
    global_max_first_tie: bool = True        # global MAX routes eps to the FIRST maximum in row-major order (False: the last)
    # updaters
    adagrad_history_init_eps: bool = True    # AdaGrad's history starts at eps (else at 0)
    adamax_floor_no_eps: bool = True         # AdaMax: u_inf gets + 1e-32 and the denominator has no eps (else u_inf + eps)
    nadam_v_uncorrected: bool = True         # Nadam divides by sqrt(v) + eps (else by sqrt(v / (1-b2^t)) + eps)
    # L2 gradient normalization
    bn_stats_normalized: bool = True         # BatchNorm mean/var pseudo-gradients count in the layer's norm and are scaled
    l2norm_zero_floor: float = 1e-5          # Renormalize divides by this instead of a zero norm
    # CnnLossLayer.computeScore: score /= getInputMiniBatchSize() (True); False: the row mean over N*H*W (score and gradient / (H*W) more)
    cnn_loss_score_per_minibatch: bool = True
    # weight constraints
    constraint_eps: float = 1e-6                  # BaseConstraint.DEFAULT_EPSILON
    unit_norm_zero_group_unchanged: bool = True   # UnitNorm leaves an all-zero group as it is (DL4J: 0/0 = NaN)
    # the library's Box-Muller: u = ((x_even >> 9) + 0.5) 2^-23 and v = (x_odd >> 8) 2^-24, so |z| <= sqrt(-2 ln 2^-24); DL4J draws its own
    box_muller_u_shift: int = 9
    box_muller_v_shift: int = 8
    # weight noise
    dropconnect_inverted: bool = False            # DropConnect applies ND4J's DropOut op, not DropOutInverted: W' = keep ? W : 0, not / p
    # DL4J's `train && isWeight || (applyToBias && isBias)` also perturbs biases at inference; the library perturbs nothing there (a deviation)
    noise_on_bias_in_inference: bool = False
    # weight initialization
    lecun_uniform_three_over_sqrt: bool = True    # LECUN_UNIFORM's bound 3 / sqrt(fanIn), recalled from WeightInitUtil (not sqrt(3 / fanIn))
    var_scaling_uniform_three_over_sqrt: bool = True  # VAR_SCALING_UNIFORM_FAN_{IN,OUT,AVG} bounds 3 / sqrt(fan), recalled the same way
    xavier_legacy_shape01: bool = True            # XAVIER_LEGACY's std 1 / sqrt(shape[0] + shape[1]) = 1 / sqrt(nIn + nOut) for every GEMM W
    truncation_sigmas: float = 2.0                # TruncatedNormalDistribution and VAR_SCALING_NORMAL_*: values beyond this many std are redrawn
    normal_scaled_by_fan_in: bool = True          # NORMAL is N(0, 1 / sqrt(fanIn)), not unit variance
    # regularization
    batchnorm_unregularized: bool = True          # beta3's BatchNormalization.getL1ByParam / getL2ByParam return 0 for all four parameters
    # PReLULayer
    prelu_alpha_init_zero: bool = True            # PReLULayer.Builder sets weightInit(ZERO) itself (a new PReLU is a ReLU), not the global init
    prelu_alpha_regularized: bool = True          # "W" is a weight parameter: the layer's l1 / l2 (and the global builder's) regularize alpha
    prelu_zero_is_negative: bool = False          # libnd4j prelu compares x < 0: x = +-0 is not negative (dy passes, no slope term)
    # loss weights and labels masks
    masked_score_per_minibatch: bool = True       # BaseOutputLayer.computeScore divides the masked sum by the minibatch, not the unmasked count
    mcxent_per_output_mask_refused: bool = True   # LossMCXENT throws "Per output masking for MCXENT + softmax: not supported"
    weightless_losses: tuple = ("hinge", "squared_hinge", "wasserstein")     # the losses without a weights constructor in beta3
    cnn_mask_channels: tuple = ("one", "all")     # a CnnLossLayer's NCHW masks: one value per pixel [N, 1, H, W], or one per output [N, C, H, W]


DEFAULT_QUIRKS = Quirks()


# --------------------------------------------------------------------------------------------------
# Activations (org.nd4j.linalg.activations.impl.*): forward and "backprop(z, eps) = eps * f'(z)".
# --------------------------------------------------------------------------------------------------
def _sigmoid(z):
    out = np.empty_like(z)
    pos = z >= 0
    out[pos] = 1.0 / (1.0 + np.exp(-z[pos]))
    ez = np.exp(z[~pos])
    out[~pos] = ez / (1.0 + ez)
    return out


ACTS = ("identity", "tanh", "sigmoid", "relu", "lrelu")
# b2g_activation codes 5-16, restated in float64 with f'(z) taken from the pre-activation z, as IActivation.backprop(in, epsilon) takes it
EXT_ACTS = ("elu", "selu", "softplus", "softsign", "hardtanh", "hardsigmoid", "relu6", "swish", "cube", "rationaltanh", "rectifiedtanh",
            "thresholdedrelu")
ACT_CODES = {k: 5 + i for i, k in enumerate(EXT_ACTS)}
ACT_ALPHA_DEFAULTS = {"elu": 1.0, "thresholdedrelu": 1.0}      # ELU's alpha, ThresholdedReLU's theta
SELU_LAMBDA, SELU_ALPHA = 1.0507009873554805, 1.6732632423543772
RT_A, RT_C = 1.7159, 1.41645


def _check_ext(name, q):
    if name not in EXT_ACTS:
        raise ValueError(name)
    if name == "thresholdedrelu" and not q.thresholded_relu_in_beta3:
        raise ValueError("ThresholdedReLU is not part of DL4J 1.0.0-beta3 under Quirks.thresholded_relu_in_beta3 = False")


def forward(name: str, z, alpha: float = None, q: Quirks = DEFAULT_QUIRKS) -> np.ndarray:
    """f(z) in float64 of an activation of codes 5-16 (alpha None: the kind's default)."""
    _check_ext(name, q)
    z = np.asarray(z, np.float64)
    a = ACT_ALPHA_DEFAULTS.get(name, 0.0) if alpha is None else float(alpha)
    if name == "elu":
        return np.where(z >= 0, z, a * np.expm1(np.minimum(z, 0)))
    if name == "selu":
        return SELU_LAMBDA * np.where(z > 0, z, SELU_ALPHA * np.expm1(np.minimum(z, 0)))
    if name == "softplus":
        return np.maximum(z, 0) + np.log1p(np.exp(-np.abs(z)))
    if name == "softsign":
        return z / (1 + np.abs(z))
    if name == "hardtanh":
        return np.clip(z, -1.0, 1.0)
    if name == "hardsigmoid":
        return np.clip(0.2 * z + 0.5, 0.0, 1.0)
    if name == "relu6":
        return np.clip(z, 0.0, 6.0)
    if name == "swish":
        return z * _sigmoid(z)
    if name == "cube":
        return z ** 3
    if name == "rationaltanh":
        y = 2.0 * z / 3.0
        A = 1 + np.abs(y) + y * y + RT_C * y ** 4
        return RT_A * np.sign(y) * (1 - 1 / A)
    if name == "rectifiedtanh":
        return np.maximum(0.0, np.tanh(z))
    return np.where(z > a, z, 0.0)          # thresholdedrelu


def derivative(name: str, z, alpha: float = None, q: Quirks = DEFAULT_QUIRKS) -> np.ndarray:
    """f'(z) in float64 of an activation of codes 5-16."""
    _check_ext(name, q)
    z = np.asarray(z, np.float64)
    a = ACT_ALPHA_DEFAULTS.get(name, 0.0) if alpha is None else float(alpha)
    if name == "elu":
        return np.where(z >= 0, 1.0, a * np.exp(np.minimum(z, 0)))
    if name == "selu":
        return np.where(z > 0, SELU_LAMBDA, SELU_LAMBDA * SELU_ALPHA * np.exp(np.minimum(z, 0)))
    if name == "softplus":
        return _sigmoid(z)
    if name == "softsign":
        return 1 / (1 + np.abs(z)) ** 2
    if name == "hardtanh":
        inside = (z >= -1) & (z <= 1) if q.hardtanh_closed else (z > -1) & (z < 1)
        return np.where(inside, 1.0, 0.0)
    if name == "hardsigmoid":
        inside = (z >= -2.5) & (z <= 2.5) if q.hardsigmoid_closed else (z > -2.5) & (z < 2.5)
        return np.where(inside, 0.2, 0.0)
    if name == "relu6":
        inside = (z > 0) & (z < 6) if q.relu6_open else (z >= 0) & (z <= 6)
        return np.where(inside, 1.0, 0.0)
    if name == "swish":
        s = _sigmoid(z)
        return s * (1 + z * (1 - s))
    if name == "cube":
        return 3 * z * z
    if name == "rationaltanh":
        y = 2.0 * z / 3.0
        A = 1 + np.abs(y) + y * y + RT_C * y ** 4
        return RT_A * (2.0 / 3.0) * (1 + np.sign(y) * (2 * y + 4 * RT_C * y ** 3)) / (A * A)
    if name == "rectifiedtanh":
        t = np.tanh(z)
        return np.where(z > 0, 1 - t * t, 0.0)
    return np.where(z > a, 1.0, 0.0)        # thresholdedrelu


def act_forward(name: str, z: np.ndarray, alpha: float = 0.01, q: Quirks = DEFAULT_QUIRKS) -> np.ndarray:
    if name in EXT_ACTS:
        return forward(name, z, alpha, q)
    if name == "identity":
        return z
    if name == "tanh":
        return np.tanh(z)
    if name == "sigmoid":
        return _sigmoid(z)
    if name == "relu":
        return np.maximum(z, 0)
    if name == "lrelu":  # ActivationLReLU, default alpha 0.01 (DCGAN passes 0.2 explicitly)
        return np.where(z > 0, z, alpha * z)
    raise ValueError(name)


def act_backward(name: str, z: np.ndarray, eps: np.ndarray, alpha: float = 0.01, q: Quirks = DEFAULT_QUIRKS) -> np.ndarray:
    if name in EXT_ACTS:
        return eps * derivative(name, z, alpha, q)
    if name == "identity":
        return eps
    if name == "tanh":
        t = np.tanh(z)
        return eps * (1 - t * t)
    if name == "sigmoid":
        s = _sigmoid(z)
        return eps * s * (1 - s)
    if name == "relu":
        return eps * (z > 0)
    if name == "lrelu":
        return eps * np.where(z > 0, 1.0, alpha)
    raise ValueError(name)


# The layers call the activations through these bindings, so code that wraps the module's act_forward / act_backward for its own calls
# does not change what a Net computes.
_layer_act_forward, _layer_act_backward = act_forward, act_backward


# --------------------------------------------------------------------------------------------------
# Updaters (org.nd4j.linalg.learning.config.* / org.nd4j.linalg.learning.*Updater).  With t = iteration + 1:
#   rmsprop    c = rho*c + (1-rho)*g^2;  u = lr*g / (sqrt(c) + eps)                       (c starts at eps)
#   adam       m, v;  u = lr*sqrt(1-b2^t)/(1-b1^t) * m / (sqrt(v) + eps)
#   nesterovs  vPrev = v;  v = mu*v - lr*g;  u = mu*vPrev - (1+mu)*v
#   adagrad    h += g^2;  u = lr*g / (sqrt(h) + eps)                                   (h starts at eps)
#   adamax     m = b1*m + (1-b1)*g;  u_inf = max(b2*u_inf, |g|) + 1e-32;  u = lr/(1-b1^t) * m / u_inf
#   nadam      Adam's m, v;  u = lr * (b1*m + (1-b1)*g) / (1-b1^t) / (sqrt(v) + eps)
#   amsgrad    Adam's m, v;  vhat = max(vhat, v);  u = lr*sqrt(1-b2^t)/(1-b1^t) * m / (sqrt(vhat) + eps)
#   adadelta   msg = rho*msg + (1-rho)*g^2;  u = sqrt(msdx + eps)/sqrt(msg + eps) * g;  msdx = rho*msdx + (1-rho)*u^2   (no learning rate)
#   sgd        u = lr*g;   noop  u = g
# The state slots of a parameter are in the library's order (state0, state1, state2).
# --------------------------------------------------------------------------------------------------
EXT_UPDATERS = ("nesterovs", "adagrad", "adamax", "nadam", "amsgrad", "adadelta")
N_STATE = {"sgd": 0, "noop": 0, "rmsprop": 1, "adam": 2, "nesterovs": 1, "adagrad": 1, "adamax": 2, "nadam": 2, "amsgrad": 3, "adadelta": 2}


@dataclasses.dataclass
class UpdaterCfg:
    kind: str = "sgd"            # one of N_STATE
    lr: float = 1e-3
    rms_decay: float = 0.95      # NB: reference passes RmsProp(lr, 1e-8, 1e-8) => rms_decay = 1e-8 (J:133)
    beta1: float = 0.9           # Nesterovs' momentum and AdaDelta's rho, as in b2g_layer_desc
    beta2: float = 0.999
    eps: float = 1e-8

    def state_mult(self) -> int:
        return N_STATE[self.kind]


def RmsProp(lr, rms_decay=0.95, eps=1e-8):
    """Argument order as DL4J's ctor RmsProp(learningRate, rmsDecay, epsilon)."""
    return UpdaterCfg("rmsprop", lr=lr, rms_decay=rms_decay, eps=eps)


def Adam(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8):
    return UpdaterCfg("adam", lr=lr, beta1=beta1, beta2=beta2, eps=eps)


def Sgd(lr):
    return UpdaterCfg("sgd", lr=lr)


def updater_cfg(u) -> Optional[UpdaterCfg]:
    """An updater spec dict (gan_deeplearning4j_b200.models) -> UpdaterCfg; a scheduled lr gives its value at 0, the constant the library
    keeps for it."""
    if u is None:
        return None
    k = u["kind"]
    lr = u.get("lr", 0.0)
    if isinstance(lr, dict):
        lr = value(lr, 0)
    if k == "rmsprop":
        return RmsProp(lr, u.get("rms_decay", 0.95), u.get("eps", 1e-8))
    if k == "adam":
        return Adam(lr, u.get("beta1", 0.9), u.get("beta2", 0.999), u.get("eps", 1e-8))
    if k == "sgd":
        return Sgd(lr)
    if k == "noop":
        return UpdaterCfg("noop")
    if k == "nesterovs":
        return UpdaterCfg(k, lr=lr, beta1=u.get("momentum", 0.9))
    if k == "adagrad":
        return UpdaterCfg(k, lr=lr, eps=u.get("eps", 1e-6))
    if k == "adadelta":
        return UpdaterCfg(k, lr=0.0, beta1=u.get("rho", 0.95), eps=u.get("eps", 1e-6))
    if k in ("adamax", "nadam", "amsgrad"):
        return UpdaterCfg(k, lr=lr, beta1=u.get("beta1", 0.9), beta2=u.get("beta2", 0.999), eps=u.get("eps", 1e-8))
    raise ValueError(f"unknown updater kind {k!r}")


def init_state(u: UpdaterCfg, shape, dtype=np.float64, q: Quirks = DEFAULT_QUIRKS) -> List[np.ndarray]:
    """The initial state slots of one parameter tensor."""
    if u.kind == "rmsprop":
        return [np.full(shape, u.eps if q.rmsprop_cache_init_eps else 0.0, dtype)]
    st = [np.zeros(shape, dtype) for _ in range(N_STATE[u.kind])]
    if u.kind == "adagrad" and q.adagrad_history_init_eps:
        st[0][...] = u.eps
    return st


def update(u: UpdaterCfg, st, g, t: int, q: Quirks = DEFAULT_QUIRKS, lr: Optional[float] = None):
    """The updater step u(g) of one parameter tensor at t = iteration + 1 and learning rate lr (None: u.lr); the state slots st are updated
    in place."""
    lr, b1, b2, eps = u.lr if lr is None else lr, u.beta1, u.beta2, u.eps
    if u.kind == "noop":
        return g
    if u.kind == "sgd":
        return lr * g
    if u.kind == "rmsprop":
        c = st[0]
        c[...] = u.rms_decay * c + (1 - u.rms_decay) * g * g
        return lr * g / (np.sqrt(c) + eps)
    if u.kind == "adam":
        m, v = st
        m[...] = b1 * m + (1 - b1) * g
        v[...] = b2 * v + (1 - b2) * g * g
        if q.adam_eps_outside:
            alpha_t = lr * np.sqrt(1 - b2 ** t) / (1 - b1 ** t)
            return alpha_t * m / (np.sqrt(v) + eps)
        return lr * (m / (1 - b1 ** t)) / (np.sqrt(v / (1 - b2 ** t)) + eps)
    if u.kind == "nesterovs":
        v = st[0]; v_prev = v.copy()
        v[...] = b1 * v - lr * g
        return b1 * v_prev - (1 + b1) * v
    if u.kind == "adagrad":
        h = st[0]
        h[...] = h + g * g
        return lr * g / (np.sqrt(h) + eps)
    if u.kind == "adamax":
        m, ui = st
        m[...] = b1 * m + (1 - b1) * g
        if q.adamax_floor_no_eps:
            ui[...] = np.maximum(b2 * ui, np.abs(g)) + 1e-32
            return lr / (1 - b1 ** t) * m / ui
        ui[...] = np.maximum(b2 * ui, np.abs(g))
        return lr / (1 - b1 ** t) * m / (ui + eps)
    if u.kind in ("nadam", "amsgrad"):
        m, v = st[0], st[1]
        m[...] = b1 * m + (1 - b1) * g
        v[...] = b2 * v + (1 - b2) * g * g
        if u.kind == "nadam":
            vv = v if q.nadam_v_uncorrected else v / (1 - b2 ** t)
            return lr * (b1 * m + (1 - b1) * g) / (1 - b1 ** t) / (np.sqrt(vv) + eps)
        vh = st[2]
        vh[...] = np.maximum(vh, v)
        return lr * np.sqrt(1 - b2 ** t) / (1 - b1 ** t) * m / (np.sqrt(vh) + eps)
    if u.kind == "adadelta":
        msg, msdx = st
        msg[...] = b1 * msg + (1 - b1) * g * g
        d = np.sqrt(msdx + eps) / np.sqrt(msg + eps) * g
        msdx[...] = b1 * msdx + (1 - b1) * d * d
        return d
    raise ValueError(u.kind)


# --------------------------------------------------------------------------------------------------
# Learning-rate schedules (org.nd4j.linalg.schedule.ISchedule).  value(i) in double, i = the iteration count before the update's increment
# (ITERATION) or the epoch count (EPOCH):
#   exponential  initial * gamma^i                       inverse  initial / (1 + gamma*i)^power
#   sigmoid      initial / (1 + exp(-gamma*(i - step)))  step     initial * decay_rate^floor(i / step)
#   map          the value at the largest key <= i
# The updater uses value(i) rounded to fp32 once in place of its constant lr.  The schedules are the dicts gan_deeplearning4j_b200.models
# builds.
# --------------------------------------------------------------------------------------------------
def value(sched, i) -> float:
    """ISchedule.valueAt in double for the schedule's own counter value i."""
    k, i = sched["schedule"], float(i)
    if k == "exponential":
        return sched["initial"] * math.pow(sched["gamma"], i)
    if k == "inverse":
        return sched["initial"] / math.pow(1.0 + sched["gamma"] * i, sched["power"])
    if k == "sigmoid":
        return sched["initial"] / (1.0 + math.exp(-sched["gamma"] * (i - sched["step"])))
    if k == "step":
        return sched["initial"] * math.pow(sched["decay_rate"], math.floor(i / sched["step"]))
    if k == "map":
        best = None
        for key, v in sched["values"]:
            if key <= i and (best is None or key > best[0]):
                best = (key, v)
        assert best is not None, "a MapSchedule must hold key 0"
        return float(best[1])
    raise ValueError(k)


def lr_at(sched, iteration: int, epoch: int) -> np.float32:
    """The fp32 learning rate of an update at (iteration before the increment, epoch)."""
    return np.float32(value(sched, epoch if sched.get("type", "iteration") == "epoch" else iteration))


# --------------------------------------------------------------------------------------------------
# L2 gradient normalization (BaseMultiLayerUpdater.preApply), between the division by mb and the updater:
#   renormalize_l2_per_layer        g <- g / ||g_layer||  (a zero norm divides by `l2norm_zero_floor` instead; the threshold is ignored)
#   renormalize_l2_per_param_type   the same per parameter tensor
#   clip_l2_per_layer               g <- g * threshold / ||g_layer||  when ||g_layer|| > threshold
#   clip_l2_per_param_type          the same per parameter tensor
# A layer is one layer with parameters that is not frozen; its BatchNorm mean/var pseudo-gradients (not divided by mb) are inside its norm
# and scaled with it when `bn_stats_normalized` holds.  The multiplier is rounded to fp32 once, as the library does.
# --------------------------------------------------------------------------------------------------
GRAD_NORMS = ("none", "renormalize_l2_per_layer", "renormalize_l2_per_param_type", "clip_l2_per_layer", "clip_l2_per_param_type")


def multiplier(sumsq: float, mode: str, threshold: float, q: Quirks = DEFAULT_QUIRKS) -> np.float32:
    """The fp32 multiplier of one norm group from its sum of squares."""
    norm = math.sqrt(sumsq)
    if mode.startswith("renormalize"):
        return np.float32(1.0 / (norm if norm != 0.0 else q.l2norm_zero_floor))
    thr = float(np.float32(threshold))
    return np.float32(thr / norm) if norm > thr else np.float32(1.0)


def norm_groups(net, g, mode, q: Quirks = DEFAULT_QUIRKS):
    """The mode's norm groups over the divided gradients g: lists of (layer, param) keys, in parameter order."""
    groups = {}
    for (li, p) in g:
        l = net.layers[li]
        if p in l.noop_names() and not q.bn_stats_normalized:
            continue
        groups.setdefault(li if mode.endswith("per_layer") else (li, p), []).append((li, p))
    return list(groups.values())


def normalize(net, g, mode, threshold, q: Quirks = DEFAULT_QUIRKS):
    """Applies the mode to the divided gradients g {(layer, param): g} (a new dict); also returns the groups' norms."""
    out, norms = dict(g), []
    for keys in norm_groups(net, g, mode, q):
        ss = sum(float((np.asarray(g[k], np.float64) ** 2).sum()) for k in keys)
        norms.append(math.sqrt(ss))
        m = multiplier(ss, mode, threshold, q)
        for k in keys:
            out[k] = g[k] * float(m)
    return out, norms


# --------------------------------------------------------------------------------------------------
# Weight constraints (LayerConstraint: MaxNorm, MinMaxNorm, UnitNorm, NonNegative; the dicts of models.max_norm, ...).  They run after
# theta -= u in every update (``Net.apply_update``), never on a FrozenLayer, and never after averaging, set_params_flat or
# compute_gradient_and_score.
# --------------------------------------------------------------------------------------------------
CONSTRAINT_KINDS = ("max_norm", "min_max_norm", "unit_norm", "non_negative")
CONSTRAINT_ON = ("all", "weights", "bias")      # also the order a tensor's lists apply in: constrainAllParameters, Weights, Bias


def constraint_multiplier(c: Dict, norm, q: Quirks = DEFAULT_QUIRKS):
    """The fp32 multiplier of a group of L2 norm `norm` (float64 arrays), computed in double and rounded once."""
    norm = np.asarray(norm, np.float64)
    eps = q.constraint_eps
    k = c["constraint"]
    if k == "max_norm":
        m = np.minimum(norm, c["max"]) / (norm + eps)
    elif k == "min_max_norm":
        rate = c.get("rate", 1.0)
        m = (rate * np.minimum(np.maximum(norm, c["min"]), c["max"]) + (1.0 - rate) * norm) / (norm + eps)
    elif k == "unit_norm":
        with np.errstate(divide="ignore", invalid="ignore"):
            m = 1.0 / norm
        if q.unit_norm_zero_group_unchanged:
            m = np.where(norm == 0.0, 1.0, m)
    else:
        raise ValueError(k)
    return m.astype(np.float32)


def apply_constraint(w: np.ndarray, c: Dict, q: Quirks = DEFAULT_QUIRKS) -> np.ndarray:
    """One constraint on one parameter in its DL4J shape ([n] vectors as [1, n]; float64 or float32)."""
    dt = w.dtype
    if c["constraint"] == "non_negative":
        return np.where(w < 0, np.zeros((), dt), w)
    if w.ndim == 1:                    # b, gamma, beta, mean, var: DL4J's [1, n]
        return apply_constraint(w.reshape(1, -1), c, q).reshape(w.shape)
    dims = tuple(sorted(set(c.get("dims", ())))) or tuple(range(w.ndim))
    norm = np.sqrt((w.astype(np.float64) ** 2).sum(axis=dims, keepdims=True))
    return (w * constraint_multiplier(c, norm, q).astype(dt)).astype(dt)


def constraints_by_param(layer: Layer, constraints: Sequence[Dict]) -> Dict[str, List[Dict]]:
    """One layer's constraints as parameter name -> the ordered list its tensor runs (DL4J initializeConstraints): on a layer with parameters
    that is not frozen, "weights" reaches W, "bias" b and "all" every parameter, where the layer has them (a PReLU's alpha takes none: the
    library refuses them); each list runs the all-parameter constraints, then the weight, then the bias ones, each in the order given.
    ValueError for an unknown target or kind."""
    for c in constraints:
        if c.get("on", "weights") not in CONSTRAINT_ON or c.get("constraint") not in CONSTRAINT_KINDS:
            raise ValueError(f"constraint {c!r}: targets {CONSTRAINT_ON}, kinds {CONSTRAINT_KINDS}")
    live = layer.has_params and not getattr(layer, "frozen", False) and not isinstance(layer, PReLU)
    names = [p for p, _, _ in layer.param_specs()] if live else []
    reach = {"all": names, "weights": [p for p in names if p == "W"], "bias": [p for p in names if p == "b"]}
    out: Dict[str, List[Dict]] = {}
    for c in sorted(constraints, key=lambda c: CONSTRAINT_ON.index(c.get("on", "weights"))):    # stable: the given order within a target
        for p in reach[c.get("on", "weights")]:
            out.setdefault(p, []).append(c)
    return out


# --------------------------------------------------------------------------------------------------
# im2col / col2im (libnd4j helpers::im2col / col2im; ConvolutionMode.Truncate)
# --------------------------------------------------------------------------------------------------
def out_size(n, k, s, p):
    return (n - k + 2 * p) // s + 1


def im2col(x: np.ndarray, kh, kw, sh, sw, ph, pw) -> np.ndarray:
    """x [N,C,H,W] -> cols [N, oH, oW, C, kH, kW] (a strided view of the zero-padded input)."""
    n, c, h, w = x.shape
    oh, ow = out_size(h, kh, sh, ph), out_size(w, kw, sw, pw)
    xp = np.pad(x, ((0, 0), (0, 0), (ph, ph), (pw, pw))) if (ph or pw) else x
    s = xp.strides
    return np.lib.stride_tricks.as_strided(
        xp, shape=(n, oh, ow, c, kh, kw),
        strides=(s[0], s[2] * sh, s[3] * sw, s[1], s[2], s[3]), writeable=False)


def col2im(cols: np.ndarray, x_shape, kh, kw, sh, sw, ph, pw) -> np.ndarray:
    """Adjoint of im2col: cols [N,oH,oW,C,kH,kW] scatter-added into [N,C,H,W]."""
    n, c, h, w = x_shape
    oh, ow = cols.shape[1], cols.shape[2]
    xp = np.zeros((n, c, h + 2 * ph, w + 2 * pw), dtype=cols.dtype)
    for i in range(kh):
        for j in range(kw):
            xp[:, :, i:i + sh * oh:sh, j:j + sw * ow:sw] += cols[:, :, :, :, i, j].transpose(0, 3, 1, 2)
    return xp[:, :, ph:ph + h, pw:pw + w]


# --------------------------------------------------------------------------------------------------
# Layers.  Each has: param_specs() -> [(name, shape, order)], forward(x, train), backward(eps) -> eps_in
# and leaves *summed* (not minibatch-averaged) gradients in self.grads, as DL4J layers do.
# --------------------------------------------------------------------------------------------------
class Layer:
    name: str = ""
    index: int = 0                  # the layer's chain index in the CUDA library's layer array (its spec position): the draws' L
    updater: Optional[UpdaterCfg] = None
    l2: float = 0.0
    weight_noise: Optional[Dict] = None     # a conv, deconv or dense layer's DropConnect / WeightNoise
    noisy: Optional[Dict] = None            # its W' (and b') of the current train-mode pass, in W's shape, or None
    has_params = False
    q: Quirks = DEFAULT_QUIRKS      # a Net gives its quirks to the layers that have none of their own

    def param_specs(self) -> List[Tuple[str, Tuple[int, ...], str]]:
        return []

    def l2_names(self) -> Tuple[str, ...]:
        """The parameters the layer's l2 reaches."""
        return ()

    def _p(self, name):
        """The parameter a forward or an input gradient reads: the pass's noisy operand if it has one."""
        return self.noisy[name] if self.noisy is not None and name in self.noisy else self.params[name]

    def noop_names(self) -> Tuple[str, ...]:
        return ()

    def init(self, rng: np.random.Generator, dtype):
        self.params: Dict[str, np.ndarray] = {}
        self.grads: Dict[str, np.ndarray] = {}

    def out_shape(self, in_shape):
        return in_shape


class Conv2D(Layer):
    """o.d.nn.layers.convolution.ConvolutionLayer: cross-correlation, Truncate mode (J:135-140)."""
    has_params = True

    def __init__(self, n_in, n_out, kernel, stride=(1, 1), padding=(0, 0), activation="identity", alpha=0.01,
                 updater=None, l2=0.0, name="", has_bias=True):
        self.n_in, self.n_out = n_in, n_out
        self.k, self.s, self.p = tuple(kernel), tuple(stride), tuple(padding)
        self.activation, self.alpha = activation, alpha
        self.updater, self.l2, self.name, self.has_bias = updater, l2, name, has_bias

    def param_specs(self):
        # ConvolutionParamInitializer: flattened view is [b | W], W 'c' order [nOut,nIn,kH,kW]
        w = ("W", (self.n_out, self.n_in) + self.k, "c")
        return [("b", (self.n_out,), "c"), w] if self.has_bias else [w]

    def l2_names(self):
        return ("W",)

    def fans(self):
        kh, kw = self.k
        return self.n_in * kh * kw, self.n_out * kh * kw / (self.s[0] * self.s[1])

    def init(self, rng, dtype):
        super().init(rng, dtype)
        fi, fo = self.fans()
        self.params["W"] = (rng.standard_normal((self.n_out, self.n_in) + self.k) * np.sqrt(2.0 / (fi + fo))).astype(dtype)
        if self.has_bias:
            self.params["b"] = np.zeros(self.n_out, dtype)

    def out_shape(self, s):
        n, c, h, w = s
        return (n, self.n_out, out_size(h, self.k[0], self.s[0], self.p[0]), out_size(w, self.k[1], self.s[1], self.p[1]))

    def forward(self, x, train):
        n = x.shape[0]
        cols = im2col(x, *self.k, *self.s, *self.p)
        oh, ow = cols.shape[1], cols.shape[2]
        self._x_shape = x.shape
        self._cols2d = np.ascontiguousarray(cols).reshape(n * oh * ow, -1)
        w2d = self._p("W").reshape(self.n_out, -1)
        z2d = self._cols2d @ w2d.T
        if self.has_bias:
            z2d = z2d + self._p("b")
        self._z = z2d.reshape(n, oh, ow, self.n_out).transpose(0, 3, 1, 2)
        return _layer_act_forward(self.activation, self._z, self.alpha, self.q)

    def backward(self, eps):
        delta = _layer_act_backward(self.activation, self._z, eps, self.alpha, self.q)
        n, o, oh, ow = delta.shape
        d2d = delta.transpose(0, 2, 3, 1).reshape(-1, o)
        self.grads["W"] = (d2d.T @ self._cols2d).reshape(self.params["W"].shape)
        if self.has_bias:
            self.grads["b"] = d2d.sum(0)
        w2d = self._p("W").reshape(o, -1)
        dcols = (d2d @ w2d).reshape(n, oh, ow, self.n_in, *self.k)
        return col2im(dcols, self._x_shape, *self.k, *self.s, *self.p)


class Deconv2D(Layer):
    """DL4J Deconvolution2D / libnd4j deconv2d: out = s*(in-1)+k-2p; W [nIn,nOut,kH,kW]; flattened [b | W]."""
    has_params = True

    def __init__(self, n_in, n_out, kernel, stride=(1, 1), padding=(0, 0), activation="identity", alpha=0.01,
                 updater=None, l2=0.0, name="", has_bias=True):
        self.n_in, self.n_out = n_in, n_out
        self.k, self.s, self.p = tuple(kernel), tuple(stride), tuple(padding)
        self.activation, self.alpha = activation, alpha
        self.updater, self.l2, self.name, self.has_bias = updater, l2, name, has_bias

    def param_specs(self):
        w = ("W", (self.n_in, self.n_out) + self.k, "c")
        return [("b", (self.n_out,), "c"), w] if self.has_bias else [w]

    def l2_names(self):
        return ("W",)

    def fans(self):
        kh, kw = self.k
        return self.n_in * kh * kw, self.n_out * kh * kw / (self.s[0] * self.s[1])

    def init(self, rng, dtype):
        super().init(rng, dtype)
        fi, fo = self.fans()
        self.params["W"] = (rng.standard_normal((self.n_in, self.n_out) + self.k) * np.sqrt(2.0 / (fi + fo))).astype(dtype)
        if self.has_bias:
            self.params["b"] = np.zeros(self.n_out, dtype)

    def out_shape(self, s):
        n, c, h, w = s
        return (n, self.n_out, self.s[0] * (h - 1) + self.k[0] - 2 * self.p[0], self.s[1] * (w - 1) + self.k[1] - 2 * self.p[1])

    def forward(self, x, train):
        n, c, h, w = x.shape
        self._x2d = x.transpose(0, 2, 3, 1).reshape(-1, c)
        self._x_shape = x.shape
        osh = self.out_shape(x.shape)
        w2d = self._p("W").reshape(self.n_in, -1)               # [Cin, Cout*kH*kW]
        cols = (self._x2d @ w2d).reshape(n, h, w, self.n_out, *self.k)
        z = col2im(cols, osh, *self.k, *self.s, *self.p)
        if self.has_bias:
            z = z + self._p("b")[None, :, None, None]
        self._z = z
        return _layer_act_forward(self.activation, z, self.alpha, self.q)

    def backward(self, eps):
        delta = _layer_act_backward(self.activation, self._z, eps, self.alpha, self.q)
        n, c, h, w = self._x_shape
        dcols = np.ascontiguousarray(im2col(delta, *self.k, *self.s, *self.p)).reshape(n * h * w, -1)  # [pix, Cout*kH*kW]
        self.grads["W"] = (self._x2d.T @ dcols).reshape(self.params["W"].shape)
        if self.has_bias:
            self.grads["b"] = delta.sum((0, 2, 3))
        w2d = self._p("W").reshape(self.n_in, -1)
        return (dcols @ w2d.T).reshape(n, h, w, c).transpose(0, 3, 1, 2)


class Dense(Layer):
    """DenseLayer/BaseLayer: z = xW + b; W [nIn,nOut] 'f' order; flattened [W | b] (J:155-158)."""
    has_params = True

    def __init__(self, n_in, n_out, activation="identity", alpha=0.01, updater=None, l2=0.0, name="", has_bias=True):
        self.n_in, self.n_out = n_in, n_out
        self.activation, self.alpha = activation, alpha
        self.updater, self.l2, self.name, self.has_bias = updater, l2, name, has_bias

    def param_specs(self):
        w = ("W", (self.n_in, self.n_out), "f")
        return [w, ("b", (self.n_out,), "c")] if self.has_bias else [w]

    def l2_names(self):
        return ("W",)

    def fans(self):
        return self.n_in, self.n_out

    def init(self, rng, dtype):
        super().init(rng, dtype)
        self.params["W"] = (rng.standard_normal((self.n_in, self.n_out)) * np.sqrt(2.0 / (self.n_in + self.n_out))).astype(dtype)
        if self.has_bias:
            self.params["b"] = np.zeros(self.n_out, dtype)

    def out_shape(self, s):
        return (s[0], self.n_out)

    def forward(self, x, train):
        self._x = x
        self._z = x @ self._p("W")
        if self.has_bias:
            self._z = self._z + self._p("b")
        return _layer_act_forward(self.activation, self._z, self.alpha, self.q)

    def backward(self, eps):
        delta = _layer_act_backward(self.activation, self._z, eps, self.alpha, self.q)
        self._delta = delta
        self.grads["W"] = self._x.T @ delta
        if self.has_bias:
            self.grads["b"] = delta.sum(0)
        return delta @ self._p("W").T


GEMM = (Conv2D, Deconv2D, Dense)          # the layers with a W: Output and OutputSoftmax are Dense


class BatchNorm(Layer):
    """o.d.nn.layers.normalization.BatchNormalization (J:132-134): decay 0.9, eps 1e-5, biased batch var,
    running mean/var stored as *parameters* and moved by pseudo-gradients through a NoOp updater."""
    has_params = True

    def __init__(self, n, decay=0.9, eps=1e-5, updater=None, name=""):
        self.n, self.decay, self.eps = n, decay, eps
        self.updater, self.name, self.l2 = updater, name, 0.0

    def param_specs(self):
        return [("gamma", (self.n,), "c"), ("beta", (self.n,), "c"), ("mean", (self.n,), "c"), ("var", (self.n,), "c")]

    def noop_names(self):
        return ("mean", "var")

    def init(self, rng, dtype):
        super().init(rng, dtype)
        self.params["gamma"] = np.ones(self.n, dtype)
        self.params["beta"] = np.zeros(self.n, dtype)
        self.params["mean"] = np.zeros(self.n, dtype)
        self.params["var"] = np.ones(self.n, dtype)

    def _bc(self, v, ndim):
        return v[None, :, None, None] if ndim == 4 else v[None, :]

    def forward(self, x, train):
        axes = (0, 2, 3) if x.ndim == 4 else (0,)
        if train:
            mu = x.mean(axes)
            var = ((x - self._bc(mu, x.ndim)) ** 2).mean(axes)     # biased
            self._mu, self._var = mu, var
        else:
            mu, var = self.params["mean"], self.params["var"]
        std = np.sqrt(var + self.eps)
        self._std = std
        self._xhat = (x - self._bc(mu, x.ndim)) / self._bc(std, x.ndim)
        self._m = x.size // self.n
        return self._bc(self.params["gamma"], x.ndim) * self._xhat + self._bc(self.params["beta"], x.ndim)

    def backward(self, eps):
        nd = eps.ndim
        axes = (0, 2, 3) if nd == 4 else (0,)
        g = self.params["gamma"]
        xhat, std, m = self._xhat, self._std, self._m
        self.grads["beta"] = eps.sum(axes)
        self.grads["gamma"] = (eps * xhat).sum(axes)
        # running-stat pseudo-gradients: theta <- theta - (1-decay)(theta - batch_stat)
        self.grads["mean"] = (1 - self.decay) * (self.params["mean"] - self._mu)
        self.grads["var"] = (1 - self.decay) * (self.params["var"] - self._var)
        dxhat = eps * self._bc(g, nd)
        # dx = (1/std) * (dxhat - mean(dxhat) - xhat*mean(dxhat*xhat))
        return (dxhat - self._bc(dxhat.sum(axes) / m, nd) - xhat * self._bc((dxhat * xhat).sum(axes) / m, nd)) / self._bc(std, nd)


class ActivationLayer(Layer):
    """o.d.nn.conf.layers.ActivationLayer (north_star's ReLU / LeakyReLU after BatchNormalization)."""

    def __init__(self, activation, alpha=0.01, name=""):
        self.activation, self.alpha, self.name = activation, alpha, name

    def init(self, rng, dtype):
        super().init(rng, dtype)

    def forward(self, x, train):
        self._z = x
        return _layer_act_forward(self.activation, x, self.alpha, self.q)

    def backward(self, eps):
        return _layer_act_backward(self.activation, self._z, eps, self.alpha, self.q)


class PReLU(Layer):
    """PReLULayer.Builder().inputShape(in_shape).sharedAxes(shared_axes) (B2G_LAYER_PRELU): in_shape (C, H, W) or (F,), shared_axes DL4J's
    1-based axes.
      forward   y = x < 0 ? alpha * x : x
      backward  dx = x < 0 ? alpha * eps : eps;  dalpha = sum over the minibatch and the shared axes of (x < 0 ? x * eps : 0)
    alpha ("W") has DL4J's weight shape: in_shape with every shared axis of extent 1, so in the NCHW layout it broadcasts over the minibatch
    and the shared axes as it is.  A FrozenLayer PReLU is the same function in both modes and passes an input gradient (Net's backward walk
    goes through it)."""
    has_params = True

    def __init__(self, in_shape, shared_axes=(), updater=None, l2=0.0, name=""):
        self.in_shape = tuple(int(d) for d in in_shape)
        self.shared = tuple(sorted({int(a) for a in shared_axes}))
        if any(a < 1 or a > len(self.in_shape) for a in self.shared):
            raise ValueError(f"prelu {name!r}: shared axes {self.shared} outside the input's {len(self.in_shape)} dimension(s)")
        self.alpha_shape = tuple(1 if i + 1 in self.shared else d for i, d in enumerate(self.in_shape))
        self.updater, self.l2, self.name = updater, l2, name

    def param_specs(self):
        return [("W", self.alpha_shape, "c")]

    def l2_names(self):
        return ("W",) if self.q.prelu_alpha_regularized else ()

    def init(self, rng, dtype):
        super().init(rng, dtype)
        if not self.q.prelu_alpha_init_zero:
            raise NotImplementedError("only beta3's ZERO initial alpha is restated")
        self.params["W"] = np.zeros(self.alpha_shape, dtype)

    def _neg(self, x):
        return x <= 0 if self.q.prelu_zero_is_negative else x < 0

    def forward(self, x, train):
        self._x = x
        return np.where(self._neg(x), self.params["W"][None] * x, x)

    def backward(self, eps):
        x, neg = self._x, self._neg(self._x)
        if not getattr(self, "frozen", False):
            axes = (0,) + self.shared           # DL4J axis a is array axis a of the [N, ...] activation
            self.grads["W"] = np.where(neg, x * eps, 0.0).sum(axis=axes, keepdims=True).reshape(self.alpha_shape)
        return np.where(neg, self.params["W"][None] * eps, eps)


class MaxPool(Layer):
    """SubsamplingLayer(PoolingType.MAX) (J:141-144): Truncate mode; ties -> first in window row-major order."""

    def __init__(self, kernel=(2, 2), stride=(1, 1), name=""):
        self.k, self.s, self.name = tuple(kernel), tuple(stride), name

    def init(self, rng, dtype):
        super().init(rng, dtype)

    def out_shape(self, s):
        n, c, h, w = s
        return (n, c, out_size(h, self.k[0], self.s[0], 0), out_size(w, self.k[1], self.s[1], 0))

    def forward(self, x, train):
        cols = im2col(x, *self.k, *self.s, 0, 0)                       # [N,oH,oW,C,kH,kW]
        n, oh, ow, c = cols.shape[:4]
        flat = cols.reshape(n, oh, ow, c, -1)
        self._arg = flat.argmax(-1)                                     # first max in row-major window order
        self._x_shape = x.shape
        return np.take_along_axis(flat, self._arg[..., None], -1)[..., 0].transpose(0, 3, 1, 2)

    def backward(self, eps):
        n, c, oh, ow = eps.shape
        kh, kw = self.k
        dflat = np.zeros((n, oh, ow, c, kh * kw), dtype=eps.dtype)
        np.put_along_axis(dflat, self._arg[..., None], eps.transpose(0, 2, 3, 1)[..., None], -1)
        return col2im(dflat.reshape(n, oh, ow, c, kh, kw), self._x_shape, kh, kw, *self.s, 0, 0)


# Average, sum and p-norm pooling (b2g_pooling), in float64.  Truncate geometry OH = (H + 2 ph - kh) / sh + 1; positions outside the input
# are zero padding.
#   AVG    y = window sum / (kh*kw)                dx += eps / (kh*kw)
#   SUM    y = window sum                          dx += eps
#   PNORM  y = (sum |x|^p)^(1/p)                   dx += eps * sign(x)|x|^(p-1) / max(y^(p-1), 1e-8)
# GlobalPoolingLayer pools over H x W to [mb, C]; MAX routes eps to the first maximum in row-major pixel order.  The p-norm floor is
# SubsamplingLayer's eps; DL4J's GlobalPoolingLayer has no floor (a zero map gives NaN there), so for global pooling the floor is a
# deliberate deviation of the library, kept here as the default.
POOLINGS = ("max", "avg", "sum", "pnorm")
POOL_CODES = {k: i for i, k in enumerate(POOLINGS)}
PNORM_EPS = 1e-8


def _pnorm_den(y, p, q):
    d = y ** (p - 1)
    return np.maximum(d, PNORM_EPS) if q.pnorm_denominator_floor else d


def _pnorm_num(x, p):
    return np.sign(x) * np.abs(x) ** (p - 1)


def pool2d_forward(kind, x, kernel, stride, padding, p=2, q: Quirks = DEFAULT_QUIRKS):
    """x [N,C,H,W] float64 -> y [N,C,OH,OW]."""
    (kh, kw), (sh, sw), (ph, pw) = kernel, stride, padding
    cols = im2col(np.asarray(x, np.float64), kh, kw, sh, sw, ph, pw)          # [N,OH,OW,C,kh,kw], zero padded
    if kind == "avg":
        if q.avg_include_pad_in_divisor:
            div = kh * kw
        else:
            div = im2col(np.ones((1, 1) + x.shape[2:]), kh, kw, sh, sw, ph, pw).sum((-2, -1))[0, :, :, 0][None, :, :, None]
        y = cols.sum((-2, -1)) / div
    elif kind == "sum":
        y = cols.sum((-2, -1))
    elif kind == "pnorm":
        y = (np.abs(cols) ** p).sum((-2, -1)) ** (1.0 / p)
    else:
        raise ValueError(kind)
    return y.transpose(0, 3, 1, 2)


def pool2d_backward(kind, x, y, eps, kernel, stride, padding, p=2, q: Quirks = DEFAULT_QUIRKS):
    """dL/dx [N,C,H,W] from eps = dL/dy [N,C,OH,OW] (y = the forward's output)."""
    (kh, kw), (sh, sw), (ph, pw) = kernel, stride, padding
    x = np.asarray(x, np.float64)
    e = np.asarray(eps, np.float64).transpose(0, 2, 3, 1)[..., None, None]      # [N,OH,OW,C,1,1]
    shape = e.shape[:4] + (kh, kw)
    if kind == "avg":
        if q.avg_include_pad_in_divisor:
            dcols = np.broadcast_to(e / (kh * kw), shape)
        else:
            cnt = im2col(np.ones((1, 1) + x.shape[2:]), kh, kw, sh, sw, ph, pw).sum((-2, -1))[0, :, :, 0][None, :, :, None, None, None]
            dcols = np.broadcast_to(e / cnt, shape)
    elif kind == "sum":
        dcols = np.broadcast_to(e, shape)
    elif kind == "pnorm":
        cols = im2col(x, kh, kw, sh, sw, ph, pw)
        yy = np.asarray(y, np.float64).transpose(0, 2, 3, 1)[..., None, None]
        dcols = e * _pnorm_num(cols, p) / _pnorm_den(yy, p, q)
    else:
        raise ValueError(kind)
    return col2im(np.ascontiguousarray(dcols), x.shape, kh, kw, sh, sw, ph, pw)


def global_forward(kind, x, p=2, q: Quirks = DEFAULT_QUIRKS):
    """x [N,C,H,W] (or [N,C]) -> (y [N,C], MAX's row-major pixel index [N,C] or None)."""
    x = np.asarray(x, np.float64)
    f = x.reshape(x.shape[0], x.shape[1], -1)
    if kind == "max":
        idx = f.argmax(-1) if q.global_max_first_tie else f.shape[-1] - 1 - f[..., ::-1].argmax(-1)
        return np.take_along_axis(f, idx[..., None], -1)[..., 0], idx
    if kind == "avg":
        return f.mean(-1), None
    if kind == "sum":
        return f.sum(-1), None
    if kind == "pnorm":
        return (np.abs(f) ** p).sum(-1) ** (1.0 / p), None
    raise ValueError(kind)


def global_backward(kind, x, y, idx, eps, p=2, q: Quirks = DEFAULT_QUIRKS):
    x = np.asarray(x, np.float64)
    f = x.reshape(x.shape[0], x.shape[1], -1)
    e = np.asarray(eps, np.float64)[..., None]
    if kind == "max":
        d = np.zeros_like(f)
        np.put_along_axis(d, idx[..., None], e, -1)
    elif kind == "avg":
        d = np.broadcast_to(e / f.shape[-1], f.shape)
    elif kind == "sum":
        d = np.broadcast_to(e, f.shape)
    elif kind == "pnorm":
        d = e * _pnorm_num(f, p) / _pnorm_den(np.asarray(y, np.float64)[..., None], p, q)
    else:
        raise ValueError(kind)
    return np.ascontiguousarray(d).reshape(x.shape)


class Subsampling(Layer):
    """SubsamplingLayer.Builder(PoolingType.AVG / SUM / PNORM).kernelSize().stride().padding().pnorm()."""

    def __init__(self, kind, kernel, stride=(1, 1), padding=(0, 0), p=2, name=""):
        self.kind, self.k, self.s, self.pad, self.p, self.name = kind, tuple(kernel), tuple(stride), tuple(padding), p, name

    def out_shape(self, s):
        n, c, h, w = s
        return (n, c, out_size(h, self.k[0], self.s[0], self.pad[0]), out_size(w, self.k[1], self.s[1], self.pad[1]))

    def forward(self, x, train):
        self._x = x
        self._y = pool2d_forward(self.kind, x, self.k, self.s, self.pad, self.p, self.q)
        return self._y

    def backward(self, eps):
        return pool2d_backward(self.kind, self._x, self._y, eps, self.k, self.s, self.pad, self.p, self.q)


class GlobalPooling(Layer):
    """GlobalPoolingLayer.Builder(PoolingType).pnorm(p): [N,C,H,W] -> [N,C]."""

    def __init__(self, kind="max", p=2, name=""):
        self.kind, self.p, self.name = kind, p, name

    def out_shape(self, s):
        return (s[0], s[1])

    def forward(self, x, train):
        self._x = x
        self._y, self._idx = global_forward(self.kind, x, self.p, self.q)
        return self._y

    def backward(self, eps):
        return global_backward(self.kind, self._x, self._y, self._idx, eps, self.p, self.q)


class Upsample2D(Layer):
    """Upsampling2D.Builder(size) (J:201-202): nearest neighbour; backward sums each size x size block."""

    def __init__(self, size=2, name=""):
        self.size, self.name = size, name

    def init(self, rng, dtype):
        super().init(rng, dtype)

    def out_shape(self, s):
        return (s[0], s[1], s[2] * self.size, s[3] * self.size)

    def forward(self, x, train):
        return x.repeat(self.size, 2).repeat(self.size, 3)

    def backward(self, eps):
        n, c, h, w = eps.shape
        f = self.size
        return eps.reshape(n, c, h // f, f, w // f, f).sum((3, 5))


class Reshape(Layer):
    """FeedForwardToCnnPreProcessor(h,w,c) (J:200) / CnnToFeedForwardPreProcessor: 'c'-order reshape."""

    def __init__(self, to_shape: Tuple[int, ...], name=""):
        self.to_shape, self.name = tuple(to_shape), name

    def init(self, rng, dtype):
        super().init(rng, dtype)

    def out_shape(self, s):
        return (s[0],) + self.to_shape

    def forward(self, x, train):
        self._in_shape = x.shape
        return x.reshape((x.shape[0],) + self.to_shape)

    def backward(self, eps):
        return eps.reshape(self._in_shape)


# --------------------------------------------------------------------------------------------------
# The library's random draws.  ND4J's random stream cannot be restated, so every draw is the CUDA library's own definition (include/b200gan.h),
# restated exactly: parity with DL4J holds in distribution, with the library element for element.  Draw index j takes word j & 3 of
# Philox4x32-10(ctr = {j >> 2, c1, c2, c3}, key = {lo32(S), hi32(S)}), S = the net's seed (0 -> 666), with counter words 1-3
#   DropoutLayers and weight noise  {lo32(P), hi32(P), L | r << 16}   (pass P, layer L, rank r < 2^15)
#   weight initialization           {k, 0, L | 2^31}                  (round k)
# so the two streams never share a counter.  A keep bit is x < floor(p 2^32); a normal pairs words (x0, x1) -> z0, z1 and (x2, x3) -> z2, z3
# through box_muller; a uniform is fmaf(upper - lower, (x >> 8) 2^-24, lower).
# --------------------------------------------------------------------------------------------------
_M32 = np.uint64(0xFFFFFFFF)
WEIGHT_INIT_TAG = 0x80000000
Z_MAX = math.sqrt(-2.0 * math.log(2.0 ** -24))          # the largest |z| box_muller gives


def philox4x32_10(ctr, key):
    """Philox4x32-10 (Random123 constants), vectorised: ctr = 4 arrays / ints of 32-bit words, key = 2.  Returns the 4 output words (uint32)."""
    c = [np.asarray(v, np.uint64) & _M32 for v in ctr]
    k0, k1 = (np.uint64(int(v) & 0xFFFFFFFF) for v in key)
    m0, m1, w0, w1, sh = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), np.uint64(0x9E3779B9), np.uint64(0xBB67AE85), np.uint64(32)
    for r in range(10):
        if r:
            k0, k1 = (k0 + w0) & _M32, (k1 + w1) & _M32
        p0, p1 = m0 * c[0], m1 * c[2]          # 32 x 32 -> 64-bit products, exact in uint64
        c = [(p1 >> sh) ^ c[1] ^ k0, p1 & _M32, (p0 >> sh) ^ c[3] ^ k1, p0 & _M32]
    return [v.astype(np.uint32) for v in c]


def philox_words(seed, j0, j1, c1, c2, c3):
    """The word of each draw index j in [j0, j1) (uint32): word j & 3 of Philox4x32-10({j >> 2, c1, c2, c3}, {lo32(S), hi32(S)})."""
    seed = int(seed) or 666
    g = np.arange(j0 >> 2, ((j1 - 1) >> 2) + 1, dtype=np.uint64)
    words = np.stack(philox4x32_10((g, c1, c2, c3), (seed & 0xFFFFFFFF, seed >> 32)), -1).ravel()
    return words[j0 - 4 * (j0 >> 2):][:j1 - j0]


def dropout_counter(rank, layer, pass_):
    """Counter words 1-3 of the DropoutLayer and weight-noise draws: {lo32(P), hi32(P), L | r << 16}."""
    pass_ = int(pass_)
    return pass_ & 0xFFFFFFFF, pass_ >> 32, int(layer) | (int(rank) << 16)


def keep_bits(words, p):
    """x < floor(p 2^32) of each word, p taken as fp32."""
    return words < np.uint64(math.floor(float(np.float32(p)) * 2.0 ** 32))


def box_muller(x_even, x_odd, q: Quirks = DEFAULT_QUIRKS):
    """float64 normals (z_even, z_odd) of Philox word pairs, from the library's exact u and v."""
    u = ((np.asarray(x_even, np.uint64) >> np.uint64(q.box_muller_u_shift)).astype(np.float64) + 0.5) * 2.0 ** -23
    v = (np.asarray(x_odd, np.uint64) >> np.uint64(q.box_muller_v_shift)).astype(np.float64) * 2.0 ** -24
    r = np.sqrt(-2.0 * np.log(u))
    return r * np.cos(2 * np.pi * v), r * np.sin(2 * np.pi * v)


def normals(words, q: Quirks = DEFAULT_QUIRKS):
    """The float64 normal of each word of whole counters (a multiple of 4 words): pair (x0, x1) -> z0, z1, pair (x2, x3) -> z2, z3."""
    w4 = words.reshape(-1, 4)
    z = np.empty(w4.shape)
    z[:, 0], z[:, 1] = box_muller(w4[:, 0], w4[:, 1], q)
    z[:, 2], z[:, 3] = box_muller(w4[:, 2], w4[:, 3], q)
    return z.ravel()


def fmaf(a, b, c):
    """fp32 fmaf(a, b, c) for fp32 a, c and float64 b: exact in double where a * b fits (uniform draws), one rounding to fp32."""
    return (np.float64(np.float32(a)) * np.asarray(b, np.float64) + np.float64(np.float32(c))).astype(np.float32)


def uniform_fmaf(lower, upper, words):
    """The fp32 uniform of each word: fmaf(upper - lower, (x >> 8) 2^-24, lower), upper - lower in fp32."""
    u = (words >> np.uint64(8)).astype(np.float64) * 2.0 ** -24
    return fmaf(np.float32(upper) - np.float32(lower), u, lower)


# DropoutLayer.Builder(IDropout) (B2G_LAYER_DROPOUT, b2g_dropout_kind), with the retain probability p, GaussianDropout's rate or GaussianNoise's
# stddev, each taken as fp32; inference and a FrozenLayer are the identity.  Element e = ((row*h + y)*w + x)*c + ch (its NHWC index in the
# pass) draws with j = e, SpatialDropout's (row, channel) with j = row * C + ch:
#   dropout          y = x * m,  m = keep / p                          dx = dy * m
#   gaussian_dropout y = x * m,  m = 1 + sqrt(rate / (1 - rate)) z     dx = dy * m
#   gaussian_noise   y = x + stddev z                                  dx = dy
#   alpha_dropout    y = a (keep ? x : alpha') + b                     dx = dy * keep * a   (alpha_coefficients)
#   spatial_dropout  the dropout of each whole [H, W] map
DROPOUT_KINDS = ("dropout", "gaussian_dropout", "gaussian_noise", "alpha_dropout", "spatial_dropout")
VALUE_KEY = {"dropout": "p", "gaussian_dropout": "rate", "gaussian_noise": "stddev", "alpha_dropout": "p", "spatial_dropout": "p"}


def dropout_mask(seed, rank, layer, pass_, rows, h, w, c, p, row0=0):
    """Keep mask of a DropoutLayer (True = kept) for rows [row0, row0 + rows) of pass `pass_`, returned NCHW [rows, c, h, w]; all kept at
    p >= 1."""
    per = h * w * c
    e0, e1 = row0 * per, (row0 + rows) * per
    if np.float32(p) >= 1:
        keep = np.ones(e1 - e0, bool)
    else:
        keep = keep_bits(philox_words(seed, e0, e1, *dropout_counter(rank, layer, pass_)), p)
    return keep.reshape(rows, h, w, c).transpose(0, 3, 1, 2)


def dropout_normals(seed, rank, layer, pass_, rows, h, w, c, row0=0, q: Quirks = DEFAULT_QUIRKS):
    """The normal z of each element of rows [row0, row0 + rows) of pass `pass_`, in float64, NCHW [rows, c, h, w]."""
    per = h * w * c
    e0, e1 = row0 * per, (row0 + rows) * per
    g0 = e0 >> 2
    z = normals(philox_words(seed, 4 * g0, 4 * (((e1 - 1) >> 2) + 1), *dropout_counter(rank, layer, pass_)), q)
    return z[e0 - 4 * g0:][:e1 - e0].reshape(rows, h, w, c).transpose(0, 3, 1, 2)


def spatial_mask(seed, rank, layer, pass_, rows, c, p, row0=0):
    """SpatialDropout's keep bit of each (row, channel) of rows [row0, row0 + rows), [rows, c]."""
    if np.float32(p) >= 1:
        return np.ones((rows, c), bool)
    return keep_bits(philox_words(seed, row0 * c, (row0 + rows) * c, *dropout_counter(rank, layer, pass_)), p).reshape(rows, c)


def clamp_value(kind, v) -> np.float32:
    """A scheduled value clamped into its kind's range (the library's documented deviation): rate to [0, 1 - 2^-24], stddev to >= 0, p to
    [2^-32, 1]."""
    v = np.float32(v)
    if kind == "gaussian_dropout":
        return np.float32(min(max(v, np.float32(0)), np.float32(1 - 2.0 ** -24)))
    if kind == "gaussian_noise":
        return np.float32(max(v, np.float32(0)))
    return np.float32(min(max(v, np.float32(2.0 ** -32)), np.float32(1)))


def gaussian_sigma(rate) -> np.float32:
    """GaussianDropout's stddev sqrt(rate / (1 - rate)), in double from the fp32 rate, rounded to fp32 once."""
    r = float(np.float32(rate))
    return np.float32(math.sqrt(r / (1.0 - r)))


def alpha_coefficients(p):
    """AlphaDropout's (a, b, alpha') for the fp32 retain probability p: alpha' = -lambda alpha (SELU's constants),
    a = 1 / sqrt(p + alpha'^2 p (1 - p)), b = -a (1 - p) alpha', each in double and rounded to fp32 once."""
    p = float(np.float32(p))
    ap = -SELU_LAMBDA * SELU_ALPHA
    a = 1.0 / math.sqrt(p + ap * ap * p * (1.0 - p))
    return np.float32(a), np.float32(-a * (1.0 - p) * ap), np.float32(ap)


class DropoutState:
    """The draw inputs a net's DropoutLayers and noisy layers share: seed (the library's b2g_net_config.seed), rank, pass counter P, explicit
    draws.  Like the library, the last stochastic DropoutLayer of a train-mode forward advances P once it has drawn (weight noise does when the
    pass has no such layer); `queue` holds explicit (pass, first row) draws that replace the counter for the next forwards without advancing
    it.  `net`: the owning Net; `lead`: None, or the Net whose counters the next passes read their scheduled values at (gan_step's G pass
    through D reads G's)."""

    def __init__(self, seed=666, rank=0, net=None):
        self.seed, self.rank, self.pass_, self.queue, self.net, self.lead = seed, rank, 0, [], net, None

    def counters(self):
        """The (iteration, epoch) a pass reads scheduled dropout values and DropConnect p at: the lead's, else the owning net's, else (0, 0)."""
        net = self.lead if self.lead is not None else self.net
        return (net.iteration, net.epoch) if net is not None else (0, 0)

    def current(self):
        return self.queue[0] if self.queue else (self.pass_, 0)

    def finish(self):          # end of a stochastic train-mode forward
        if self.queue:
            self.queue.pop(0)
        else:
            self.pass_ += 1


class Dropout(Layer):
    """DropoutLayer.Builder(IDropout): `kind` one of DROPOUT_KINDS with its value (VALUE_KEY: p, rate or stddev) and an optional schedule of
    it.  A Net shares its DropoutState among its DropoutLayers.  Train mode draws from that state; the identity cases (p = 1, rate = 0 or
    stddev = 0 without a schedule, frozen, inference) draw nothing and count no pass."""

    def __init__(self, value, name="", index=0, state=None, frozen=False, kind="dropout", schedule=None):
        assert kind in DROPOUT_KINDS, kind
        self.value, self.name, self.index, self.state, self.frozen = float(np.float32(value)), name, index, state, frozen
        self.kind, self.schedule, self.last, self._m = kind, schedule, False, None

    def active(self):
        if self.frozen:
            return False
        if self.schedule is not None:          # a scheduled layer is stochastic whatever its value
            return True
        return self.value > 0 if self.kind in ("gaussian_dropout", "gaussian_noise") else self.value < 1

    def value_at(self, iteration, epoch) -> float:
        """The value a train-mode pass at (iteration, epoch) uses: the schedule's fp32 value clamped into the kind's range, or the constant."""
        if self.schedule is None:
            return self.value
        return float(clamp_value(self.kind, lr_at(self.schedule, iteration, epoch)))

    def forward(self, x, train):
        self._m = None
        if not train or not self.active():
            return x
        value = self.value_at(*self.state.counters())
        pass_, row0 = self.state.current()
        _, c, h, w = x.shape if x.ndim == 4 else (x.shape[0], x.shape[1], 1, 1)
        args = (self.state.seed, self.state.rank, self.index, pass_, x.shape[0])
        t = x.dtype.type
        if self.kind == "dropout":
            keep = dropout_mask(*args, h, w, c, value, row0).reshape(x.shape)
            self._m = keep * t(np.float32(1) / np.float32(value)); y = x * self._m
        elif self.kind in ("gaussian_noise", "gaussian_dropout"):
            z = dropout_normals(*args, h, w, c, row0, self.q).reshape(x.shape)
            if self.kind == "gaussian_noise":
                y = x + t(np.float32(value)) * z
            else:
                self._m = 1 + t(gaussian_sigma(value)) * z; y = x * self._m
        elif self.kind == "alpha_dropout":
            keep = dropout_mask(*args, h, w, c, value, row0).reshape(x.shape)
            a, b, ap = (t(v) for v in alpha_coefficients(value))
            self._m = keep * a; y = a * np.where(keep, x, ap) + b
        else:
            if x.ndim != 4 or h * w == 1:
                raise ValueError("SpatialDropout needs a [N, C, H, W] input")
            keep = spatial_mask(*args[:4], x.shape[0], c, value, row0)[:, :, None, None]
            self._m = np.broadcast_to(keep * t(np.float32(1) / np.float32(value)), x.shape); y = x * self._m
        if self.last:
            self.state.finish()
        return y

    def backward(self, eps):
        return eps if self._m is None else eps * self._m


# Weight noise (b2g_weight_noise: DL4J's DropConnect and WeightNoise) on a conv, deconv or dense layer's `weight_noise` dict.  A train-mode
# pass draws W' (and b' with apply_to_bias) of every noisy layer once at its top (Net.forward), from the clean parameters in the net's dtype;
# that layer's forward and input gradient run on them, and its weight and bias gradients are taken straight through.  The draw index j is the
# element's index in the library's internal [A][taps][B] order (internal_w), b's from bias_j0 on:
#   DropConnect   W' = keep ? W : 0                     WeightNoise   n = NORMAL fmaf(std, z, mean) or UNIFORM (uniform_fmaf);
#                                                                     W' = W + n (additive) or W * n
def internal_w(W):
    """W (DL4J's shape) in the library's internal [A][taps][B] order, flattened: conv [nOut][kH*kW][nIn], transposed conv [nIn][kH*kW][nOut],
    dense [nOut][nIn]."""
    W = np.asarray(W)
    if W.ndim == 2:
        return W.T.ravel()
    return W.reshape(W.shape[0], W.shape[1], -1).transpose(0, 2, 1).ravel()


def dl4j_w(flat, shape):
    """The inverse of internal_w: the internal order back to W's shape."""
    flat = np.asarray(flat)
    if len(shape) == 2:
        return flat.reshape(shape[1], shape[0]).T
    return flat.reshape(shape[0], -1, shape[1]).transpose(0, 2, 1).reshape(shape)


def bias_j0(n_w: int) -> int:
    """Draw index of bias element 0: 4 * ceil(n_W / 4), so W and b never share a Philox counter."""
    return 4 * ((n_w + 3) // 4)


def drop_connect_p(wn, counters=(0, 0)) -> np.float32:
    """DropConnect's retain probability of a pass: the constant, or the schedule's fp32 value at the pass's (iteration, epoch) clamped to
    [2^-32, 1]."""
    p = wn["p"]
    if isinstance(p, dict):
        return clamp_value("dropout", lr_at(p, *counters))
    return np.float32(p)


def weight_noise_draw(wn, n, j0, seed, rank, layer, pass_, p=None, q: Quirks = DEFAULT_QUIRKS):
    """The draws of n elements with indices j0 .. j0 + n - 1 (j0 a multiple of 4): DropConnect's keep bits (bool), or WeightNoise's noise in
    fp32."""
    assert j0 % 4 == 0
    words = philox_words(seed, j0, ((j0 + n + 3) // 4) * 4, *dropout_counter(rank, layer, pass_))
    if wn["weight_noise"] == "drop_connect":
        if np.float32(p) >= 1:
            return np.ones(n, bool)
        return keep_bits(words[:n], p)
    d = wn["distribution"]
    if d["distribution"] == "normal":
        return fmaf(d["std"], normals(words, q)[:n], d["mean"])
    return uniform_fmaf(d["lower"], d["upper"], words[:n])


def weight_noise_apply(wn, w, d, p=None, q: Quirks = DEFAULT_QUIRKS):
    """W' from the clean values w and the draws d, in w's dtype (float32: the library's fp32 operand, each result rounded once)."""
    t = w.dtype.type
    if wn["weight_noise"] == "drop_connect":
        kept = w / t(np.float32(p)) if q.dropconnect_inverted else w
        return np.where(d, kept, t(0))
    n = d.astype(w.dtype)
    return (w + n if wn.get("additive", True) else w * n).astype(w.dtype)


def noisy_operands(layer, wn, index, seed, rank, pass_, counters=(0, 0), dtype=np.float32, q: Quirks = DEFAULT_QUIRKS):
    """(W' in the internal order, b' or None) of one layer for pass `pass_`, from its parameters taken as `dtype`."""
    p = drop_connect_p(wn, counters) if wn["weight_noise"] == "drop_connect" else None
    w = internal_w(layer.params["W"]).astype(dtype)
    w_n = weight_noise_apply(wn, w, weight_noise_draw(wn, w.size, 0, seed, rank, index, pass_, p, q), p, q)
    b_n = None
    if wn.get("apply_to_bias", False) and getattr(layer, "has_bias", False):
        b = np.asarray(layer.params["b"]).astype(dtype)
        b_n = weight_noise_apply(wn, b, weight_noise_draw(wn, b.size, bias_j0(w.size), seed, rank, index, pass_, p, q), p, q)
    return w_n, b_n


def weight_noise_active(layer) -> bool:
    """A layer whose train-mode passes draw: it has weight noise, is not frozen, and is not a constant DropConnect(1)."""
    wn = layer.weight_noise
    if wn is None or getattr(layer, "frozen", False):
        return False
    return wn["weight_noise"] != "drop_connect" or isinstance(wn["p"], dict) or np.float32(wn["p"]) < 1


# Weight initialization (b2g_weight_init: DL4J's WeightInit, Distribution and biasInit), each scheme's distribution from the layer's fans().
# The draw: L = the layer's index in the library's desc array, j = the element's index in DL4J's view order of W (b2g_net_get_param's);
# round k draws from counter {j >> 2, k, 0, L | 2^31}.  NORMAL: fmaf(std, z, mean), z of round 0's Box-Muller pairs (float64 here; the
# device's is fp32, so normal draws agree within its tolerance).  UNIFORM: uniform_fmaf.  TRUNCATED_NORMAL: z of the first round k < 16 with
# |z| <= truncation_sigmas, else round 15's z clamped.  LOG_NORMAL: exp of the NORMAL value.  BINOMIAL: the count over rounds t < nTrials of
# keep_bits(x_t, p).  CONSTANT, ZERO, ONES, IDENTITY: no draw.
SCHEMES = ("distribution", "zero", "ones", "sigmoid_uniform", "normal", "lecun_normal", "uniform", "xavier", "xavier_uniform", "xavier_fan_in",
           "xavier_legacy", "relu", "relu_uniform", "identity", "lecun_uniform", "var_scaling_normal_fan_in", "var_scaling_normal_fan_out",
           "var_scaling_normal_fan_avg", "var_scaling_uniform_fan_in", "var_scaling_uniform_fan_out", "var_scaling_uniform_fan_avg")
DISTRIBUTIONS = ("normal", "uniform", "truncated_normal", "log_normal", "binomial", "constant", "orthogonal")
WEIGHT_INIT_ROUNDS = 16


def resolve(wi, layer, q: Quirks = DEFAULT_QUIRKS):
    """What the scheme draws on the layer: (kind, a, b) with kind a distribution name or "identity"; a, b fp32, each computed in double and
    rounded once (binomial: (nTrials, p))."""
    scheme = wi["weight_init"]
    fi, fo = (float(v) for v in layer.fans())
    N = lambda sd: ("normal", np.float32(0), np.float32(sd))
    U = lambda r: ("uniform", -np.float32(r), np.float32(r))
    T = lambda sd: ("truncated_normal", np.float32(0), np.float32(sd))
    u3 = lambda fan: 3.0 / math.sqrt(fan) if q.var_scaling_uniform_three_over_sqrt else math.sqrt(3.0 / fan)
    if scheme == "distribution":
        d = wi["distribution"]
        kind = d["distribution"]
        if kind in ("normal", "truncated_normal", "log_normal"):
            return kind, np.float32(d["mean"]), np.float32(d["std"])
        if kind == "uniform":
            return kind, np.float32(d["lower"]), np.float32(d["upper"])
        if kind == "binomial":
            return kind, int(d["n_trials"]), np.float32(d["p"])
        if kind == "constant":
            return kind, np.float32(d["value"]), np.float32(0)
        raise ValueError(kind)
    table = {
        "zero": lambda: ("constant", np.float32(0), np.float32(0)),
        "ones": lambda: ("constant", np.float32(1), np.float32(0)),
        "sigmoid_uniform": lambda: U(4.0 * math.sqrt(6.0 / (fi + fo))),
        "normal": lambda: N(1.0 / math.sqrt(fi) if q.normal_scaled_by_fan_in else 1.0),
        "lecun_normal": lambda: N(1.0 / math.sqrt(fi)),
        "uniform": lambda: U(1.0 / math.sqrt(fi)),
        "xavier": lambda: N(math.sqrt(2.0 / (fi + fo))),
        "xavier_uniform": lambda: U(math.sqrt(6.0) / math.sqrt(fi + fo)),
        "xavier_fan_in": lambda: N(1.0 / math.sqrt(fi)),
        "xavier_legacy": lambda: N(1.0 / math.sqrt(layer.n_in + layer.n_out) if q.xavier_legacy_shape01 else 1.0 / math.sqrt(fi + fo)),
        "relu": lambda: N(math.sqrt(2.0 / fi)),
        "relu_uniform": lambda: U(math.sqrt(6.0 / fi)),
        "identity": lambda: ("identity", np.float32(0), np.float32(0)),
        "lecun_uniform": lambda: U(3.0 / math.sqrt(fi) if q.lecun_uniform_three_over_sqrt else math.sqrt(3.0 / fi)),
        "var_scaling_normal_fan_in": lambda: T(math.sqrt(1.0 / fi)),
        "var_scaling_normal_fan_out": lambda: T(math.sqrt(1.0 / fo)),
        "var_scaling_normal_fan_avg": lambda: T(math.sqrt(2.0 / (fi + fo))),
        "var_scaling_uniform_fan_in": lambda: U(u3(fi)),
        "var_scaling_uniform_fan_out": lambda: U(u3(fo)),
        "var_scaling_uniform_fan_avg": lambda: U(u3((fi + fo) / 2.0)),
    }
    return table[scheme]()


def weight_init_words(seed, layer_index, n, k):
    """Round k's Philox word of every view index j < n."""
    return philox_words(seed, 0, n, int(k), 0, int(layer_index) | WEIGHT_INIT_TAG)


def weight_init_normals(seed, layer_index, n, k=0, q: Quirks = DEFAULT_QUIRKS):
    """Round k's float64 normal of every view index j < n (a tail element's pair partner exists past n)."""
    return normals(weight_init_words(seed, layer_index, 4 * ((n + 3) // 4), k), q)[:n]


def truncated_z(seed, layer_index, n, q: Quirks = DEFAULT_QUIRKS):
    """The z of the first round k < 16 with |z| <= the truncation, else round 15's z clamped."""
    lim = q.truncation_sigmas
    z = np.zeros(n)
    todo = np.ones(n, bool)
    for k in range(WEIGHT_INIT_ROUNDS):
        t = weight_init_normals(seed, layer_index, n, k, q)
        hit = todo & (np.abs(t) <= lim)
        z[hit] = t[hit]
        todo &= ~hit
        if k == WEIGHT_INIT_ROUNDS - 1:
            z[todo] = np.clip(t[todo], -lim, lim)
        if not todo.any():
            break
    return z


def weight_init_draw(kind, a, b, n, seed, layer_index, n_in=None, q: Quirks = DEFAULT_QUIRKS):
    """n fp32 values in view order.  identity: n_in = nIn of the square dense W (view index j = o nIn + i)."""
    if kind == "normal":
        return fmaf(b, weight_init_normals(seed, layer_index, n, 0, q), a)
    if kind == "log_normal":
        return np.exp(fmaf(b, weight_init_normals(seed, layer_index, n, 0, q), a).astype(np.float64)).astype(np.float32)
    if kind == "truncated_normal":
        return fmaf(b, truncated_z(seed, layer_index, n, q), a)
    if kind == "uniform":
        return uniform_fmaf(a, b, weight_init_words(seed, layer_index, n, 0))
    if kind == "binomial":
        c = np.zeros(n, np.int64)
        for t in range(int(a)):
            c += keep_bits(weight_init_words(seed, layer_index, n, t), b)
        return c.astype(np.float32)
    if kind == "constant":
        return np.full(n, np.float32(a), np.float32)
    if kind == "identity":
        j = np.arange(n)
        return (j // n_in == j % n_in).astype(np.float32)
    raise ValueError(kind)


def weights(wi, layer, seed, layer_index, q: Quirks = DEFAULT_QUIRKS):
    """W of a conv, deconv or dense layer in DL4J's flattened view order (b2g_net_get_param's), fp32."""
    kind, a, b = resolve(wi, layer, q)
    if kind == "identity" and (not isinstance(layer, Dense) or layer.n_in != layer.n_out):
        raise ValueError("IDENTITY needs a square dense W")
    n = layer.n_in * layer.n_out * int(np.prod(getattr(layer, "k", (1, 1))))
    return weight_init_draw(kind, a, b, n, seed, layer_index, layer.n_in, q)


def init_layer(layer, wi, seed, layer_index, q: Quirks = DEFAULT_QUIRKS):
    """The layer's W and b (if it has one) as b2g_net_init_weights leaves them, in the layer's dtype."""
    flat = weights(wi, layer, seed, layer_index, q)
    order = next(o for p, _, o in layer.param_specs() if p == "W")
    W = layer.params["W"]
    layer.params["W"] = flat.astype(W.dtype).reshape(W.shape, order=order.upper())
    if "b" in layer.params:
        layer.params["b"] = np.full(layer.params["b"].shape, np.float32(wi.get("bias_init", 0.0)), layer.params["b"].dtype)
    return layer


def xent_score_and_grad(z: np.ndarray, y: np.ndarray, clip_eps: float, s=None):
    """LossBinaryXENT with a sigmoid activation (J:159-163).  Returns (sum of per-example losses, dL/dz); s: the per-element weight and mask
    product both are scaled by (None: unweighted).

    clip_eps > 0: p = clip(sigmoid(z), eps, 1-eps); grad = (p-y)/(p(1-p)) * sigmoid'(z)   (DL4J-exact)
    clip_eps = 0: BCE-with-logits (north_star): loss = softplus(z) - y z; grad = sigmoid(z) - y.
    """
    if clip_eps > 0:
        sg = _sigmoid(z)
        p = np.clip(sg, clip_eps, 1 - clip_eps)
        loss = -(y * np.log(p) + (1 - y) * np.log(1 - p))
        grad = (p - y) / (p * (1 - p)) * sg * (1 - sg)
    else:
        loss = np.maximum(z, 0) + np.log1p(np.exp(-np.abs(z))) - y * z
        grad = _sigmoid(z) - y
    if s is None:
        return loss.sum(), grad
    return float((loss * s).sum()), grad * s


# Regression and margin losses (b2g_loss codes 2-8; org.nd4j.linalg.lossfunctions.impl.*).  Each is ILossFunction.computeGradient(labels,
# preOutput, activationFn): a = act(z), dL/dz = dL/da * act'(a) with the derivative taken from the output a, per-example scores summed over
# the nOut outputs:
#   mse            sum (a-y)^2 / nOut          2(a-y) / nOut
#   l1             sum |a-y|                   sign(a-y)              (sign(0) = 0)
#   l2             sum (a-y)^2                 2(a-y)
#   mae            sum |a-y| / nOut            sign(a-y) / nOut
#   hinge          sum max(0, 1 - y a)         -y where 1 - y a > 0 (strictly), else 0
#   squared_hinge  sum max(0, 1 - y a)^2       -2y max(0, 1 - y a)
#   wasserstein    sum y a / nOut              y / nOut               (the / nOut: Quirks.wasserstein_per_output)
# On an activation of codes 5-16 the loss takes a = f(z) with the identity and multiplies dL/da by f'(z).
LOSSES = ("mse", "l1", "l2", "mae", "hinge", "squared_hinge", "wasserstein")
LOSS_CODES = {"mse": 2, "l1": 3, "l2": 4, "mae": 5, "hinge": 6, "squared_hinge": 7, "wasserstein": 8}


def act_grad_from_out(act: str, a: np.ndarray, alpha: float = 0.01) -> np.ndarray:
    """f'(z) from the output a = f(z), as the library's act_grad_from_out takes it (LeakyReLU: sign(a) = sign(z) for alpha > 0)."""
    if act == "identity":
        return np.ones_like(a)
    if act == "tanh":
        return 1 - a * a
    if act == "sigmoid":
        return a * (1 - a)
    if act == "relu":
        return (a > 0).astype(a.dtype)
    if act == "lrelu":
        return np.where(a > 0, 1.0, alpha).astype(a.dtype)
    raise ValueError(act)


def per_output(loss: str, q: Quirks = DEFAULT_QUIRKS) -> bool:
    """Whether the loss divides its score and gradient by nOut."""
    return loss in ("mse", "mae") or (loss == "wasserstein" and q.wasserstein_per_output)


def _elem_score_and_grad(loss, act, alpha, z, y, q):
    """The per-element scores (before the / nOut of the per-output losses) and dL/dz of a loss of codes 2-8."""
    if act in EXT_ACTS:
        l, g = _elem_score_and_grad(loss, "identity", 0.0, forward(act, z, alpha, q), y, q)
        return l, g * derivative(act, z, alpha, q)
    a = act_forward(act, z, alpha)
    e, m = a - y, 1 - y * a
    if loss in ("mse", "l2"):
        l, g = e * e, 2 * e
    elif loss in ("l1", "mae"):
        l, g = np.abs(e), np.sign(e)
    elif loss == "hinge":
        l, g = np.maximum(m, 0), np.where(m > 0, -y, 0.0)
    elif loss == "squared_hinge":
        l, g = np.maximum(m, 0) ** 2, -2 * y * np.maximum(m, 0)
    elif loss == "wasserstein":
        l, g = y * a, y * np.ones_like(a)
    else:
        raise ValueError(loss)
    if per_output(loss, q):
        g = g / z.shape[1]
    return l, g * act_grad_from_out(act, a, alpha)


def score_and_grad(loss: str, act: str, alpha: float, z: np.ndarray, y: np.ndarray, q: Quirks = DEFAULT_QUIRKS, s=None):
    """z, y: [N, nOut].  Returns (sum over the N examples of the per-example scores, dL/dz [N, nOut]); s: the per-element weight and mask
    product both are scaled by (None: unweighted)."""
    l, g = _elem_score_and_grad(loss, act, alpha, z, y, q)
    score = l.sum() if s is None else (l * s).sum()
    if per_output(loss, q):
        score = score / z.shape[1]
    return float(score), g if s is None else g * s


# Per-output loss weights w_j and labels masks m_rj (semantics at b2g_loss).  For row r (an example, or a pixel of a CnnLossLayer) and
# column j (an output, or a channel):
#   XENT, codes 2-8   score terms w_j m_rj l(a_rj, y_rj), dz_rj = w_j m_rj dz_rj
#   MCXENT            score -m_r sum_j w_j y_rj log clamp(p_rj), dz_rj = m_r (p_rj sum_k w_k y_rk - w_j y_rj) (weighted), m_r (p_rj - y_rj)
# The score stays the loss sum over the minibatch; MSE, MAE and Wasserstein still divide by nOut / C.  A mask is [N, 1] or [N, nOut] on
# OUTPUT / LOSS layers and NCHW [N, 1, H, W] or [N, C, H, W] on a CnnLossLayer.
def check_weights(loss, weights, cols, q: Quirks = DEFAULT_QUIRKS):
    """The loss weights as float64 [cols] (None stays None), refused as the library refuses them."""
    if weights is None:
        return None
    w = np.asarray(weights, np.float64).ravel()
    if loss in q.weightless_losses:
        raise NotImplementedError(f"{loss} takes no per-output weights")
    if w.size != cols:
        raise ValueError(f"{w.size} loss weights for {cols} outputs")
    if not np.all(np.isfinite(w)):
        raise ValueError("loss weights must be finite")
    return w


def check_mask(loss, mask, rows, cols, q: Quirks = DEFAULT_QUIRKS):
    """The mask as float64 rows: [rows, 1] or [rows, cols] (None stays None)."""
    if mask is None:
        return None
    m = np.asarray(mask, np.float64).reshape(rows, -1)
    if m.shape[1] not in (1, cols):
        raise ValueError(f"mask width {m.shape[1]}: 1 or {cols}")
    if m.shape[1] > 1 and loss == "mcxent" and q.mcxent_per_output_mask_refused:
        raise NotImplementedError("per-output masking for MCXENT + softmax is not supported")
    return m


def loss_scale(z, w, m):
    """The per-element product of the weights w [C] and the mask m [R, 1 | C] on rows z [R, C]; None when both are absent."""
    if w is None and m is None:
        return None
    s = np.ones_like(z)
    if w is not None:
        s = s * w[None, :]
    if m is not None:
        s = s * m
    return s


def rows_score_and_grad(loss, act, alpha, z, y, w=None, m=None, q: Quirks = DEFAULT_QUIRKS):
    """The loss on rows z, y [R, C], weighted by w [C] and masked by m [R, 1 | C] (None: that part absent): (summed score, dL/dz [R, C])."""
    if loss == "mcxent":
        return mcxent_softmax_score_and_grad(z, y, w=w, m=m)
    s = loss_scale(z, w, m)
    if loss == "xent":
        return xent_score_and_grad(z, y, q.xent_clip_eps, s)
    return score_and_grad(loss, act, alpha, z, y, q, s)


def _score_and_eps(layer, loss, y, weights, mask):
    """(summed score, dL/dz) of an OutputLayer or LossLayer on its pre-activations as [N, nOut] rows."""
    z = layer._z
    y = np.asarray(y, z.dtype)
    zr = z.reshape(y.shape)
    w, m = check_weights(loss, weights, zr.shape[1], layer.q), check_mask(loss, mask, zr.shape[0], zr.shape[1], layer.q)
    s, g = rows_score_and_grad(loss, layer.loss_act, layer.loss_alpha, zr, y, w, m, layer.q)
    return s, g.reshape(z.shape)


class LossLayer(Layer):
    """o.d.nn.conf.layers.LossLayer(loss, activation): the loss on activation(incoming pre-activations), no parameters.  XENT is on the
    sigmoid.  Accepts [N,nOut] or [N,nOut,1,1] (DCGAN D-last conv emits the logit)."""

    def __init__(self, name="", quirks: Optional[Quirks] = None, loss="xent", activation="identity", alpha=0.01):
        self.name, self.loss, self.loss_alpha = name, loss, alpha
        if quirks is not None:
            self.q = quirks
        self.loss_act = "sigmoid" if loss == "xent" else activation

    def forward(self, x, train):
        self._z = x
        return _layer_act_forward(self.loss_act, x, self.loss_alpha, self.q)

    def score_and_eps(self, y, weights=None, mask=None):
        """(summed score, dL/dz) on labels y, with per-output weights and a labels mask (None: that part absent)."""
        return _score_and_eps(self, self.loss, y, weights, mask)


def to_rows(a):
    """[N, C, H, W] -> [N*H*W, C] (pixel-major, channel-minor: the engine's NHWC buffer)."""
    return np.ascontiguousarray(np.moveaxis(a, 1, -1)).reshape(-1, a.shape[1])


def from_rows(r, shape):
    n, c, h, w = shape
    return np.ascontiguousarray(r.reshape(n, h, w, c).transpose(0, 3, 1, 2))


def softmax_channels(z):
    """The softmax over dimension 1: the classes of [N, C] rows, the channels of each pixel of an [N, C, H, W] map."""
    e = np.exp(z - z.max(1, keepdims=True))
    return e / e.sum(1, keepdims=True)


class CnnLossLayer(LossLayer):
    """CnnLossLayer.Builder(loss).activation(act) (B2G_LAYER_CNN_LOSS): no parameters.  The [N, C, H, W] map becomes [N*H*W, C] rows
    (reshape4dTo2d), each row takes the loss of LossLayer / Output, and the score is summed over the rows.  forward returns the activated map
    (sigmoid for XENT, the per-pixel softmax over the channels for MCXENT, act otherwise).  The score's divisor, the minibatch rather than the
    pixel count, is a medium-confidence recall behind Quirks.cnn_loss_score_per_minibatch."""

    def __init__(self, name="", quirks: Optional[Quirks] = None, loss="xent", activation="identity", alpha=0.01):
        super().__init__(name, quirks, loss, activation, alpha)
        if loss == "mcxent":
            self.loss_act = "softmax"

    def forward(self, x, train):
        x = np.asarray(x)
        if x.ndim == 2:                       # a feed-forward input is the 1x1 map
            x = x.reshape(x.shape + (1, 1))
        self._z = x
        if self.loss == "mcxent":
            return softmax_channels(x)
        return _layer_act_forward(self.loss_act, x, self.loss_alpha, self.q)

    def score_and_eps(self, y, weights=None, mask=None):
        z = self._z
        n, c, h, w = z.shape
        zr, yr = to_rows(z), to_rows(np.asarray(y, z.dtype).reshape(z.shape))
        if mask is not None:
            mask = np.asarray(mask, np.float64).reshape(n, -1, h, w)
            if mask.shape[1] not in (1, c):
                raise ValueError(f"mask channels {mask.shape[1]}: 1 or {c}")
            mask = to_rows(mask)
        wt, m = check_weights(self.loss, weights, c, self.q), check_mask(self.loss, mask, zr.shape[0], c, self.q)
        s, g = rows_score_and_grad(self.loss, self.loss_act, self.loss_alpha, zr, yr, wt, m, self.q)
        g = from_rows(g, z.shape)
        if not self.q.cnn_loss_score_per_minibatch:
            hw = z.shape[2] * z.shape[3]
            s, g = s / hw, g / hw
        return float(s), g


class Output(Dense):
    """OutputLayer.Builder(loss).activation(act).nOut(n) = Dense + the loss on act(z); XENT is on the sigmoid (J:159-163)."""

    def __init__(self, n_in, n_out, updater=None, l2=0.0, name="", quirks: Optional[Quirks] = None, loss="xent", activation="identity",
                 alpha=0.01):
        super().__init__(n_in, n_out, activation="identity", updater=updater, l2=l2, name=name)
        if quirks is not None:
            self.q = quirks
        self.loss, self.loss_alpha = loss, alpha
        self.loss_act = "sigmoid" if loss == "xent" else activation

    def forward(self, x, train):
        z = super().forward(x, train)          # the identity Dense: z; the loss applies the activation
        return _layer_act_forward(self.loss_act, z, self.loss_alpha, self.q)

    def score_and_eps(self, y, weights=None, mask=None):
        return _score_and_eps(self, self.loss, y, weights, mask)

    def backward(self, eps):   # eps is already dL/dz
        self.grads["W"] = self._x.T @ eps
        self.grads["b"] = eps.sum(0)
        return eps @ self._p("W").T


def mcxent_softmax_score_and_grad(z: np.ndarray, y: np.ndarray, clip_eps: float = 1e-10, w=None, m=None):
    """LossMCXENT with a softmax activation (J:357-362): p = softmax(z) clipped to [eps, 1-eps] for the log
    (softmaxClipEps default 1e-10); loss = -sum y log p; dL/dz = p - y (DL4J's softmax+MCXENT shortcut).  w [C], m [R, 1]: the class
    weights and the row mask (None: absent)."""
    zs = z - z.max(1, keepdims=True)
    e = np.exp(zs)
    p = e / e.sum(1, keepdims=True)
    pc = np.clip(p, clip_eps, 1 - clip_eps) if clip_eps > 0 else p
    s = loss_scale(z, w, m)
    if s is None:
        return float(-(y * np.log(pc)).sum()), p - y
    mr = m if m is not None else 1.0
    if w is not None:
        wy = w[None, :] * y
        return float(-((y * np.log(pc)) * s).sum()), mr * (p * wy.sum(1, keepdims=True) - wy)
    return float(-((y * np.log(pc)) * s).sum()), mr * (p - y)


class OutputSoftmax(Dense):
    """OutputLayer.Builder(LossFunction.MCXENT).activation(Activation.SOFTMAX).nOut(10) (J:357-362): the transfer-learning head."""

    loss, loss_act, loss_alpha = "mcxent", "softmax", None

    def __init__(self, n_in, n_out, updater=None, l2=0.0, name=""):
        super().__init__(n_in, n_out, activation="identity", updater=updater, l2=l2, name=name)

    def forward(self, x, train):
        return softmax_channels(super().forward(x, train))

    def score_and_eps(self, y, weights=None, mask=None):
        return _score_and_eps(self, self.loss, y, weights, mask)

    def backward(self, eps):
        self.grads["W"] = self._x.T @ eps
        self.grads["b"] = eps.sum(0)
        return eps @ self._p("W").T


# --------------------------------------------------------------------------------------------------
# Graph vertices (B2G_LAYER_ELEMENTWISE / B2G_LAYER_MERGE, semantics at b2g_elementwise_op in include/b200gan.h).  A vertex reads the
# spine (the layer before it) and the output of an earlier layer, its skip source `src` (an index into the Net's layers).  order 0: the
# inputs are (spine, skip); order 1: (skip, spine).  forward(x_spine, x_skip, train); backward(eps) -> (eps_spine, eps_skip).
# --------------------------------------------------------------------------------------------------
EW_OPS = ("add", "subtract", "product", "average", "max")


def ew_forward(op, a, b):
    if op == "add":
        return a + b
    if op == "subtract":
        return a - b
    if op == "product":
        return a * b
    if op == "average":
        return (a + b) * 0.5
    return np.where(a >= b, a, b)           # a tie takes the first input


def ew_backward(op, e, a, b):
    """(dL/da, dL/db) of ew_forward; MAX sends e to the larger input, a tie to the first."""
    if op == "add":
        return e, e
    if op == "subtract":
        return e, -e
    if op == "product":
        return e * b, e * a
    if op == "average":
        return e * 0.5, e * 0.5
    first = a >= b
    return np.where(first, e, 0.0), np.where(first, 0.0, e)


class Vertex(Layer):
    def __init__(self, src, order, name=""):
        self.src, self.order, self.name = src, order, name

    def out_shape(self, s, s_skip):
        return s


class ElementWiseVertex(Vertex):
    """new ElementWiseVertex(op): no parameters."""

    def __init__(self, op, src, order, name=""):
        if op not in EW_OPS:
            raise ValueError(op)
        super().__init__(src, order, name)
        self.op = op

    def forward(self, x, skip, train):
        self._a, self._b = (x, skip) if self.order == 0 else (skip, x)
        return ew_forward(self.op, self._a, self._b)

    def backward(self, eps):
        da, db = ew_backward(self.op, eps, self._a, self._b)
        return (da, db) if self.order == 0 else (db, da)


class MergeVertex(Vertex):
    """new MergeVertex(): the inputs concatenated along dimension 1 in input order; no parameters."""

    def out_shape(self, s, s_skip):
        return (s[0], s[1] + s_skip[1]) + tuple(s[2:])

    def forward(self, x, skip, train):
        first, second = (x, skip) if self.order == 0 else (skip, x)
        self._c = first.shape[1]
        return np.concatenate((first, second), axis=1)

    def backward(self, eps):
        first, second = eps[:, :self._c], eps[:, self._c:]
        spine, skip = (first, second) if self.order == 0 else (second, first)
        return np.ascontiguousarray(spine), np.ascontiguousarray(skip)


# --------------------------------------------------------------------------------------------------
# Network = ComputationGraph as a spine plus skip edges: layer i reads layer i-1's output, and a vertex also reads its skip source's.
# (Every graph in the reference is a chain.)  The backward walks the spine in reverse; a vertex leaves the skip input's share of its epsilon
# in the source's accumulator, which joins the spine epsilon when the walk reaches the source.
# --------------------------------------------------------------------------------------------------
class Net:
    """mask_seed, rank: the DropoutLayer masks' seed and rank (the library's b2g_net_config.seed and the replica's rank)."""

    def __init__(self, layers: Sequence[Layer], seed=666, dtype=np.float64, grad_clip: float = 0.0,
                 quirks: Quirks = DEFAULT_QUIRKS, mask_seed=666, rank=0):
        self.layers = list(layers)
        self.dtype = dtype
        self.grad_clip = grad_clip      # ClipElementWiseAbsoluteValue threshold (J:123-124); 0 = off
        self.q = quirks
        self.iteration = self.epoch = 0
        self.gradient_normalization, self.gradient_normalization_threshold, self.grad_norm_last_norms = "none", 1.0, []
        self.schedules: Dict[str, dict] = {}      # layer name -> schedule (None: the constant lr)
        self.layer_constraints: Dict[str, Dict[str, List[Dict]]] = {}     # layer name -> parameter -> its ordered constraints
        self.layer_regularization: Dict[str, Tuple[float, float, float]] = {}     # layer name -> (l1, l1Bias, l2Bias) beside its l2
        self.dropout = DropoutState(mask_seed, rank, self)
        self.loss_weights: Optional[np.ndarray] = None      # the loss layer's per-output weights (None: unweighted)
        self._skip_acc: Dict[int, np.ndarray] = {}    # skip source index -> the skip shares the current backward has met
        rng = np.random.default_rng(seed)
        for l in self.layers:
            if "q" not in vars(l):        # a layer built with its own quirks, or already in a net, keeps them
                l.q = quirks
            l.init(rng, dtype)
        self._link_dropout()
        self.state: Dict[Tuple[int, str], List[np.ndarray]] = {}
        for li, l in enumerate(self.layers):
            if not l.has_params:
                continue
            u = l.updater or UpdaterCfg("sgd", 0.0)
            for pname, shape, _ in l.param_specs():
                if N_STATE[u.kind] and pname not in l.noop_names():
                    self.state[(li, pname)] = init_state(u, shape, dtype, self.q)

    # ---- the library Net's settings ------------------------------------------------------------
    def set_gradient_normalization(self, mode: str, threshold: float = 1.0):
        """DL4J's GradientNormalization (one of GRAD_NORMS) for every layer, from the next update on."""
        assert mode in GRAD_NORMS, mode
        self.gradient_normalization, self.gradient_normalization_threshold = mode, threshold

    def set_lr_schedule(self, schedule: Optional[dict], layer: Optional[str] = None):
        """setLearningRate(ISchedule) (layer None: every layer whose updater has a learning rate) or setLearningRate(layer, ISchedule);
        schedule None = back to the layer's constant lr."""
        if layer is None:
            names = [l.name for l in self.layers if l.has_params and l.updater is not None and l.updater.kind not in ("noop", "adadelta")]
        else:
            names = [layer]
        for name in names:
            self.schedules[name] = schedule

    def learning_rate(self, layer: str) -> float:
        """The learning rate the layer's next update uses: its schedule's fp32 value at the current iteration / epoch, else its constant."""
        l = self.layer(layer)
        return self._lr(l, l.updater)

    def _lr(self, l: Layer, u: UpdaterCfg) -> float:
        sched = self.schedules.get(l.name)
        return float(lr_at(sched, self.iteration, self.epoch)) if sched is not None else u.lr

    def set_epoch(self, epoch: int):
        self.epoch = epoch

    def set_constraints(self, constraints: Optional[Sequence[Dict]], layer: Optional[str] = None):
        """Replaces the constraints of one layer (layer None: of every layer with parameters), as Layer.Builder.constrainWeights /
        constrainBias / constrainAllParameters would have set them; None or [] removes them.  Applied from the next update on."""
        new = {l.name: constraints_by_param(l, list(constraints or ())) for l in self.layers if l.has_params and layer in (None, l.name)}
        self.layer_constraints = {name: per for name, per in {**self.layer_constraints, **new}.items() if per}      # new: all validated

    def apply_constraints(self):
        """Model.applyConstraints: each live (not frozen) layer's tensors, each through its list in order."""
        for l in self.layers:
            if l.name in self.layer_constraints and not getattr(l, "frozen", False):
                for p, lst in self.layer_constraints[l.name].items():
                    for c in lst:
                        l.params[p] = apply_constraint(l.params[p], c, self.q)

    def _link_dropout(self):
        """The DropoutLayers' shared state, and the last-stochastic-layer flag: the last active DropoutLayer of a pass advances P."""
        drops = [l for l in self.layers if isinstance(l, Dropout)]
        for l in drops:
            l.state, l.last = self.dropout, False
        active = [l for l in drops if l.active()]
        if active:
            active[-1].last = True

    def set_dropout_schedule(self, schedule: Optional[dict], layer: Optional[str] = None):
        """The library Net's set_dropout_schedule: layer None = every non-frozen DropoutLayer; schedule None = the constant."""
        for l in self.layers:
            if isinstance(l, Dropout) and (l.name == layer if layer is not None else not l.frozen):
                l.schedule = schedule
        self._link_dropout()

    def dropout_value(self, layer: str) -> float:
        """The value the DropoutLayer's next train-mode pass uses, at the net's own counters."""
        return self.layer(layer).value_at(self.iteration, self.epoch)

    def set_weight_noise(self, wn: Optional[Dict], layer: Optional[str] = None):
        """The library Net's set_weight_noise: layer None = every non-frozen conv, deconv or dense layer; wn None clears."""
        for l in self.layers:
            if isinstance(l, GEMM) and (l.name == layer if layer is not None else not getattr(l, "frozen", False)):
                l.weight_noise = wn

    def set_loss_weights(self, weights):
        """The loss layer's per-output weights (None: unweighted), checked against its outputs at every score."""
        self.loss_weights = None if weights is None else np.asarray(weights, np.float64).ravel()

    def dropout_pass(self) -> int:
        """The dropout pass counter P: train-mode forwards that drew a DropoutLayer mask or weight noise."""
        return self.dropout.pass_

    def set_dropout_pass(self, p: int):
        self.dropout.pass_ = p

    def _has_active_dropout(self) -> bool:
        """A stochastic pass: a DropoutLayer or a noisy layer draws."""
        return any((isinstance(l, Dropout) and l.active()) or weight_noise_active(l) for l in self.layers)

    # ---- DL4J flattened parameter vector -------------------------------------------------------
    def param_table(self):
        out = []
        for li, l in enumerate(self.layers):
            for pname, shape, order in l.param_specs():
                out.append((li, l.name, pname, shape, order))
        return out

    def num_params(self):
        return sum(int(np.prod(s)) for _, _, _, s, _ in self.param_table())

    def params_flat(self):
        return np.concatenate([self.layers[li].params[p].ravel(order=o.upper()) for li, _, p, _, o in self.param_table()])

    def set_params_flat(self, v):
        off = 0
        for li, _, p, shape, o in self.param_table():
            n = int(np.prod(shape))
            self.layers[li].params[p] = np.asarray(v[off:off + n], self.dtype).reshape(shape, order=o.upper()).copy()
            off += n

    def grads_flat(self):
        """ComputationGraph.gradient() flattened; frozen layers (no gradient) contribute zeros."""
        return np.concatenate([(self.layers[li].grads[p] if p in self.layers[li].grads else np.zeros(sh, self.dtype)).ravel(order=o.upper())
                               for li, _, p, sh, o in self.param_table()])

    def layer(self, name) -> Layer:
        for l in self.layers:
            if l.name == name:
                return l
        raise KeyError(name)

    # ---- forward / backward --------------------------------------------------------------------
    def forward(self, x, train: bool, collect: bool = False):
        self._skip_acc = {}
        for l in self.layers:
            l.noisy = None
        noisy = [l for l in self.layers if weight_noise_active(l)] if train else []
        if noisy:               # W' (and b') of every noisy layer at the top of the pass
            pass_, _ = self.dropout.current()
            for l in noisy:
                w, b = noisy_operands(l, l.weight_noise, l.index, self.dropout.seed, self.dropout.rank, pass_, self.dropout.counters(), self.dtype,
                                      l.q)
                l.noisy = {"W": dl4j_w(w, l.params["W"].shape)} | ({"b": b} if b is not None else {})
            if not any(isinstance(l, Dropout) and l.active() for l in self.layers):
                self.dropout.finish()
        acts = []
        a = np.asarray(x, self.dtype)
        for l in self.layers:
            # FrozenLayer (TransferLearning.setFeatureExtractor, J:350) always runs its layer in test mode
            t = train and not getattr(l, "frozen", False)
            a = l.forward(a, acts[l.src], t) if isinstance(l, Vertex) else l.forward(a, t)
            acts.append(a)
        return (a, acts) if collect else a

    def output(self, x):
        """ComputationGraph.output(x): inference mode => BatchNorm uses its mean/var parameters (J:420)."""
        return self.forward(x, train=False)

    def _backward(self, eps, lo: int, hi: int, collect: bool):
        """The backward walk: layers hi-1 down to lo, LossLayers left to the caller.  A vertex's skip share goes into its source's accumulator
        (the first consumer visited writes it, later ones add); a source adds its accumulator to the spine epsilon before its own backward."""
        epss = []
        for i in range(hi - 1, lo - 1, -1):
            l = self.layers[i]
            if isinstance(l, LossLayer):
                continue
            acc = self._skip_acc.pop(i, None)
            if acc is not None:
                eps = eps + acc.reshape(eps.shape)
            if isinstance(l, Vertex):
                eps, g = l.backward(eps)
                self._skip_acc[l.src] = self._skip_acc[l.src] + g if l.src in self._skip_acc else g
            else:
                eps = l.backward(eps)
            if collect:
                epss.append(eps)
        return (eps, epss[::-1]) if collect else eps

    def backward_from(self, eps, stop_at: int = 0, collect: bool = False):
        """Back-propagate eps (w.r.t. the output of the last non-loss layer handled by the caller)."""
        return self._backward(eps, stop_at, len(self.layers), collect)

    # Regularization (b2g_regularization: DL4J's l1, l2, l1Bias and l2Bias), per parameter as beta3's getL1ByParam / getL2ByParam:
    #   update  theta -= updater(g) + l2 * theta (W);  then theta -= l2Bias * theta (b) + l1 * sign(theta_before),  sign(+-0) = 0;  then the
    #           constraints.  The two subtractions are rounded to the net's dtype one after the other, as the library applies them.
    #   score   sum(loss) / mb + calc_l2() + calc_l1()
    def reg_coefs(self, layer: Layer, param: str) -> Tuple[float, float]:
        """(l1, l2) of one parameter: a conv, deconv, dense or output layer's W takes its l1 and l2, its b l1Bias and l2Bias, a PReLU's alpha
        ("W") its l1 and l2 as a weight; everything else (BatchNorm, every other layer) (0, 0).  l1, l1Bias and l2Bias are the net's
        layer_regularization, l2 the layer's."""
        if isinstance(layer, BatchNorm) and not layer.q.batchnorm_unregularized:
            raise NotImplementedError("only beta3's unregularized BatchNorm is restated")
        l1, l1_bias, l2_bias = self.layer_regularization.get(layer.name, (0.0, 0.0, 0.0))
        if isinstance(layer, PReLU):
            return (l1, float(layer.l2)) if param == "W" and layer.q.prelu_alpha_regularized else (0.0, 0.0)
        if not isinstance(layer, GEMM):
            return 0.0, 0.0
        if param == "W":
            return l1, float(layer.l2)
        if param == "b":
            return l1_bias, l2_bias
        return 0.0, 0.0

    def _reg_sum(self, which, norm):
        s = [0.0, 0.0]          # the PReLU terms are summed apart and added last, as the library sums them
        for l in self.layers:
            if l.has_params and not getattr(l, "frozen", False):     # FrozenLayer.calcL1() == calcL2() == 0
                for p, _, _ in l.param_specs():
                    c = self.reg_coefs(l, p)[which]
                    if c:
                        s[isinstance(l, PReLU)] += norm(c, l.params[p].astype(np.float64))
        return s[0] + s[1]

    def calc_l2(self) -> float:
        """ComputationGraph.calcL2(true): sum of 0.5 * l2 * ||W||^2 + 0.5 * l2_bias * ||b||^2 over the live layers."""
        return self._reg_sum(1, lambda c, v: 0.5 * c * float((v ** 2).sum()))

    def calc_l1(self) -> float:
        """ComputationGraph.calcL1(true): sum of l1 * ||W||_1 + l1_bias * ||b||_1 over the live layers."""
        return self._reg_sum(0, lambda c, v: c * float(np.abs(v).sum()))

    def l2_score(self):
        """The score's whole regularization term."""
        return self.calc_l2() + self.calc_l1()

    def compute_gradient_and_score(self, x, y, collect=False, pass_=None, row0=0, mask=None):
        """ComputationGraph.computeGradientAndScore: train-mode forward, loss, backprop.
        Gradients are minibatch *sums*; score = sum(loss)/mb + l2_score().
        pass_: the DropoutLayers draw rows [row0, row0 + mb) of that pass, and the pass counter is left alone.  mask: the labels mask."""
        if mask is not None and not self.q.masked_score_per_minibatch:
            raise NotImplementedError("only the minibatch divisor is restated")
        if pass_ is not None and self._has_active_dropout():
            self.dropout.queue.append((pass_, row0))
        out, acts = self.forward(x, train=True, collect=True)
        loss_sum, eps_in, epss = self._loss_backward(y) if mask is None else self._loss_backward(y, mask)
        score = float(loss_sum) / x.shape[0] + self.l2_score()
        if collect:
            return score, acts, epss, eps_in
        return score

    def _loss_backward(self, y, mask=None):
        """After a forward: the last layer's score on labels y (weighted by loss_weights, masked by mask), then the backward of its own
        parameters (an OutputLayer's) and the prefix.  Returns (loss sum, eps at the prefix's input, the prefix's epsilons).  Unmasked
        callers pass y alone, so a subclass that scores its own way may override the one-argument form."""
        last = self.layers[-1]
        loss_sum, eps = last.score_and_eps(np.asarray(y, self.dtype), self.loss_weights, mask)
        if last.has_params:
            eps = last.backward(eps)
        return (loss_sum,) + self.backward_from_prefix(eps, collect=True)

    def backward_from_prefix(self, eps, collect=False):
        """Backprop through all layers except the final loss-bearing one; stops at the frozen feature extractor (a frozen PReLU passes its
        input gradient)."""
        hi = len(self.layers) - 1
        lo = max((i + 1 for i in range(hi) if getattr(self.layers[i], "frozen", False) and not isinstance(self.layers[i], PReLU)), default=0)
        return self._backward(eps, lo, hi, collect)

    # ---- updater: BaseMultiLayerUpdater.update + UpdaterBlock + params.subi ----------------------
    def apply_update(self, mb: int, grads: Optional[Dict[Tuple[int, str], np.ndarray]] = None, frozen_from: Optional[int] = None):
        """g/=mb -> L2 normalization -> clip -> updater at the layer's lr -> +l2*W -> theta -= g -> theta -= the l1 and l2Bias terms ->
        constraints.  (SURVEY.md 8a row a9.)"""
        t = self.iteration + 1
        live = [(li, l) for li, l in enumerate(self.layers)
                if l.has_params and not getattr(l, "frozen", False)]     # FrozenLayer: no gradient, no update, no l2 decay
        g_all = {}
        for li, l in live:
            for pname, _, _ in l.param_specs():
                g = (grads[(li, pname)] if grads is not None else l.grads[pname]).astype(self.dtype).copy()
                if not (pname in l.noop_names() and self.q.bn_stats_minibatch_exempt):
                    g = g / mb
                g_all[(li, pname)] = g
        if self.gradient_normalization != "none":
            assert self.grad_clip == 0, "DL4J allows one gradient normalization per layer"
            g_all, self.grad_norm_last_norms = normalize(self, g_all, self.gradient_normalization, self.gradient_normalization_threshold, self.q)
        for li, l in live:
            u = l.updater or UpdaterCfg("sgd", 0.0)
            lr = self._lr(l, u)
            for pname, _, _ in l.param_specs():
                g = g_all[(li, pname)]
                noop = pname in l.noop_names()
                if self.grad_clip > 0 and (not noop or self.q.bn_stats_clipped):
                    g = np.clip(g, -self.grad_clip, self.grad_clip)
                upd = g if noop else update(u, self.state.get((li, pname)), g, t, self.q, lr)
                l1, l2 = self.reg_coefs(l, pname)
                l2_bias = l2 if pname == "b" else 0.0
                before = l.params[pname]
                if l.l2 and pname in l.l2_names():
                    if self.q.l2_after_updater:
                        upd = upd + l.l2 * before
                    else:
                        raise NotImplementedError("only the pre-beta4 post-updater l2 form is restated")
                l.params[pname] = (before - upd).astype(self.dtype)
                if l1 or l2_bias:
                    t_reg = (l2_bias * before if l2_bias else 0.0) + (l1 * np.sign(before) if l1 else 0.0)
                    l.params[pname] = (l.params[pname] - t_reg).astype(self.dtype)
        self.iteration += 1
        if self.layer_constraints:
            self.apply_constraints()

    def fit(self, x, y, mask=None):
        """ComputationGraph.fit(DataSet) for one minibatch (Solver -> StochasticGradientDescent.optimize); mask: the labels mask."""
        score = self.compute_gradient_and_score(x, y, mask=mask)
        self.apply_update(x.shape[0])
        return score


# --------------------------------------------------------------------------------------------------
# Synchronous parameter averaging (ParameterAveragingTrainingMaster; Python/gan.ipynb:177-187)
# --------------------------------------------------------------------------------------------------
def parameter_average(nets: Sequence[Net], into: Net):
    """Theta <- mean_i theta_i, and likewise the updater state (J:325-330; SURVEY.md 3.3)."""
    for li, l in enumerate(into.layers):
        if not l.has_params:
            continue
        for pname, _, _ in l.param_specs():
            l.params[pname] = sum(n.layers[li].params[pname] for n in nets) / len(nets)
            if (li, pname) in into.state:
                for k in range(len(into.state[(li, pname)])):
                    into.state[(li, pname)][k] = sum(n.state[(li, pname)][k] for n in nets) / len(nets)


# --------------------------------------------------------------------------------------------------
# The GAN step.
# --------------------------------------------------------------------------------------------------
def gan_step(G: Net, D: Net, x_real, z_d, z_g, y_real, y_fake, y_gen, fake_bn_train: bool = False, *, m_real=None, m_fake=None, m_gen=None):
    """The aliased G+D adversarial step the CUDA path executes (what J:408-471 computes for one real batch
    when the three graphs dis / gan / gen share storage instead of exchanging 28 setParam copies, and the
    two D minibatches are combined as one averaged update instead of two Spark workers):

      1. x_fake = G.output(z_d)            inference-mode BN (J:420)         [fake_bn_train=True: batch stats]
      2. D grads on (x_real, y_real) and (x_fake, y_fake) as two separate minibatches (separate BN batch
         statistics, as the two Spark workers have); summed, scaled by 1/(2N) (= the mean of the two
         workers' per-minibatch gradients); BN running-stat pseudo-gradients averaged over the two; one
         D updater step.
      3. G grads through D on z_g with labels y_gen (J:465-471): G and D both run train-mode BN; D's
         parameters, running stats and updater state are NOT touched (the reference's lr-0 "frozen" copy
         is overwritten from dis next iteration, J:429-460); one G updater step.
    D's DropoutLayers and weight noise draw as the library draws them, which runs the two D minibatches as one 2N-row pass: the real and fake
    minibatches are rows [0, N) and [N, 2N) of pass P, and the G step's D pass is P + 1 (the counter ends at P + 2).  D's scheduled dropout
    values and DropConnect p are read at D's counters in the D step and at G's in the G step's pass through D (the reference's stacked gan graph
    counts its own fits).  m_real, m_fake, m_gen: the labels masks of the three loss evaluations (None: unmasked).
    Returns dict(loss_d_real, loss_d_fake, loss_g, x_fake).
    """
    n = x_real.shape[0]
    if D._has_active_dropout():
        P = D.dropout.pass_
        D.dropout.queue += [(P, 0), (P, n)]
        D.dropout.pass_ = P + 1
    x_fake = G.forward(z_d, train=fake_bn_train)
    # --- D step
    s_real = D.compute_gradient_and_score(x_real, y_real, mask=m_real) - D.l2_score()
    g_real = {(li, p): l.grads[p].copy() for li, l in enumerate(D.layers) if l.has_params for p, _, _ in l.param_specs()}
    s_fake = D.compute_gradient_and_score(x_fake, y_fake, mask=m_fake) - D.l2_score()
    g_sum = {}
    for li, l in enumerate(D.layers):
        if not l.has_params:
            continue
        for p, _, _ in l.param_specs():
            if p in l.noop_names():
                g_sum[(li, p)] = 0.5 * (g_real[(li, p)] + l.grads[p])     # averaged pseudo-gradient
            else:
                g_sum[(li, p)] = g_real[(li, p)] + l.grads[p]
    D.apply_update(2 * n, grads=g_sum)
    # --- G step (through D, D untouched)
    xg = G.forward(z_g, train=True)
    D.dropout.lead = G
    try:
        D.forward(xg, train=True)
    finally:
        D.dropout.lead = None
    d_params_before = {(li, p): l.params[p] for li, l in enumerate(D.layers) if l.has_params for p, _, _ in l.param_specs()}
    loss_sum, eps_x, _ = D._loss_backward(y_gen) if m_gen is None else D._loss_backward(y_gen, m_gen)
    G.backward_from(eps_x.reshape(xg.shape))
    G.apply_update(n)
    for (li, p), v in d_params_before.items():
        D.layers[li].params[p] = v
    return dict(loss_d_real=s_real, loss_d_fake=s_fake, loss_g=float(loss_sum) / n, x_fake=x_fake)


def gan_iteration_reference(dis: Net, gen: Net, gan: Net, n_gen_layers: int, x_real, z_d, z_g, y_real, y_fake, y_gen,
                            workers: int = 2):
    """Literal replay of one loop body J:408-510 with three separate graphs and Spark parameter averaging:
    dis is fit by two workers (real batch / fake batch, one local iteration each) whose parameters AND
    updater state are averaged (SURVEY.md 3.3); D -> gan copy; gan fit on (z_g, 1); gan -> gen copy."""
    import copy
    x_fake = gen.output(z_d)
    w = [copy.deepcopy(dis) for _ in range(2)]
    s0 = w[0].fit(x_real, y_real)
    s1 = w[1].fit(x_fake.reshape(x_real.shape) if x_fake.shape != x_real.shape else x_fake, y_fake)
    parameter_average(w, dis)
    dis.iteration = w[0].iteration
    # J:429-460: dis -> gan_dis_*
    for k, l in enumerate(dis.layers):
        if l.has_params:
            for p, _, _ in l.param_specs():
                gan.layers[n_gen_layers + k].params[p] = l.params[p].copy()
    s2 = gan.fit(z_g, y_gen)
    # J:474-510: gan_* -> gen_*
    for k, l in enumerate(gen.layers):
        if l.has_params:
            for p, _, _ in l.param_specs():
                l.params[p] = gan.layers[k].params[p].copy()
    return dict(score_d_real=s0, score_d_fake=s1, score_gan=s2, x_fake=x_fake)


# --------------------------------------------------------------------------------------------------
# Model zoo: the nets of SURVEY.md Appendix A (C1, reference file) and Appendix B (C2-C4 DCGAN), C5 MLP.
# --------------------------------------------------------------------------------------------------
def reference_discriminator(lr=0.002, dtype=np.float64, seed=666, prefix="dis", quirks=DEFAULT_QUIRKS) -> Net:
    """J:118-165.  Global: tanh, Xavier, l2 1e-4, clip 1.0, RmsProp(lr,1e-8,1e-8)."""
    u = lambda: RmsProp(lr, 1e-8, 1e-8)
    L = [
        Reshape((1, 28, 28), name=f"{prefix}_ff2cnn"),
        BatchNorm(1, updater=u(), name=f"{prefix}_batch_layer_1"),
        Conv2D(1, 64, (5, 5), (2, 2), (0, 0), "tanh", updater=u(), l2=1e-4, name=f"{prefix}_conv2d_layer_2"),
        MaxPool((2, 2), (1, 1), name=f"{prefix}_maxpool_layer_3"),
        Conv2D(64, 128, (5, 5), (2, 2), (0, 0), "tanh", updater=u(), l2=1e-4, name=f"{prefix}_conv2d_layer_4"),
        MaxPool((2, 2), (1, 1), name=f"{prefix}_maxpool_layer_5"),
        Reshape((1152,), name=f"{prefix}_cnn2ff"),
        Dense(1152, 1024, "tanh", updater=u(), l2=1e-4, name=f"{prefix}_dense_layer_6"),
        Output(1024, 1, updater=u(), l2=1e-4, name=f"{prefix}_output_layer_7"),
    ]
    return Net(L, seed=seed, dtype=dtype, grad_clip=1.0, quirks=quirks)


def reference_generator_layers(lr, z=2, prefix="gen"):
    u = lambda: RmsProp(lr, 1e-8, 1e-8)
    return [
        BatchNorm(z, updater=u(), name=f"{prefix}_batch_1"),
        Dense(z, 1024, "tanh", updater=u(), l2=1e-4, name=f"{prefix}_dense_layer_2"),
        Dense(1024, 6272, "tanh", updater=u(), l2=1e-4, name=f"{prefix}_dense_layer_3"),
        BatchNorm(6272, updater=u(), name=f"{prefix}_batch_4"),
        Reshape((128, 7, 7), name=f"{prefix}_ff2cnn"),
        Upsample2D(2, name=f"{prefix}_deconv2d_5"),
        Conv2D(128, 64, (5, 5), (1, 1), (2, 2), "tanh", updater=u(), l2=1e-4, name=f"{prefix}_conv2d_6"),
        Upsample2D(2, name=f"{prefix}_deconv2d_7"),
        Conv2D(64, 1, (5, 5), (1, 1), (2, 2), "sigmoid", updater=u(), l2=1e-4, name=f"{prefix}_conv2d_8"),
    ]


def reference_generator(lr=0.0, z=2, dtype=np.float64, seed=666, quirks=DEFAULT_QUIRKS) -> Net:
    """J:173-221 (the lr-0 "frozen" copy used for gen.output)."""
    return Net(reference_generator_layers(lr, z, "gen"), seed=seed, dtype=dtype, grad_clip=1.0, quirks=quirks)


def reference_gan(gen_lr=0.004, z=2, dtype=np.float64, seed=666, quirks=DEFAULT_QUIRKS) -> Tuple[Net, int]:
    """J:228-310: trainable G stacked on lr-0 D.  NB the gan graph sets no l2 on... it does (J:233-237)."""
    g = reference_generator_layers(gen_lr, z, "gan")
    d = reference_discriminator(0.0, dtype, seed, "gan_dis", quirks).layers
    # gen output is [N,1,28,28]; dis's ff2cnn reshape is a no-op on it
    return Net(g + d, seed=seed, dtype=dtype, grad_clip=1.0, quirks=quirks), len(g)


def reference_computer_vision(dis: Net, lr=0.002, n_classes=10, seed=666, quirks=DEFAULT_QUIRKS) -> Net:
    """J:337-364: TransferLearning.GraphBuilder(dis).setFeatureExtractor("dis_dense_layer_6").removeVertexKeepConnections(output)
    .addLayer("dis_batch", BatchNormalization(1024)).addLayer("dis_output_layer_7", OutputLayer(MCXENT, softmax, 10)).
    The trunk layers are shared objects' copies marked frozen (FrozenLayer); fine-tune config: l2 1e-4, clip 1.0, RmsProp(lr,1e-8,1e-8)."""
    import copy
    trunk = [copy.deepcopy(l) for l in dis.layers[:-1]]
    for l in trunk:
        l.frozen = True
    u = lambda: RmsProp(lr, 1e-8, 1e-8)
    head = [BatchNorm(1024, updater=u(), name="dis_batch"), OutputSoftmax(1024, n_classes, updater=u(), l2=1e-4, name="dis_output_layer_7")]
    net = Net(head, seed=seed, dtype=dis.dtype, grad_clip=1.0, quirks=quirks)     # initialises only the new layers
    net.layers = trunk + head
    net.state = {(li + len(trunk), p): v for (li, p), v in net.state.items()}
    return net


def dcgan_generator(size=64, z=100, nf=64, nc=3, lr=2e-4, beta1=0.5, dtype=np.float64, seed=666, quirks=DEFAULT_QUIRKS) -> Net:
    """SURVEY.md Appendix B: ConvTranspose2D(4x4)+BN+ReLU stack, tanh output; Adam(lr, beta1, 0.999)."""
    u = lambda: Adam(lr, beta1, 0.999, 1e-8)
    n_up = int(np.log2(size)) - 2               # 64 -> 4 stride-2 stages, 128 -> 5
    ch = nf * 2 ** (n_up - 1)
    L: List[Layer] = [Reshape((z, 1, 1), name="gen_ff2cnn"),
                      Deconv2D(z, ch, (4, 4), (1, 1), (0, 0), updater=u(), name="gen_deconv_1", has_bias=False),
                      BatchNorm(ch, updater=u(), name="gen_bn_1"), ActivationLayer("relu", name="gen_act_1")]
    for i in range(n_up - 1):
        L += [Deconv2D(ch, ch // 2, (4, 4), (2, 2), (1, 1), updater=u(), name=f"gen_deconv_{i + 2}", has_bias=False),
              BatchNorm(ch // 2, updater=u(), name=f"gen_bn_{i + 2}"), ActivationLayer("relu", name=f"gen_act_{i + 2}")]
        ch //= 2
    L += [Deconv2D(ch, nc, (4, 4), (2, 2), (1, 1), "tanh", updater=u(), name=f"gen_deconv_{n_up + 1}")]
    return Net(L, seed=seed, dtype=dtype, quirks=quirks)


def dcgan_discriminator(size=64, nf=64, nc=3, lr=2e-4, beta1=0.5, dtype=np.float64, seed=667, quirks=DEFAULT_QUIRKS) -> Net:
    """SURVEY.md Appendix B: Conv(4x4 s2 p1)+LeakyReLU(0.2) ; (Conv+BN+LeakyReLU)* ; Conv(4x4 s1 p0) -> logit; XENT."""
    u = lambda: Adam(lr, beta1, 0.999, 1e-8)
    n_down = int(np.log2(size)) - 2
    L: List[Layer] = [Conv2D(nc, nf, (4, 4), (2, 2), (1, 1), "lrelu", 0.2, updater=u(), name="dis_conv_1")]
    ch = nf
    for i in range(n_down - 1):
        L += [Conv2D(ch, ch * 2, (4, 4), (2, 2), (1, 1), updater=u(), name=f"dis_conv_{i + 2}", has_bias=False),
              BatchNorm(ch * 2, updater=u(), name=f"dis_bn_{i + 2}"), ActivationLayer("lrelu", 0.2, name=f"dis_act_{i + 2}")]
        ch *= 2
    L += [Conv2D(ch, 1, (4, 4), (1, 1), (0, 0), updater=u(), name=f"dis_conv_{n_down + 1}"),
          LossLayer(name="dis_loss")]
    return Net(L, seed=seed, dtype=dtype, quirks=quirks)


def mlp_generator(z=100, hidden=1024, d=256, lr=2e-4, beta1=0.5, dtype=np.float64, seed=666, quirks=DEFAULT_QUIRKS) -> Net:
    u = lambda: Adam(lr, beta1, 0.999, 1e-8)
    return Net([Dense(z, hidden, "relu", updater=u(), name="gen_dense_1"),
                Dense(hidden, hidden, "relu", updater=u(), name="gen_dense_2"),
                Dense(hidden, d, "tanh", updater=u(), name="gen_dense_3")], seed=seed, dtype=dtype, quirks=quirks)


def mlp_discriminator(d=256, hidden=1024, lr=2e-4, beta1=0.5, dtype=np.float64, seed=667, quirks=DEFAULT_QUIRKS) -> Net:
    u = lambda: Adam(lr, beta1, 0.999, 1e-8)
    return Net([Dense(d, hidden, "lrelu", 0.2, updater=u(), name="dis_dense_1"),
                Dense(hidden, hidden, "lrelu", 0.2, updater=u(), name="dis_dense_2"),
                Output(hidden, 1, updater=u(), name="dis_output")], seed=seed, dtype=dtype, quirks=quirks)


def synthetic_batch(n, size=64, nc=3, z=100, seed=666, dtype=np.float32):
    """SURVEY.md 8d synthetic inputs: x~U(-1,1) NCHW, z~U(-1,1) (J:420,465), labels 1+0.05N / 0+0.05N (J:405-406), y_gen=1 (J:466)."""
    rng = np.random.default_rng(seed)
    x = rng.uniform(-1, 1, (n, nc, size, size)).astype(dtype)
    z_d = rng.uniform(-1, 1, (n, z)).astype(dtype)
    z_g = rng.uniform(-1, 1, (n, z)).astype(dtype)
    y_real = (1 + 0.05 * rng.standard_normal((n, 1))).astype(dtype)
    y_fake = (0 + 0.05 * rng.standard_normal((n, 1))).astype(dtype)
    y_gen = np.ones((n, 1), dtype)
    return x, z_d, z_g, y_real, y_fake, y_gen


# --------------------------------------------------------------------------------------------------
# Layer specs (gan_deeplearning4j_b200.models / engine.LAYER_TYPES) -> Net
# --------------------------------------------------------------------------------------------------
def net_from_specs(specs, input_shape, *, quirks: Quirks = DEFAULT_QUIRKS, dtype=np.float64, seed=1, grad_clip=0.0, flat_input=True,
                   mask_seed=666, rank=0, constraints: Optional[Sequence[Dict]] = None) -> Net:
    """The Net of the layer specs the CUDA engine consumes.  input_shape: (C,H,W) or (F,).  flat_input: prepend the convolutionalFlat
    reshape (the oracle's layer indices are then the specs' + 1).  A spec's scheduled lr becomes the layer's schedule; its constant lr is
    the schedule's value at 0, as the library keeps it.  An activation's alpha defaults as engine.layer_desc fills it.  Each layer's `index`
    is its position in `specs` (the library's index, the L of its draws).  A vertex's inputs are resolved by vertex_inputs.  mask_seed, rank:
    see Net.  A spec's "constraints" are its layer's; constraints: the global builder's, for every layer whose own reach none of its
    parameters, as DL4J's builder fills them in.  A GEMM or PReLU spec's "l1", "l1_bias" and "l2_bias" are the net's layer_regularization
    (its "l2" the layer's); a GEMM
    spec's "weight_noise" is its layer's, and its "weight_init" replaces the seeded draw as b2g_net_init_weights does right after creation
    (seed mask_seed).  The last spec's "loss_weights" are the net's."""
    layers, by_layer = [], {}
    shape = (1,) + tuple(input_shape)
    if len(input_shape) == 3 and flat_input:
        layers.append(Reshape(tuple(input_shape), name="in_reshape"))      # convolutionalFlat accepts [N,784] or [N,1,28,28]
    shapes = [shape] * len(layers)          # each layer's output shape
    skips = vertex_inputs(specs, len(layers))
    schedules, inits, regs = {}, [], {}
    for s in specs[:-1]:
        if s.get("loss_weights") is not None:
            raise ValueError("loss_weights belong to the net's last (loss) layer")
    for i, s in enumerate(specs):
        t, name = s["type"], s.get("name", "")
        u = updater_cfg(s.get("updater"))
        if u is not None and isinstance(s["updater"].get("lr"), dict) and u.kind != "noop":
            schedules[name] = s["updater"]["lr"]
        act = s.get("activation", "identity")
        alpha = s.get("alpha", ACT_ALPHA_DEFAULTS.get(act, 0.01))
        n_in = s.get("n_in") or (int(np.prod(shape[1:])) if t in ("dense", "output") else shape[1])
        k, st, pad = s.get("kernel"), s.get("stride", (1, 1)), s.get("padding", (0, 0))
        if t == "conv2d":
            l = Conv2D(n_in, s["n_out"], k, st, pad, act, alpha, u, s.get("l2", 0.0), name, s.get("has_bias", True))
        elif t == "deconv2d":
            l = Deconv2D(n_in, s["n_out"], k, st, pad, act, alpha, u, s.get("l2", 0.0), name, s.get("has_bias", True))
        elif t == "dense":
            l = Dense(n_in, s["n_out"], act, alpha, u, s.get("l2", 0.0), name, s.get("has_bias", True))
        elif t == "output" and s.get("loss", "xent") == "mcxent":
            l = OutputSoftmax(n_in, s["n_out"], u, s.get("l2", 0.0), name)
        elif t == "output":
            l = Output(n_in, s["n_out"], u, s.get("l2", 0.0), name, loss=s.get("loss", "xent"), activation=act, alpha=alpha)
        elif t == "loss":
            l = LossLayer(name, loss=s.get("loss", "xent"), activation=act, alpha=alpha)
        elif t == "cnn_loss":
            if i != len(specs) - 1:
                raise ValueError("a cnn_loss spec must be the last layer")
            l = CnnLossLayer(name, loss=s.get("loss", "xent"), activation=act, alpha=alpha)
        elif t == "elementwise":
            l = ElementWiseVertex(s["op"], *skips[i], name)
        elif t == "merge":
            l = MergeVertex(*skips[i], name)
        elif t == "batchnorm":
            l = BatchNorm(shape[1], s.get("decay", 0.9), s.get("eps", 1e-5), u, name)
        elif t == "activation":
            l = ActivationLayer(act, alpha, name)
        elif t == "maxpool":
            l = MaxPool(k, st, name)
        elif t == "subsampling":
            l = Subsampling(s["pooling"], k, st, pad, s.get("pnorm", 0), name)
        elif t == "global_pooling":
            l = GlobalPooling(s.get("pooling", "max"), s.get("pnorm", 2), name)
        elif t == "upsample2d":
            l = Upsample2D(s.get("size", 2), name)
        elif t == "prelu":
            l = PReLU(shape[1:], s.get("shared_axes", ()), u, s.get("l2", 0.0), name)
        elif t == "dropout":
            kind = s.get("kind", "dropout")
            v = s[VALUE_KEY[kind]]
            sched = v if isinstance(v, dict) else None
            l = Dropout(value(sched, 0) if sched else v, name, kind=kind, schedule=sched)
        elif t == "ff_to_cnn":
            h, w, c = s["to"]; l = Reshape((c, h, w), name)
        elif t == "cnn_to_ff":
            l = Reshape((int(np.prod(shape[1:])),), name)
        else:
            raise ValueError(t)
        l.index = i
        if s.get("frozen", False):
            l.frozen = True
        reg = tuple(float(s.get(k, 0.0)) for k in ("l1", "l1_bias", "l2_bias"))
        if isinstance(l, GEMM + (PReLU,)) and any(reg):
            regs[name] = reg
        if isinstance(l, GEMM):
            l.weight_noise = s.get("weight_noise")
        if s.get("weight_init") is not None:
            if not isinstance(l, GEMM):
                raise NotImplementedError(f"{t} {name!r}: weight_init is restated on conv, deconv and dense layers")
            inits.append((l, s["weight_init"]))
        per = constraints_by_param(l, s.get("constraints", ())) or constraints_by_param(l, constraints or ())
        if per:
            by_layer[name] = per
        layers.append(l)
        shape = l.out_shape(shape, shapes[l.src]) if isinstance(l, Vertex) else l.out_shape(shape)
        shapes.append(shape)
    net = Net(layers, seed=seed, dtype=dtype, grad_clip=grad_clip, quirks=quirks, mask_seed=mask_seed, rank=rank)
    for l, wi in inits:
        init_layer(l, wi, mask_seed, l.index, quirks)
    for name, sched in schedules.items():
        net.set_lr_schedule(sched, name)
    net.layer_constraints, net.layer_regularization = by_layer, regs
    if specs and specs[-1].get("loss_weights") is not None:
        last = net.layers[-1]
        net.set_loss_weights(check_weights(last.loss, specs[-1]["loss_weights"], shape[1], quirks))
    return net


def vertex_inputs(specs, off=0):
    """Each vertex spec's "inputs" as (j, order): j the skip source's layer index (its position in the specs + off), order 0 when the inputs
    are (spine, source) and 1 when they are (source, spine); None for the other specs.  The spine is the previous spec and the source the one
    earlier spec of the other name.  ValueError for any other graph."""
    out = []
    for i, s in enumerate(specs):
        if s["type"] not in ("elementwise", "merge"):
            out.append(None)
            continue
        inputs, earlier = list(s.get("inputs", ())), [p.get("name", "") for p in specs[:i]]
        if len(inputs) != 2 or not earlier or earlier[-1] not in inputs:
            raise ValueError(f"vertex {s.get('name', '')!r}: inputs {inputs} are not the previous layer and one skip source")
        order = 0 if inputs[0] == earlier[-1] else 1
        hits = [j for j, name in enumerate(earlier) if name == inputs[1 - order]]
        if len(hits) != 1:
            raise ValueError(f"vertex {s.get('name', '')!r}: input {inputs[1 - order]!r} names {len(hits)} earlier layers (needs exactly one)")
        out.append((hits[0] + off, order))
    return out
