"""Layer-spec builders for the networks on the path (SURVEY.md Appendix A/B): the reference file's own graphs
(C1: J:118-310), the north_star DCGAN (C2-C4) and the MLP-GAN (C5).  A spec is a list of plain dicts that
`engine.Net` turns into b2g_layer_desc structs -- the same information the Java facade's builders collect."""
from __future__ import annotations

import math
from typing import Dict, List


def rmsprop(lr, rms_decay=0.95, eps=1e-8):
    """new RmsProp(learningRate, rmsDecay, epsilon) -- NB the reference passes (lr, 1e-8, 1e-8) (J:133)."""
    return {"kind": "rmsprop", "lr": lr, "rms_decay": rms_decay, "eps": eps}


def adam(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8):
    return {"kind": "adam", "lr": lr, "beta1": beta1, "beta2": beta2, "eps": eps}


def sgd(lr):
    return {"kind": "sgd", "lr": lr}


# org.nd4j.linalg.learning.config.{Nesterovs, AdaGrad, AdaMax, Nadam, AMSGrad, AdaDelta, NoOp} with DL4J's defaults; the update each computes is
# stated at b2g_updater in include/b200gan.h.  lr may be a schedule (below) for every kind but AdaDelta, which has no learning rate.
def nesterovs(lr=0.1, momentum=0.9):
    """new Nesterovs(learningRate, momentum)."""
    return {"kind": "nesterovs", "lr": lr, "momentum": momentum}


def adagrad(lr=0.1, eps=1e-6):
    """new AdaGrad(learningRate, epsilon); the history starts at epsilon."""
    return {"kind": "adagrad", "lr": lr, "eps": eps}


def adamax(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8):
    return {"kind": "adamax", "lr": lr, "beta1": beta1, "beta2": beta2, "eps": eps}


def nadam(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8):
    return {"kind": "nadam", "lr": lr, "beta1": beta1, "beta2": beta2, "eps": eps}


def amsgrad(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8):
    return {"kind": "amsgrad", "lr": lr, "beta1": beta1, "beta2": beta2, "eps": eps}


def adadelta(rho=0.95, eps=1e-6):
    """new AdaDelta(rho, epsilon): no learning rate."""
    return {"kind": "adadelta", "rho": rho, "eps": eps}


def noop():
    return {"kind": "noop"}


# ------------------------------------------------------------------ learning-rate schedules ------------
# org.nd4j.linalg.schedule.*: pass one as an updater's lr (new Adam(ISchedule): adam(lr=step_schedule(2e-4, 0.5, 1000))) or to
# Net.set_lr_schedule.  type = ScheduleType: "iteration" (the updater's iteration count) or "epoch" (Net.set_epoch).  The arithmetic is
# stated at b2g_lr_schedule in include/b200gan.h.
def exponential_schedule(initial, gamma, type="iteration"):
    """ExponentialSchedule: initial * gamma^i."""
    return {"schedule": "exponential", "type": type, "initial": initial, "gamma": gamma}


def inverse_schedule(initial, gamma, power, type="iteration"):
    """InverseSchedule: initial / (1 + gamma*i)^power."""
    return {"schedule": "inverse", "type": type, "initial": initial, "gamma": gamma, "power": power}


def sigmoid_schedule(initial, gamma, step_size, type="iteration"):
    """SigmoidSchedule: initial / (1 + exp(-gamma*(i - step_size)))."""
    return {"schedule": "sigmoid", "type": type, "initial": initial, "gamma": gamma, "step": step_size}


def step_schedule(initial, decay_rate, step, type="iteration"):
    """StepSchedule: initial * decay_rate^floor(i / step)."""
    return {"schedule": "step", "type": type, "initial": initial, "decay_rate": decay_rate, "step": step}


def map_schedule(values, type="iteration"):
    """MapSchedule: the value at the largest key <= i; values = {int: float} or [(key, value), ...] and must hold key 0.  Stored as a list of
    [key, value] pairs sorted by key (a JSON object would turn the keys into strings)."""
    pairs = sorted((int(k), float(v)) for k, v in (values.items() if isinstance(values, dict) else values))
    return {"schedule": "map", "type": type, "values": [[k, v] for k, v in pairs]}


# ------------------------------------------------------------------ weight constraints -----------------
# org.deeplearning4j.nn.conf.constraint.*: put them in a layer spec's "constraints" list (Layer.Builder.constrainWeights / constrainBias /
# constrainAllParameters) or pass them as Net(..., constraints=[...]) (the global builder's: a layer whose own list reaches none of its
# parameters takes them).  dims are DL4J dimensions of the parameter (conv W [nOut, nIn, kH, kW], deconv W [nIn, nOut, kH, kW], dense W
# [nIn, nOut], vectors [1, n]); the norm is taken over them once per index of the others, () = over everything.  on: "weights", "bias" or
# "all".  Arithmetic at b2g_constraint in include/b200gan.h.
def max_norm(max, dims, on="weights") -> Dict:
    """new MaxNormConstraint(maxNorm, dimensions...)."""
    return {"constraint": "max_norm", "max": float(max), "dims": [int(d) for d in dims], "on": on}


def min_max_norm(min, max, dims, rate=1.0, on="weights") -> Dict:
    """new MinMaxNormConstraint(min, max, rate, dimensions...) (rate 1.0: MinMaxNormConstraint(min, max, dimensions...))."""
    return {"constraint": "min_max_norm", "min": float(min), "max": float(max), "rate": float(rate), "dims": [int(d) for d in dims], "on": on}


def unit_norm(dims, on="weights") -> Dict:
    """new UnitNormConstraint(dimensions...)."""
    return {"constraint": "unit_norm", "dims": [int(d) for d in dims], "on": on}


def non_negative(on="weights") -> Dict:
    """new NonNegativeConstraint()."""
    return {"constraint": "non_negative", "on": on}


# ------------------------------------------------------------------ IDropout kinds of a DropoutLayer ---------------------
# DropoutLayer.Builder(IDropout) (b2g_dropout_kind in include/b200gan.h); a "dropout" spec without "kind" is DropoutLayer.Builder(p).  Each value
# may be a schedule (exponential_schedule, ...): new GaussianNoise(ISchedule), evaluated on the device at every train-mode forward.
def _value(v):
    return v if isinstance(v, dict) else float(v)


def gaussian_noise(stddev, name="") -> Dict:
    """new DropoutLayer.Builder(new GaussianNoise(stddev)): y = x + stddev * N(0, 1) in training."""
    return {"type": "dropout", "name": name, "kind": "gaussian_noise", "stddev": _value(stddev)}


def gaussian_dropout(rate, name="") -> Dict:
    """new DropoutLayer.Builder(new GaussianDropout(rate)): y = x * (1 + sqrt(rate / (1 - rate)) * N(0, 1)) in training."""
    return {"type": "dropout", "name": name, "kind": "gaussian_dropout", "rate": _value(rate)}


def alpha_dropout(p, name="") -> Dict:
    """new DropoutLayer.Builder(new AlphaDropout(p)), p = the retain probability: the dropout that keeps SELU's mean and variance."""
    return {"type": "dropout", "name": name, "kind": "alpha_dropout", "p": _value(p)}


def spatial_dropout(p, name="") -> Dict:
    """new DropoutLayer.Builder(new SpatialDropout(p)), p = the retain probability: whole (example, channel) maps kept or zeroed."""
    return {"type": "dropout", "name": name, "kind": "spatial_dropout", "p": _value(p)}


# ------------------------------------------------------------------ weight noise ----------------------
# Layer.Builder.weightNoise / NeuralNetConfiguration.Builder.weightNoise (b2g_weight_noise in include/b200gan.h): the value of a GEMM layer
# spec's "weight_noise" key, or of Net(..., weight_noise=...) for every GEMM layer without its own.
def drop_connect(p, apply_to_biases=False) -> Dict:
    """new DropConnect(p[, applyToBiases]), p = the retain probability of each weight (a number or a schedule); W' = keep ? W : 0, not rescaled."""
    return {"weight_noise": "drop_connect", "p": _value(p), "apply_to_bias": bool(apply_to_biases)}


def normal(mean, std) -> Dict:
    """new NormalDistribution(mean, std)"""
    return {"distribution": "normal", "mean": float(mean), "std": float(std)}


def uniform(lower, upper) -> Dict:
    """new UniformDistribution(lower, upper)"""
    return {"distribution": "uniform", "lower": float(lower), "upper": float(upper)}


def weight_noise(distribution, apply_to_bias=False, additive=True) -> Dict:
    """new WeightNoise(distribution, applyToBias, additive): W' = W + n (additive) or W * n, n drawn from normal(..) or uniform(..)."""
    return {"weight_noise": "weight_noise", "distribution": dict(distribution), "apply_to_bias": bool(apply_to_bias), "additive": bool(additive)}


# ------------------------------------------------------------------ weight initialization ---------------
# Layer.Builder / NeuralNetConfiguration.Builder .weightInit, .dist and .biasInit (b2g_weight_init in include/b200gan.h): the value of a GEMM
# layer spec's "weight_init" key, or of Net(..., weight_init=...) for every GEMM layer without its own.  The distributions below, with normal
# and uniform above, are DISTRIBUTION's.
def truncated_normal(mean, std) -> Dict:
    """new TruncatedNormalDistribution(mean, std): values beyond 2 std are redrawn"""
    return {"distribution": "truncated_normal", "mean": float(mean), "std": float(std)}


def log_normal(mean, std) -> Dict:
    """new LogNormalDistribution(mean, std): exp of a normal(mean, std)"""
    return {"distribution": "log_normal", "mean": float(mean), "std": float(std)}


def binomial(n_trials, p) -> Dict:
    """new BinomialDistribution(nTrials, p): ValueError for an nTrials that is not a whole number."""
    if not math.isfinite(float(n_trials)) or float(n_trials) != math.floor(float(n_trials)):
        raise ValueError(f"BinomialDistribution nTrials {n_trials!r} is not a whole number")
    return {"distribution": "binomial", "n_trials": int(n_trials), "p": float(p)}


def constant(value) -> Dict:
    """new ConstantDistribution(value)"""
    return {"distribution": "constant", "value": float(value)}


def weight_init(scheme, dist=None, bias_init=0.0) -> Dict:
    """.weightInit(WeightInit.<SCHEME>) with .dist(dist) for "distribution" and .biasInit(bias_init): scheme is the lower-case WeightInit name
    ("xavier", "relu", "var_scaling_normal_fan_avg", ...).  ValueError for what the engine refuses (engine.weight_init_struct)."""
    from .engine import weight_init_struct
    wi = {"weight_init": scheme, "bias_init": float(bias_init)}
    if dist is not None:
        wi["distribution"] = dict(dist)
    weight_init_struct(wi)
    return wi


# ------------------------------------------------------------------ pooling layers ---------------------
# SubsamplingLayer / GlobalPoolingLayer (b2g_pooling in include/b200gan.h).  SubsamplingLayer(MAX) is the "maxpool" spec (unpadded).
def subsampling(pooling, kernel=(1, 1), stride=(2, 2), padding=(0, 0), pnorm=None, name="") -> Dict:
    """new SubsamplingLayer.Builder(PoolingType.AVG / SUM / PNORM).kernelSize(kernel).stride(stride).padding(padding).pnorm(p) (DL4J's default
    kernel 1x1, stride 2x2).  PNORM needs pnorm, a whole number >= 1."""
    if pooling not in ("avg", "sum", "pnorm"):
        raise ValueError(f"subsampling pooling {pooling!r}: one of avg, sum, pnorm (MAX is the 'maxpool' spec)")
    spec = {"type": "subsampling", "name": name, "pooling": pooling, "kernel": tuple(kernel), "stride": tuple(stride), "padding": tuple(padding)}
    if pooling == "pnorm":
        if pnorm is None:
            raise ValueError("PNORM subsampling needs pnorm (a whole number >= 1)")
        spec["pnorm"] = int(pnorm)
    return spec


def global_pooling(pooling="max", pnorm=2, name="") -> Dict:
    """new GlobalPoolingLayer.Builder(PoolingType).pnorm(p) (DL4J's defaults MAX, p = 2): [mb, C, H, W] -> [mb, C]."""
    if pooling not in ("max", "avg", "sum", "pnorm"):
        raise ValueError(f"global pooling {pooling!r}: one of max, avg, sum, pnorm")
    spec = {"type": "global_pooling", "name": name, "pooling": pooling}
    if pooling == "pnorm":
        spec["pnorm"] = int(pnorm)
    return spec


_global_pooling_spec = global_pooling       # dcgan_discriminator's argument of the same name shadows the builder


# ------------------------------------------------------------------ per-pixel loss ---------------------
def cnn_loss(loss="xent", activation="identity", name="", alpha=None, loss_weights=None) -> Dict:
    """new CnnLossLayer.Builder(LossFunction).activation(act): the loss on every pixel of a [mb, C, H, W] map, labels [mb, C, H, W]
    (B2G_LAYER_CNN_LOSS in include/b200gan.h).  XENT implies a sigmoid per element, MCXENT a softmax over the channels of each pixel; the
    others apply `activation`.  loss_weights: the loss's per-channel weights (new LossMCXENT(weights), ...; C finite floats), or None."""
    if loss not in ("xent", "mcxent", "mse", "l1", "l2", "mae", "hinge", "squared_hinge", "wasserstein"):
        raise ValueError(f"unknown loss {loss!r}")
    if loss in ("xent", "mcxent") and activation != "identity":
        raise ValueError(f"{loss.upper()} implies its activation: activation applies to the losses other than XENT and MCXENT")
    spec = {"type": "cnn_loss", "name": name, "loss": loss}
    if loss not in ("xent", "mcxent"):
        spec.update(_act(activation, alpha))
    if loss_weights is not None:
        spec["loss_weights"] = [float(v) for v in loss_weights]
    return spec


# ------------------------------------------------------------------ learned activation -----------------
def prelu(shared_axes=(), name="", input_shape=None) -> Dict:
    """new PReLULayer.Builder().sharedAxes(shared_axes).inputShape(input_shape) (B2G_LAYER_PRELU in include/b200gan.h): y = x < 0 ? alpha*x : x
    with learned slopes alpha ("W", starting at 0), one per element of the input shape except along DL4J's shared axes (1 = C, 2 = H, 3 = W):
    (2, 3) is one slope per channel.  input_shape ([C, H, W] or [F]), when given, must be the inferred input.  Add "updater", "l1" / "l2",
    "weight_init" (zero, ones, distribution) or "frozen" like on any layer with parameters."""
    spec = {"type": "prelu", "name": name, "shared_axes": sorted({int(a) for a in shared_axes})}
    if input_shape is not None:
        spec["input_shape"] = [int(v) for v in input_shape]
    from .engine import prelu_shared_mask
    prelu_shared_mask(spec)
    return spec


def _act_layer(name, activation, alpha, updater) -> Dict:
    """The activation of a BatchNorm block: an ActivationLayer, or for activation "prelu" a PReLULayer shared over H and W (one slope per channel)
    on the block's updater."""
    if activation == "prelu":
        return dict(prelu((2, 3), name), updater=updater())
    return dict({"type": "activation", "name": name}, **_act(activation, alpha))


# ------------------------------------------------------------------ skip connections -------------------
# ElementWiseVertex / MergeVertex (B2G_LAYER_ELEMENTWISE / B2G_LAYER_MERGE in include/b200gan.h).  A vertex's inputs are layer names: one of them
# must be the layer right before it (the spine), the other any earlier layer (engine.resolve_vertices).
def elementwise(op, inputs, name="") -> Dict:
    """graphBuilder.addVertex(name, new ElementWiseVertex(Op), inputs...): op one of add, subtract, product, average, max."""
    if op not in ("add", "subtract", "product", "average", "max"):
        raise ValueError(f"unknown ElementWiseVertex op {op!r}")
    if len(inputs) != 2:
        raise ValueError("an ElementWiseVertex here takes exactly two inputs")
    return {"type": "elementwise", "name": name, "op": op, "inputs": list(inputs)}


def merge(inputs, name="") -> Dict:
    """graphBuilder.addVertex(name, new MergeVertex(), inputs...): the two inputs concatenated along the channels (features), in input order."""
    if len(inputs) != 2:
        raise ValueError("a MergeVertex here takes exactly two inputs")
    return {"type": "merge", "name": name, "inputs": list(inputs)}


def residual_block(prefix, ch, skip, lr=2e-4, beta1=0.5, activation="relu", alpha=None) -> List[Dict]:
    """An identity residual block on the ch-channel map of layer `skip`, which must be the layer right before the block:
    conv3x3 -> BatchNorm -> act -> conv3x3 -> BatchNorm -> ElementWiseVertex(Add)(., skip) -> act (the convolutions stride 1, pad 1, no bias;
    activation "prelu": PReLULayers shared over H and W)."""
    u = lambda: adam(lr, beta1, 0.999, 1e-8)
    conv = lambda k: {"type": "conv2d", "name": f"{prefix}_conv_{k}", "n_in": ch, "n_out": ch, "kernel": (3, 3), "stride": (1, 1), "padding": (1, 1),
                      "has_bias": False, "updater": u()}
    return [conv(1), {"type": "batchnorm", "name": f"{prefix}_bn_1", "updater": u()}, _act_layer(f"{prefix}_act_1", activation, alpha, u),
            conv(2), {"type": "batchnorm", "name": f"{prefix}_bn_2", "updater": u()},
            elementwise("add", [f"{prefix}_bn_2", skip], name=f"{prefix}_add"), _act_layer(f"{prefix}_act_2", activation, alpha, u)]


def unet(size=64, nc=3, n_classes=2, nf=32, depth=2, loss="mcxent", lr=1e-3, beta1=0.9, activation="relu", alpha=None) -> List[Dict]:
    """A U-Net segmentation net (Ronneberger et al. 2015) of `depth` levels into a CnnLossLayer.  Input (nc, size, size), labels [n_classes,
    size, size].  Level k (channels nf * 2^k): conv3x3 -> BatchNorm -> act, then MaxPool 2x2 s2; the bottom: conv3x3 -> BatchNorm -> act; on the
    way up Deconvolution2D 4x4 s2 p1 -> MergeVertex(up, level k's act) -> conv3x3 -> BatchNorm -> act; last a 1x1 conv onto n_classes and
    CnnLossLayer(loss)."""
    if size % (2 ** depth):
        raise ValueError(f"size {size} is not divisible by 2^depth = {2 ** depth}")
    u = lambda: adam(lr, beta1, 0.999, 1e-8)
    conv_bn_act = lambda name, c_in, c_out: [
        {"type": "conv2d", "name": f"{name}_conv", "n_in": c_in, "n_out": c_out, "kernel": (3, 3), "stride": (1, 1), "padding": (1, 1), "has_bias": False, "updater": u()},
        {"type": "batchnorm", "name": f"{name}_bn", "updater": u()}, dict({"type": "activation", "name": f"{name}_act"}, **_act(activation, alpha))]
    L, c = [], nc
    for k in range(depth):
        L += conv_bn_act(f"unet_enc{k}", c, nf * 2 ** k) + [{"type": "maxpool", "name": f"unet_pool{k}", "kernel": (2, 2), "stride": (2, 2)}]
        c = nf * 2 ** k
    L += conv_bn_act("unet_mid", c, nf * 2 ** depth)
    c = nf * 2 ** depth
    for k in reversed(range(depth)):
        ck = nf * 2 ** k
        L += [{"type": "deconv2d", "name": f"unet_up{k}", "n_in": c, "n_out": ck, "kernel": (4, 4), "stride": (2, 2), "padding": (1, 1), "updater": u()},
              merge([f"unet_up{k}", f"unet_enc{k}_act"], name=f"unet_merge{k}")]
        L += conv_bn_act(f"unet_dec{k}", 2 * ck, ck)
        c = ck
    return L + [{"type": "conv2d", "name": "unet_head", "n_in": c, "n_out": n_classes, "kernel": (1, 1), "stride": (1, 1), "padding": (0, 0), "updater": u()},
                cnn_loss(loss, name="unet_loss")]


# ------------------------------------------------------------------ C1: the reference graphs ---------
def reference_discriminator(lr=0.002, prefix="dis") -> List[Dict]:
    """J:118-165: BN -> Conv5x5 s2 (1->64) -> MaxPool 2x2 s1 -> Conv5x5 s2 (64->128) -> MaxPool -> Dense 1024 -> Output(1, sigmoid, XENT);
    global tanh / l2 1e-4 / RmsProp(lr,1e-8,1e-8).  Net config: input (1,28,28), grad_clip=1.0."""
    u = lambda: rmsprop(lr, 1e-8, 1e-8)
    return [
        {"type": "batchnorm", "name": f"{prefix}_batch_layer_1", "updater": u()},
        {"type": "conv2d", "name": f"{prefix}_conv2d_layer_2", "n_in": 1, "n_out": 64, "kernel": (5, 5), "stride": (2, 2), "activation": "tanh", "updater": u(), "l2": 1e-4},
        {"type": "maxpool", "name": f"{prefix}_maxpool_layer_3", "kernel": (2, 2), "stride": (1, 1)},
        {"type": "conv2d", "name": f"{prefix}_conv2d_layer_4", "n_in": 64, "n_out": 128, "kernel": (5, 5), "stride": (2, 2), "activation": "tanh", "updater": u(), "l2": 1e-4},
        {"type": "maxpool", "name": f"{prefix}_maxpool_layer_5", "kernel": (2, 2), "stride": (1, 1)},
        {"type": "cnn_to_ff", "name": f"{prefix}_cnn2ff"},
        {"type": "dense", "name": f"{prefix}_dense_layer_6", "n_out": 1024, "activation": "tanh", "updater": u(), "l2": 1e-4},
        {"type": "output", "name": f"{prefix}_output_layer_7", "n_out": 1, "updater": u(), "l2": 1e-4},
    ]


def reference_generator(lr=0.0, z=2, prefix="gen") -> List[Dict]:
    """J:173-221 (the "deconv" layers are Upsampling2D + Conv5x5 p2).  Input (z,), grad_clip=1.0."""
    u = lambda: rmsprop(lr, 1e-8, 1e-8)
    return [
        {"type": "batchnorm", "name": f"{prefix}_batch_1", "updater": u()},
        {"type": "dense", "name": f"{prefix}_dense_layer_2", "n_out": 1024, "activation": "tanh", "updater": u(), "l2": 1e-4},
        {"type": "dense", "name": f"{prefix}_dense_layer_3", "n_out": 6272, "activation": "tanh", "updater": u(), "l2": 1e-4},
        {"type": "batchnorm", "name": f"{prefix}_batch_4", "updater": u()},
        {"type": "ff_to_cnn", "name": f"{prefix}_ff2cnn", "to": (7, 7, 128)},
        {"type": "upsample2d", "name": f"{prefix}_deconv2d_5", "size": 2},
        {"type": "conv2d", "name": f"{prefix}_conv2d_6", "n_in": 128, "n_out": 64, "kernel": (5, 5), "padding": (2, 2), "activation": "tanh", "updater": u(), "l2": 1e-4},
        {"type": "upsample2d", "name": f"{prefix}_deconv2d_7", "size": 2},
        {"type": "conv2d", "name": f"{prefix}_conv2d_8", "n_in": 64, "n_out": 1, "kernel": (5, 5), "padding": (2, 2), "activation": "sigmoid", "updater": u(), "l2": 1e-4},
    ]


def reference_gan(gen_lr=0.004, z=2) -> List[Dict]:
    """J:228-310: trainable generator stacked on the lr-0 discriminator copy."""
    return reference_generator(gen_lr, z, "gan") + reference_discriminator(0.0, "gan_dis")


def reference_computer_vision(lr=0.002, n_classes=10) -> List[Dict]:
    """J:337-364: the discriminator trunk frozen up to dis_dense_layer_6 (setFeatureExtractor), its output layer replaced by
    BatchNormalization(1024) "dis_batch" + OutputLayer(MCXENT, softmax, 10).  Input (1,28,28), grad_clip=1.0."""
    trunk = [dict(s, frozen=True) for s in reference_discriminator(lr)[:-1]]
    u = lambda: rmsprop(lr, 1e-8, 1e-8)
    return trunk + [{"type": "batchnorm", "name": "dis_batch", "updater": u()},
                    {"type": "output", "name": "dis_output_layer_7", "n_out": n_classes, "loss": "mcxent", "updater": u(), "l2": 1e-4}]


# ------------------------------------------------------------------ C2-C4: DCGAN -----------------------
def _act(activation, alpha=None) -> Dict:
    """The spec keys of an activation: LeakyReLU carries its alpha (0.2 when not given, the DCGAN value); another kind carries alpha only when
    one is given (engine.layer_desc then fills DL4J's default)."""
    if activation == "lrelu" and alpha is None:
        alpha = 0.2
    return {"activation": activation} if alpha is None else {"activation": activation, "alpha": alpha}


def dcgan_generator(size=64, z=100, nf=64, nc=3, lr=2e-4, beta1=0.5, activation="relu", out_activation="tanh", alpha=None,
                    residual=False) -> List[Dict]:
    """ConvolutionTranspose2D(4x4)+BatchNorm+ReLU stack, tanh output (SURVEY.md Appendix B).  Input (z,).
    activation: the ActivationLayers' kind (any engine.ACTS name; alpha as in _act), or "prelu": a PReLULayer shared over H and W in place of
    each ActivationLayer; out_activation: the last deconv's.
    residual: one identity residual_block after each up-sampling stage (a ResNet-style generator)."""
    u = lambda: adam(lr, beta1, 0.999, 1e-8)
    n_up = int(math.log2(size)) - 2
    ch = nf * 2 ** (n_up - 1)
    block = lambda k, c: residual_block(f"gen_res_{k}", c, f"gen_act_{k}", lr, beta1, activation, alpha) if residual else []
    L = [{"type": "ff_to_cnn", "name": "gen_ff2cnn", "to": (1, 1, z)},
         {"type": "deconv2d", "name": "gen_deconv_1", "n_in": z, "n_out": ch, "kernel": (4, 4), "stride": (1, 1), "padding": (0, 0), "has_bias": False, "updater": u()},
         {"type": "batchnorm", "name": "gen_bn_1", "updater": u()}, _act_layer("gen_act_1", activation, alpha, u)]
    L += block(1, ch)
    for i in range(n_up - 1):
        L += [{"type": "deconv2d", "name": f"gen_deconv_{i + 2}", "n_in": ch, "n_out": ch // 2, "kernel": (4, 4), "stride": (2, 2), "padding": (1, 1), "has_bias": False, "updater": u()},
              {"type": "batchnorm", "name": f"gen_bn_{i + 2}", "updater": u()}, _act_layer(f"gen_act_{i + 2}", activation, alpha, u)]
        ch //= 2
        L += block(i + 2, ch)
    L += [{"type": "deconv2d", "name": f"gen_deconv_{n_up + 1}", "n_in": ch, "n_out": nc, "kernel": (4, 4), "stride": (2, 2), "padding": (1, 1), "updater": u(), **_act(out_activation)}]
    return L


def _loss_keys(loss, out_activation) -> Dict:
    """The spec keys of a discriminator's loss-bearing layer: none for XENT (today's specs), else the loss and the activation it applies."""
    if loss == "xent":
        if out_activation != "identity":
            raise ValueError("XENT implies the sigmoid: out_activation applies to the losses other than XENT")
        return {}
    return {"loss": loss, "activation": out_activation}


def dcgan_discriminator(size=64, nf=64, nc=3, lr=2e-4, beta1=0.5, loss="xent", out_activation="identity", activation="lrelu", alpha=None,
                        global_pooling=None, patch=False, residual=False, instance_noise=None, drop_connect=None) -> List[Dict]:
    """Conv(4x4 s2 p1)+LeakyReLU(0.2); (Conv+BatchNorm+LeakyReLU)*; Conv(4x4 s1 p0) -> logit; LossLayer(loss).  Input (nc,size,size).
    loss: "xent" (sigmoid implied), or "mse" (least-squares GAN), "hinge", "wasserstein", ... applied to out_activation(logit).
    activation / alpha: the hidden activation in place of LeakyReLU(0.2) (as in _act); "prelu": each ActivationLayer becomes a PReLULayer shared
    over H and W, and the first conv becomes identity followed by such a layer ("dis_act_1").
    global_pooling: a pooling kind ("sum" for the projected / ResNet-style head, "avg", "max", "pnorm"): GlobalPoolingLayer + OutputLayer(nOut 1,
    loss) in place of the last conv and its LossLayer.
    patch: a PatchGAN critic -- the down-sampling stages stop at the max(4, size/16) map (at most four stride-2 convs), and a 3x3 s1 p1 conv onto
    1 channel and a CnnLossLayer(loss) take the place of the last conv and its LossLayer: one logit and one label per patch (a 4x4 map up to
    64x64, 8x8 at 128x128).
    residual: one identity residual_block after each down-sampling stage (a ResNet-style critic).
    instance_noise = stddev: a GaussianNoise(stddev) DropoutLayer on the input (instance noise: real and fake images both get the noise).
    drop_connect = p: DropConnect(p) weight noise on every conv and output layer (see _with_drop_connect)."""
    if patch and global_pooling is not None:
        raise ValueError("patch and global_pooling are two different heads")
    u = lambda: adam(lr, beta1, 0.999, 1e-8)
    n_down = int(math.log2(size)) - 2
    if patch:
        n_down = min(n_down, 4)
    block = lambda k, c, skip: residual_block(f"dis_res_{k}", c, skip, lr, beta1, activation, alpha) if residual else []
    L = [] if instance_noise is None else [gaussian_noise(instance_noise, name="dis_instance_noise")]
    p = activation == "prelu"
    L += [{"type": "conv2d", "name": "dis_conv_1", "n_in": nc, "n_out": nf, "kernel": (4, 4), "stride": (2, 2), "padding": (1, 1), **({} if p else _act(activation, alpha)), "updater": u()}]
    L += [_act_layer("dis_act_1", activation, alpha, u)] if p else []
    ch = nf
    L += block(1, ch, "dis_act_1" if p else "dis_conv_1")
    for i in range(n_down - 1):
        L += [{"type": "conv2d", "name": f"dis_conv_{i + 2}", "n_in": ch, "n_out": ch * 2, "kernel": (4, 4), "stride": (2, 2), "padding": (1, 1), "has_bias": False, "updater": u()},
              {"type": "batchnorm", "name": f"dis_bn_{i + 2}", "updater": u()}, _act_layer(f"dis_act_{i + 2}", activation, alpha, u)]
        ch *= 2
        L += block(i + 2, ch, f"dis_act_{i + 2}")
    if global_pooling is not None:
        return _with_drop_connect(L + [_global_pooling_spec(global_pooling, name="dis_global_pool"),
                                       dict({"type": "output", "name": "dis_output", "n_out": 1, "updater": u()}, **_loss_keys(loss, out_activation))], drop_connect)
    if patch:
        return _with_drop_connect(L + [{"type": "conv2d", "name": f"dis_conv_{n_down + 1}", "n_in": ch, "n_out": 1, "kernel": (3, 3), "stride": (1, 1), "padding": (1, 1), "updater": u()},
                                       dict({"type": "cnn_loss", "name": "dis_loss"}, **_loss_keys(loss, out_activation))], drop_connect)
    L += [{"type": "conv2d", "name": f"dis_conv_{n_down + 1}", "n_in": ch, "n_out": 1, "kernel": (4, 4), "stride": (1, 1), "padding": (0, 0), "updater": u()},
          dict({"type": "loss", "name": "dis_loss"}, **_loss_keys(loss, out_activation))]
    return _with_drop_connect(L, drop_connect)


def _with_drop_connect(specs: List[Dict], p) -> List[Dict]:
    """p None: the specs unchanged; else each GEMM layer spec gets "weight_noise": drop_connect(p) (the global builder's weightNoise)."""
    if p is None:
        return specs
    return [dict(s, weight_noise=drop_connect(p)) if s["type"] in ("conv2d", "deconv2d", "dense", "output") else s for s in specs]


# ------------------------------------------------------------------ C5: MLP-GAN --------------------------
def mlp_generator(z=100, hidden=1024, d=256, lr=2e-4, beta1=0.5, activation="relu", out_activation="tanh", alpha=None) -> List[Dict]:
    """activation / alpha: the hidden layers' activation (as in _act); out_activation: the last layer's."""
    u = lambda: adam(lr, beta1, 0.999, 1e-8)
    return [{"type": "dense", "name": "gen_dense_1", "n_out": hidden, **_act(activation, alpha), "updater": u()},
            {"type": "dense", "name": "gen_dense_2", "n_out": hidden, **_act(activation, alpha), "updater": u()},
            {"type": "dense", "name": "gen_dense_3", "n_out": d, **_act(out_activation), "updater": u()}]


def mlp_discriminator(d=256, hidden=1024, lr=2e-4, beta1=0.5, dropout=None, loss="xent", out_activation="identity", activation="lrelu",
                      alpha=None, instance_noise=None, drop_connect=None) -> List[Dict]:
    """dropout = p: a DropoutLayer(p) (p = retain probability) after each hidden LeakyReLU, the DL4J MNIST GAN example's discriminator shape.
    loss / out_activation: the OutputLayer's loss, as for dcgan_discriminator.  activation / alpha: the hidden activation (as in _act).
    instance_noise = stddev: a GaussianNoise(stddev) DropoutLayer on the input, as for dcgan_discriminator.
    drop_connect = p: DropConnect(p) weight noise on every dense and output layer, as for dcgan_discriminator."""
    u = lambda: adam(lr, beta1, 0.999, 1e-8)
    L = [] if instance_noise is None else [gaussian_noise(instance_noise, name="dis_instance_noise")]
    for i in (1, 2):
        L.append({"type": "dense", "name": f"dis_dense_{i}", "n_out": hidden, **_act(activation, alpha), "updater": u()})
        if dropout is not None:
            L.append({"type": "dropout", "name": f"dis_dropout_{i}", "p": dropout})
    return _with_drop_connect(L + [dict({"type": "output", "name": "dis_output", "n_out": 1, "updater": u()}, **_loss_keys(loss, out_activation))], drop_connect)


# algorithmic MACs per image of the conv/deconv/dense layers (SURVEY.md 8d: F = 2*(4*G_f + 8*D_f))
def forward_macs(specs: List[Dict], input_shape) -> int:
    c, h, w = input_shape if len(input_shape) == 3 else (input_shape[0], 1, 1)
    from .engine import resolve_vertices
    macs = 0
    skips = resolve_vertices(specs)      # the merge vertices' sources by index, as b2g_net_create receives them (ValueError if not spine plus skip)
    channels = []                        # each layer's output channels
    for i, s in enumerate(specs):
        t = s["type"]
        if t == "merge":
            c += channels[skips[i][0]]
        if t == "conv2d":
            k, st, p = s["kernel"], s.get("stride", (1, 1)), s.get("padding", (0, 0))
            h, w = (h - k[0] + 2 * p[0]) // st[0] + 1, (w - k[1] + 2 * p[1]) // st[1] + 1
            macs += h * w * s["n_out"] * c * k[0] * k[1]; c = s["n_out"]
        elif t == "deconv2d":
            k, st, p = s["kernel"], s.get("stride", (1, 1)), s.get("padding", (0, 0))
            macs += h * w * c * s["n_out"] * k[0] * k[1]
            h, w = st[0] * (h - 1) + k[0] - 2 * p[0], st[1] * (w - 1) + k[1] - 2 * p[1]; c = s["n_out"]
        elif t in ("dense", "output"):
            macs += c * h * w * s["n_out"]; c, h, w = s["n_out"], 1, 1
        elif t == "maxpool":
            k, st = s["kernel"], s.get("stride", (1, 1)); h, w = (h - k[0]) // st[0] + 1, (w - k[1]) // st[1] + 1
        elif t == "subsampling":
            k, st, p = s["kernel"], s.get("stride", (1, 1)), s.get("padding", (0, 0))
            h, w = (h + 2 * p[0] - k[0]) // st[0] + 1, (w + 2 * p[1] - k[1]) // st[1] + 1
        elif t == "global_pooling":
            h, w = 1, 1
        elif t == "upsample2d":
            h, w = h * s.get("size", 2), w * s.get("size", 2)
        elif t == "ff_to_cnn":
            h, w, c = s["to"]
        elif t == "cnn_to_ff":
            c, h, w = c * h * w, 1, 1
        channels.append(c)
    return macs
