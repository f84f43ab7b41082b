package org.nd4j.linalg.activations;
/** b2g_activation codes (formulas at b2g_activation in include/b200gan.h).  LEAKYRELU's alpha travels separately (DL4J default 0.01; DCGAN passes
 *  0.2); ELU's alpha and THRESHOLDEDRELU's theta default to 1.0, or take ActivationELU(alpha) / ActivationThresholdedReLU(theta). */
public enum Activation {
    IDENTITY(0), TANH(1), SIGMOID(2), RELU(3), LEAKYRELU(4), ELU(5), SELU(6), SOFTPLUS(7), SOFTSIGN(8), HARDTANH(9), HARDSIGMOID(10), RELU6(11),
    SWISH(12), CUBE(13), RATIONALTANH(14), RECTIFIEDTANH(15), THRESHOLDEDRELU(16);
    public final int code; Activation(int c) { code = c; }
}
