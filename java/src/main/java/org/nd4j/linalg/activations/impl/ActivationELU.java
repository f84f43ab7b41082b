package org.nd4j.linalg.activations.impl;

import org.nd4j.linalg.activations.Activation;
import org.nd4j.linalg.activations.IActivation;

/** new ActivationELU(alpha): z >= 0 ? z : alpha * (e^z - 1); DL4J's default alpha is 1.0. */
public class ActivationELU implements IActivation {
    private final float alpha;
    public ActivationELU() { this(1.0); }
    public ActivationELU(double alpha) { this.alpha = (float) alpha; }
    public int code() { return Activation.ELU.code; }
    public float alpha() { return alpha; }
}
