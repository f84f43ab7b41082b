package org.nd4j.linalg.activations.impl;

import org.nd4j.linalg.activations.Activation;
import org.nd4j.linalg.activations.IActivation;

/** new ActivationThresholdedReLU(theta): z > theta ? z : 0; DL4J's default theta is 1.0. */
public class ActivationThresholdedReLU implements IActivation {
    private final float theta;
    public ActivationThresholdedReLU() { this(1.0); }
    public ActivationThresholdedReLU(double theta) { this.theta = (float) theta; }
    public int code() { return Activation.THRESHOLDEDRELU.code; }
    public float alpha() { return theta; }
}
