package org.nd4j.linalg.learning.config;
/** new AdaDelta(rho = 0.95, epsilon = 1e-6): msg = rho*msg + (1-rho)*g^2; u = sqrt(msdx + eps) / sqrt(msg + eps) * g;
 *  msdx = rho*msdx + (1-rho)*u^2.  No learning rate (so no schedule); rho goes in beta1. */
public class AdaDelta implements IUpdater {
    public static final double DEFAULT_ADADELTA_RHO = 0.95, DEFAULT_ADADELTA_EPSILON = 1e-6;
    private final double rho, eps;
    public AdaDelta() { this(DEFAULT_ADADELTA_RHO, DEFAULT_ADADELTA_EPSILON); }
    public AdaDelta(double rho, double epsilon) { this.rho = rho; eps = epsilon; }
    public int kind() { return 9; } public float lr() { return 0f; } public float beta1() { return (float) rho; } public float beta2() { return 0f; } public float eps() { return (float) eps; }
}
