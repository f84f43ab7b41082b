// new MaxNormConstraint(maxNorm, dimensions): w *= clip(norm, 0, maxNorm) / (norm + 1e-6) per group.  Arithmetic: include/b200gan.h, b2g_constraint.
package org.deeplearning4j.nn.conf.constraint;

import org.deeplearning4j.nn.api.layers.LayerConstraint;

public class MaxNormConstraint implements LayerConstraint {
    private double max; private final int dims;
    public MaxNormConstraint(double maxNorm, int... dimensions) { this.max = maxNorm; this.dims = LayerConstraint.mask(dimensions); }
    public int kind() { return 0; }
    public int dimsMask() { return dims; }
    public double maxNorm() { return max; }
    public double minNorm() { return 0.0; }
    public double rate() { return 1.0; }
}
