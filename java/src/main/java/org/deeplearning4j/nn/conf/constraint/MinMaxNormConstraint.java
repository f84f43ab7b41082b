// new MinMaxNormConstraint(min, max, [rate,] dimensions): w *= (rate * clip(norm, min, max) + (1 - rate) * norm) / (norm + 1e-6) per group.
// Arithmetic: include/b200gan.h, b2g_constraint.
package org.deeplearning4j.nn.conf.constraint;

import org.deeplearning4j.nn.api.layers.LayerConstraint;

public class MinMaxNormConstraint implements LayerConstraint {
    public static final double DEFAULT_RATE = 1.0;
    private final double min, max, rate; private final int dims;
    public MinMaxNormConstraint(double min, double max, int... dimensions) { this(min, max, DEFAULT_RATE, dimensions); }
    public MinMaxNormConstraint(double min, double max, double rate, int... dimensions) {
        this.min = min; this.max = max; this.rate = rate; this.dims = LayerConstraint.mask(dimensions);
    }
    public int kind() { return 1; }
    public int dimsMask() { return dims; }
    public double maxNorm() { return max; }
    public double minNorm() { return min; }
    public double rate() { return rate; }
}
