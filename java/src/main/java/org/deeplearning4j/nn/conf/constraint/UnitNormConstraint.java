// new UnitNormConstraint(dimensions): w /= norm per group (an all-zero group is left as it is).  Arithmetic: include/b200gan.h, b2g_constraint.
package org.deeplearning4j.nn.conf.constraint;

import org.deeplearning4j.nn.api.layers.LayerConstraint;

public class UnitNormConstraint implements LayerConstraint {
    private final int dims;
    public UnitNormConstraint(int... dimensions) { this.dims = LayerConstraint.mask(dimensions); }
    public int kind() { return 2; }
    public int dimsMask() { return dims; }
    public double maxNorm() { return 0.0; }
    public double minNorm() { return 0.0; }
    public double rate() { return 1.0; }
}
