// new NonNegativeConstraint(): w = w < 0 ? 0 : w, element-wise.  Arithmetic: include/b200gan.h, b2g_constraint.
package org.deeplearning4j.nn.conf.constraint;

import org.deeplearning4j.nn.api.layers.LayerConstraint;

public class NonNegativeConstraint implements LayerConstraint {
    public NonNegativeConstraint() { }
    public int kind() { return 3; }
    public int dimsMask() { return 0; }
    public double maxNorm() { return 0.0; }
    public double minNorm() { return 0.0; }
    public double rate() { return 1.0; }
}
