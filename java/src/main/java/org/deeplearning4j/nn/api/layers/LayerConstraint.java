// LayerConstraint: a constraint applied to a layer's parameters after every update (include/b200gan.h, b2g_constraint).
package org.deeplearning4j.nn.api.layers;

public interface LayerConstraint {
    /** b2g_constraint_kind: 0 MaxNorm, 1 MinMaxNorm, 2 UnitNorm, 3 NonNegative. */
    int kind();
    /** Bit d = DL4J dimension d of the parameter the norm is taken over; 0 = all of them. */
    int dimsMask();
    double maxNorm();
    double minNorm();
    double rate();
    /** The DL4J dimensions as the library's bit mask. */
    static int mask(int... dimensions) { int m = 0; for (int d : dimensions) m |= 1 << d; return m; }
}
