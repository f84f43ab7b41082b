package org.deeplearning4j.nn.conf.weightnoise;
import org.deeplearning4j.nn.conf.distribution.Distribution;
/** new WeightNoise(distribution[, applyToBias], additive) (DL4J 1.0.0-beta3): W' = W + n (additive) or W * n in training, n ~ distribution. */
public final class WeightNoise implements IWeightNoise {
    private final Distribution d; private final boolean bias, add;
    public WeightNoise(Distribution distribution) { this(distribution, false, true); }
    public WeightNoise(Distribution distribution, boolean additive) { this(distribution, false, additive); }
    public WeightNoise(Distribution distribution, boolean applyToBias, boolean additive) { this.d = distribution; this.bias = applyToBias; this.add = additive; }
    public int kind() { return 2; }
    public boolean applyToBias() { return bias; }
    public Distribution distribution() { return d; }
    public boolean additive() { return add; }
}
