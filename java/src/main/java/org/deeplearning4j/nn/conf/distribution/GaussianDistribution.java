package org.deeplearning4j.nn.conf.distribution;
/** new GaussianDistribution(mean, std): NormalDistribution under its other name. */
public class GaussianDistribution extends NormalDistribution {
    public GaussianDistribution(double mean, double std) { super(mean, std); }
}
