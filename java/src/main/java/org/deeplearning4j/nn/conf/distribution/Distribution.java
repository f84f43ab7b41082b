package org.deeplearning4j.nn.conf.distribution;
/** The distributions of WeightNoise and WeightInit.DISTRIBUTION (b2g_distribution_kind in include/b200gan.h): kind and its two parameters. */
public abstract class Distribution {
    public abstract int kind();
    public abstract double a();
    public abstract double b();
}
