package org.deeplearning4j.nn.conf.distribution;
/** new UniformDistribution(lower, upper). */
public class UniformDistribution extends Distribution {
    private final double lower, upper;
    public UniformDistribution(double lower, double upper) { this.lower = lower; this.upper = upper; }
    public int kind() { return 1; }
    public double a() { return lower; }
    public double b() { return upper; }
}
