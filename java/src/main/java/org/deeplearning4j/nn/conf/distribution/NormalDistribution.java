package org.deeplearning4j.nn.conf.distribution;
/** new NormalDistribution(mean, std). */
public class NormalDistribution extends Distribution {
    private final double mean, std;
    public NormalDistribution(double mean, double std) { this.mean = mean; this.std = std; }
    public int kind() { return 0; }
    public double a() { return mean; }
    public double b() { return std; }
}
