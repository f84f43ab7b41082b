package org.deeplearning4j.nn.conf.distribution;
/** new LogNormalDistribution(mean, std): exp of a normal draw. */
public class LogNormalDistribution extends Distribution {
    private final double mean, std;
    public LogNormalDistribution(double mean, double std) { this.mean = mean; this.std = std; }
    public int kind() { return 3; }
    public double a() { return mean; }
    public double b() { return std; }
}
