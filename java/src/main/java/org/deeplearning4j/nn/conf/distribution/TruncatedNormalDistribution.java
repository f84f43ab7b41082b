package org.deeplearning4j.nn.conf.distribution;
/** new TruncatedNormalDistribution(mean, std): values beyond 2 std are redrawn. */
public class TruncatedNormalDistribution extends Distribution {
    private final double mean, std;
    public TruncatedNormalDistribution(double mean, double std) { this.mean = mean; this.std = std; }
    public int kind() { return 2; }
    public double a() { return mean; }
    public double b() { return std; }
}
