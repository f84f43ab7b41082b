package org.deeplearning4j.nn.conf.distribution;
/** new BinomialDistribution(nTrials, p). */
public class BinomialDistribution extends Distribution {
    private final int nTrials; private final double p;
    public BinomialDistribution(int nTrials, double probabilityOfSuccess) { this.nTrials = nTrials; this.p = probabilityOfSuccess; }
    public int kind() { return 4; }
    public double a() { return nTrials; }
    public double b() { return p; }
}
