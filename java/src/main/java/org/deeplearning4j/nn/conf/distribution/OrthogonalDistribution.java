package org.deeplearning4j.nn.conf.distribution;
/** new OrthogonalDistribution(gain): the native call refuses it (B2G_ERR_UNSUPPORTED; it needs an SVD). */
public class OrthogonalDistribution extends Distribution {
    private final double gain;
    public OrthogonalDistribution(double gain) { this.gain = gain; }
    public int kind() { return 6; }
    public double a() { return gain; }
    public double b() { return 0; }
}
