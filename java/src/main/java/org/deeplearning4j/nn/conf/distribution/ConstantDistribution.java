package org.deeplearning4j.nn.conf.distribution;
/** new ConstantDistribution(value). */
public class ConstantDistribution extends Distribution {
    private final double value;
    public ConstantDistribution(double value) { this.value = value; }
    public int kind() { return 5; }
    public double a() { return value; }
    public double b() { return 0; }
}
