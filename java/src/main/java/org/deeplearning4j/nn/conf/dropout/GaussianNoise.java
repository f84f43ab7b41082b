package org.deeplearning4j.nn.conf.dropout;
/** new GaussianNoise(stddev), stddev >= 0: y = x + stddev * N(0, 1) in training (instance noise on a discriminator's input). */
public final class GaussianNoise implements IDropout {
    private final double v; private final org.nd4j.linalg.schedule.ISchedule s;
    public GaussianNoise(double stddev) { this.v = stddev; this.s = null; }
    public GaussianNoise(org.nd4j.linalg.schedule.ISchedule stddevSchedule) { this.v = stddevSchedule.valueAt(0, 0); this.s = stddevSchedule; }
    public org.nd4j.linalg.schedule.ISchedule schedule() { return s; }
    public int kind() { return 2; }
    public double value() { return v; }
}
