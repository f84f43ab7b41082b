package org.deeplearning4j.nn.conf.dropout;
/** new GaussianDropout(rate), rate in [0, 1): y = x * (1 + sqrt(rate / (1 - rate)) * N(0, 1)) in training. */
public final class GaussianDropout implements IDropout {
    private final double v; private final org.nd4j.linalg.schedule.ISchedule s;
    public GaussianDropout(double rate) { this.v = rate; this.s = null; }
    public GaussianDropout(org.nd4j.linalg.schedule.ISchedule rateSchedule) { this.v = rateSchedule.valueAt(0, 0); this.s = rateSchedule; }
    public org.nd4j.linalg.schedule.ISchedule schedule() { return s; }
    public int kind() { return 1; }
    public double value() { return v; }
}
