package org.deeplearning4j.nn.conf.dropout;
/** new AlphaDropout(p), p = the RETAIN probability in (0, 1]: the dropout that keeps SELU's mean and variance. */
public final class AlphaDropout implements IDropout {
    private final double v; private final org.nd4j.linalg.schedule.ISchedule s;
    public AlphaDropout(double p) { this.v = p; this.s = null; }
    public AlphaDropout(org.nd4j.linalg.schedule.ISchedule pSchedule) { this.v = pSchedule.valueAt(0, 0); this.s = pSchedule; }
    public org.nd4j.linalg.schedule.ISchedule schedule() { return s; }
    public int kind() { return 3; }
    public double value() { return v; }
}
