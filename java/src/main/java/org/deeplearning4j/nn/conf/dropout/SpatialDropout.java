package org.deeplearning4j.nn.conf.dropout;
/** new SpatialDropout(p), p = the RETAIN probability in (0, 1]: one keep draw per (example, channel) map of a convolutional input. */
public final class SpatialDropout implements IDropout {
    private final double v; private final org.nd4j.linalg.schedule.ISchedule s;
    public SpatialDropout(double p) { this.v = p; this.s = null; }
    public SpatialDropout(org.nd4j.linalg.schedule.ISchedule pSchedule) { this.v = pSchedule.valueAt(0, 0); this.s = pSchedule; }
    public org.nd4j.linalg.schedule.ISchedule schedule() { return s; }
    public int kind() { return 4; }
    public double value() { return v; }
}
