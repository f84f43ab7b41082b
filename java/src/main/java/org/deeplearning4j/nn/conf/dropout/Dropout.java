package org.deeplearning4j.nn.conf.dropout;
/** new Dropout(p), p = the RETAIN probability in (0, 1] (DL4J 1.0.0-beta3). */
public final class Dropout implements IDropout {
    private final double v; private final org.nd4j.linalg.schedule.ISchedule s;
    public Dropout(double p) { this.v = p; this.s = null; }
    public Dropout(org.nd4j.linalg.schedule.ISchedule pSchedule) { this.v = pSchedule.valueAt(0, 0); this.s = pSchedule; }
    public org.nd4j.linalg.schedule.ISchedule schedule() { return s; }
    public int kind() { return 0; }
    public double value() { return v; }
}
