package org.deeplearning4j.nn.conf.weightnoise;
/** new DropConnect(p[, applyToBiases]), p = the retain probability of each weight (DL4J 1.0.0-beta3): W' = keep ? W : 0 in training, not rescaled. */
public final class DropConnect implements IWeightNoise {
    private final double p; private final org.nd4j.linalg.schedule.ISchedule s; private final boolean bias;
    public DropConnect(double weightRetainProbability) { this(weightRetainProbability, false); }
    public DropConnect(double weightRetainProbability, boolean applyToBiases) { this.p = weightRetainProbability; this.s = null; this.bias = applyToBiases; }
    public DropConnect(org.nd4j.linalg.schedule.ISchedule weightRetainProbSchedule) { this(weightRetainProbSchedule, false); }
    public DropConnect(org.nd4j.linalg.schedule.ISchedule weightRetainProbSchedule, boolean applyToBiases) {
        this.p = weightRetainProbSchedule.valueAt(0, 0); this.s = weightRetainProbSchedule; this.bias = applyToBiases;
    }
    public int kind() { return 1; }
    public boolean applyToBias() { return bias; }
    public double p() { return p; }
    public org.nd4j.linalg.schedule.ISchedule pSchedule() { return s; }
}
