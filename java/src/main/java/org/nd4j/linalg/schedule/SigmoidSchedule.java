package org.nd4j.linalg.schedule;
/** initialValue / (1 + exp(-gamma * (i - stepSize))). */
public class SigmoidSchedule implements ISchedule {
    private final ScheduleType type; private final double initialValue, gamma; private final int stepSize;
    public SigmoidSchedule(ScheduleType scheduleType, double initialValue, double gamma, int stepSize) { type = scheduleType; this.initialValue = initialValue; this.gamma = gamma; this.stepSize = stepSize; }
    public double valueAt(int iteration, int epoch) { int i = type == ScheduleType.ITERATION ? iteration : epoch; return initialValue / (1.0 + Math.exp(-gamma * (i - stepSize))); }
    public ScheduleType getScheduleType() { return type; }
    public int kind() { return 3; }
    public double[] parameters() { return new double[] { initialValue, gamma, 0, stepSize, 0 }; }
}
