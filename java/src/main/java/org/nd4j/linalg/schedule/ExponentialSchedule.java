package org.nd4j.linalg.schedule;
/** initialValue * gamma^i. */
public class ExponentialSchedule implements ISchedule {
    private final ScheduleType type; private final double initialValue, gamma;
    public ExponentialSchedule(ScheduleType scheduleType, double initialValue, double gamma) { type = scheduleType; this.initialValue = initialValue; this.gamma = gamma; }
    public double valueAt(int iteration, int epoch) { int i = type == ScheduleType.ITERATION ? iteration : epoch; return initialValue * Math.pow(gamma, i); }
    public ScheduleType getScheduleType() { return type; }
    public int kind() { return 1; }
    public double[] parameters() { return new double[] { initialValue, gamma, 0, 0, 0 }; }
}
