package org.nd4j.linalg.schedule;
/** initialValue / (1 + gamma * i)^power. */
public class InverseSchedule implements ISchedule {
    private final ScheduleType type; private final double initialValue, gamma, power;
    public InverseSchedule(ScheduleType scheduleType, double initialValue, double gamma, double power) { type = scheduleType; this.initialValue = initialValue; this.gamma = gamma; this.power = power; }
    public double valueAt(int iteration, int epoch) { int i = type == ScheduleType.ITERATION ? iteration : epoch; return initialValue / Math.pow(1 + gamma * i, power); }
    public ScheduleType getScheduleType() { return type; }
    public int kind() { return 2; }
    public double[] parameters() { return new double[] { initialValue, gamma, power, 0, 0 }; }
}
