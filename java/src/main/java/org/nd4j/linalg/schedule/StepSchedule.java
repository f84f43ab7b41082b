package org.nd4j.linalg.schedule;
/** initialValue * decayRate^floor(i / step). */
public class StepSchedule implements ISchedule {
    private final ScheduleType type; private final double initialValue, decayRate, step;
    public StepSchedule(ScheduleType scheduleType, double initialValue, double decayRate, double step) { type = scheduleType; this.initialValue = initialValue; this.decayRate = decayRate; this.step = step; }
    public double valueAt(int iteration, int epoch) { int i = type == ScheduleType.ITERATION ? iteration : epoch; return initialValue * Math.pow(decayRate, Math.floor(i / step)); }
    public ScheduleType getScheduleType() { return type; }
    public int kind() { return 4; }
    public double[] parameters() { return new double[] { initialValue, 0, 0, step, decayRate }; }
}
