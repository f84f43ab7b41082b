package org.nd4j.linalg.learning.config;
import org.nd4j.linalg.schedule.ISchedule;
public class Adam implements IUpdater {
    private final double lr, b1, b2, eps; private final ISchedule schedule;
    public Adam(double lr) { this(lr, 0.9, 0.999, 1e-8); }
    public Adam(double lr, double beta1, double beta2, double epsilon) { this.lr = lr; b1 = beta1; b2 = beta2; eps = epsilon; schedule = null; }
    public Adam(ISchedule learningRateSchedule) { this(learningRateSchedule, 0.9, 0.999, 1e-8); }
    public Adam(ISchedule learningRateSchedule, double beta1, double beta2, double epsilon) { lr = learningRateSchedule.valueAt(0, 0); b1 = beta1; b2 = beta2; eps = epsilon; schedule = learningRateSchedule; }
    public int kind() { return 2; } public float lr() { return (float) lr; } public float beta1() { return (float) b1; } public float beta2() { return (float) b2; } public float eps() { return (float) eps; }
    public ISchedule lrSchedule() { return schedule; }
}
