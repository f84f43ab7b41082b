package org.nd4j.linalg.learning.config;
import org.nd4j.linalg.schedule.ISchedule;
/** new RmsProp(learningRate, rmsDecay, epsilon) -- the reference passes (lr, 1e-8, 1e-8) (J:133): rmsDecay=1e-8. */
public class RmsProp implements IUpdater {
    private final double lr, decay, eps; private final ISchedule schedule;
    public RmsProp(double lr, double rmsDecay, double epsilon) { this.lr = lr; this.decay = rmsDecay; this.eps = epsilon; schedule = null; }
    public RmsProp(ISchedule learningRateSchedule) { this(learningRateSchedule, 0.95, 1e-8); }
    public RmsProp(ISchedule learningRateSchedule, double rmsDecay, double epsilon) { lr = learningRateSchedule.valueAt(0, 0); decay = rmsDecay; eps = epsilon; schedule = learningRateSchedule; }
    public int kind() { return 1; } public float lr() { return (float) lr; } public float beta1() { return (float) decay; } public float beta2() { return 0f; } public float eps() { return (float) eps; }
    public ISchedule lrSchedule() { return schedule; }
}
