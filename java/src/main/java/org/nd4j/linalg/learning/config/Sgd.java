package org.nd4j.linalg.learning.config;
import org.nd4j.linalg.schedule.ISchedule;
/** new Sgd(learningRate) / new Sgd(ISchedule): u = lr * g. */
public class Sgd implements IUpdater {
    private final double lr; private final ISchedule schedule;
    public Sgd(double learningRate) { lr = learningRate; schedule = null; }
    public Sgd(ISchedule learningRateSchedule) { lr = learningRateSchedule.valueAt(0, 0); schedule = learningRateSchedule; }
    public int kind() { return 0; } public float lr() { return (float) lr; } public float beta1() { return 0f; } public float beta2() { return 0f; } public float eps() { return 1e-8f; }
    public ISchedule lrSchedule() { return schedule; }
}
