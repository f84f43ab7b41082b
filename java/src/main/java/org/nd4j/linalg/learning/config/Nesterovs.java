package org.nd4j.linalg.learning.config;
import org.nd4j.linalg.schedule.ISchedule;
/** new Nesterovs(learningRate = 0.1, momentum = 0.9): v = mu*v - lr*g; u = mu*vPrev - (1+mu)*v.  Momentum goes in beta1; momentum schedules
 *  are not supported. */
public class Nesterovs implements IUpdater {
    public static final double DEFAULT_NESTEROV_LEARNING_RATE = 0.1, DEFAULT_NESTEROV_MOMENTUM = 0.9;
    private final double lr, momentum; private final ISchedule schedule;
    public Nesterovs() { this(DEFAULT_NESTEROV_LEARNING_RATE, DEFAULT_NESTEROV_MOMENTUM); }
    public Nesterovs(double momentum) { this(DEFAULT_NESTEROV_LEARNING_RATE, momentum); }
    public Nesterovs(double learningRate, double momentum) { lr = learningRate; this.momentum = momentum; schedule = null; }
    public Nesterovs(ISchedule learningRateSchedule) { this(learningRateSchedule, DEFAULT_NESTEROV_MOMENTUM); }
    public Nesterovs(ISchedule learningRateSchedule, double momentum) { lr = learningRateSchedule.valueAt(0, 0); this.momentum = momentum; schedule = learningRateSchedule; }
    public int kind() { return 4; } public float lr() { return (float) lr; } public float beta1() { return (float) momentum; } public float beta2() { return 0f; } public float eps() { return 0f; }
    public ISchedule lrSchedule() { return schedule; }
}
