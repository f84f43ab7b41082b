package org.nd4j.linalg.learning.config;
import org.nd4j.linalg.schedule.ISchedule;
/** new Nadam(learningRate = 1e-3, beta1 = 0.9, beta2 = 0.999, epsilon = 1e-8): Adam's m, v; u = lr/(1-b1^t) * (b1*m + (1-b1)*g) / (sqrt(v) + eps). */
public class Nadam implements IUpdater {
    public static final double DEFAULT_NADAM_LEARNING_RATE = 1e-3, DEFAULT_NADAM_BETA1_MEAN_DECAY = 0.9, DEFAULT_NADAM_BETA2_VAR_DECAY = 0.999, DEFAULT_NADAM_EPSILON = 1e-8;
    private final double lr, b1, b2, eps; private final ISchedule schedule;
    public Nadam() { this(DEFAULT_NADAM_LEARNING_RATE); }
    public Nadam(double learningRate) { this(learningRate, DEFAULT_NADAM_BETA1_MEAN_DECAY, DEFAULT_NADAM_BETA2_VAR_DECAY, DEFAULT_NADAM_EPSILON); }
    public Nadam(double learningRate, double beta1, double beta2, double epsilon) { lr = learningRate; b1 = beta1; b2 = beta2; eps = epsilon; schedule = null; }
    public Nadam(ISchedule learningRateSchedule) { this(learningRateSchedule, DEFAULT_NADAM_BETA1_MEAN_DECAY, DEFAULT_NADAM_BETA2_VAR_DECAY, DEFAULT_NADAM_EPSILON); }
    public Nadam(ISchedule learningRateSchedule, double beta1, double beta2, double epsilon) { lr = learningRateSchedule.valueAt(0, 0); b1 = beta1; b2 = beta2; eps = epsilon; schedule = learningRateSchedule; }
    public int kind() { return 7; } public float lr() { return (float) lr; } public float beta1() { return (float) b1; } public float beta2() { return (float) b2; } public float eps() { return (float) eps; }
    public ISchedule lrSchedule() { return schedule; }
}
