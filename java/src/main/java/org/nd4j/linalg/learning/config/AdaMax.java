package org.nd4j.linalg.learning.config;
import org.nd4j.linalg.schedule.ISchedule;
/** new AdaMax(learningRate = 1e-3, beta1 = 0.9, beta2 = 0.999, epsilon = 1e-8): m = b1*m + (1-b1)*g; u_inf = max(b2*u_inf, |g|) + 1e-32; u = lr/(1-b1^t) * m / u_inf (epsilon unused). */
public class AdaMax implements IUpdater {
    public static final double DEFAULT_ADAMAX_LEARNING_RATE = 1e-3, DEFAULT_ADAMAX_BETA1_MEAN_DECAY = 0.9, DEFAULT_ADAMAX_BETA2_VAR_DECAY = 0.999, DEFAULT_ADAMAX_EPSILON = 1e-8;
    private final double lr, b1, b2, eps; private final ISchedule schedule;
    public AdaMax() { this(DEFAULT_ADAMAX_LEARNING_RATE); }
    public AdaMax(double learningRate) { this(learningRate, DEFAULT_ADAMAX_BETA1_MEAN_DECAY, DEFAULT_ADAMAX_BETA2_VAR_DECAY, DEFAULT_ADAMAX_EPSILON); }
    public AdaMax(double learningRate, double beta1, double beta2, double epsilon) { lr = learningRate; b1 = beta1; b2 = beta2; eps = epsilon; schedule = null; }
    public AdaMax(ISchedule learningRateSchedule) { this(learningRateSchedule, DEFAULT_ADAMAX_BETA1_MEAN_DECAY, DEFAULT_ADAMAX_BETA2_VAR_DECAY, DEFAULT_ADAMAX_EPSILON); }
    public AdaMax(ISchedule learningRateSchedule, double beta1, double beta2, double epsilon) { lr = learningRateSchedule.valueAt(0, 0); b1 = beta1; b2 = beta2; eps = epsilon; schedule = learningRateSchedule; }
    public int kind() { return 6; } public float lr() { return (float) lr; } public float beta1() { return (float) b1; } public float beta2() { return (float) b2; } public float eps() { return (float) eps; }
    public ISchedule lrSchedule() { return schedule; }
}
