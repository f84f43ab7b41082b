package org.nd4j.linalg.learning.config;
import org.nd4j.linalg.schedule.ISchedule;
/** new AdaGrad(learningRate = 0.1, epsilon = 1e-6): h = h + g^2 (h starts at epsilon); u = lr*g / (sqrt(h) + eps). */
public class AdaGrad implements IUpdater {
    public static final double DEFAULT_ADAGRAD_LEARNING_RATE = 0.1, DEFAULT_ADAGRAD_EPSILON = 1e-6;
    private final double lr, eps; private final ISchedule schedule;
    public AdaGrad() { this(DEFAULT_ADAGRAD_LEARNING_RATE, DEFAULT_ADAGRAD_EPSILON); }
    public AdaGrad(double learningRate) { this(learningRate, DEFAULT_ADAGRAD_EPSILON); }
    public AdaGrad(double learningRate, double epsilon) { lr = learningRate; eps = epsilon; schedule = null; }
    public AdaGrad(ISchedule learningRateSchedule) { this(learningRateSchedule, DEFAULT_ADAGRAD_EPSILON); }
    public AdaGrad(ISchedule learningRateSchedule, double epsilon) { lr = learningRateSchedule.valueAt(0, 0); eps = epsilon; schedule = learningRateSchedule; }
    public int kind() { return 5; } public float lr() { return (float) lr; } public float beta1() { return 0f; } public float beta2() { return 0f; } public float eps() { return (float) eps; }
    public ISchedule lrSchedule() { return schedule; }
}
