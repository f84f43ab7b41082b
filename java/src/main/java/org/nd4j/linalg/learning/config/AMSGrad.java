package org.nd4j.linalg.learning.config;
import org.nd4j.linalg.schedule.ISchedule;
/** new AMSGrad(learningRate = 1e-3, beta1 = 0.9, beta2 = 0.999, epsilon = 1e-8): Adam's m, v; vhat = max(vhat, v); u = lr*sqrt(1-b2^t)/(1-b1^t) * m / (sqrt(vhat) + eps). */
public class AMSGrad implements IUpdater {
    public static final double DEFAULT_AMSGRAD_LEARNING_RATE = 1e-3, DEFAULT_AMSGRAD_BETA1_MEAN_DECAY = 0.9, DEFAULT_AMSGRAD_BETA2_VAR_DECAY = 0.999, DEFAULT_AMSGRAD_EPSILON = 1e-8;
    private final double lr, b1, b2, eps; private final ISchedule schedule;
    public AMSGrad() { this(DEFAULT_AMSGRAD_LEARNING_RATE); }
    public AMSGrad(double learningRate) { this(learningRate, DEFAULT_AMSGRAD_BETA1_MEAN_DECAY, DEFAULT_AMSGRAD_BETA2_VAR_DECAY, DEFAULT_AMSGRAD_EPSILON); }
    public AMSGrad(double learningRate, double beta1, double beta2, double epsilon) { lr = learningRate; b1 = beta1; b2 = beta2; eps = epsilon; schedule = null; }
    public AMSGrad(ISchedule learningRateSchedule) { this(learningRateSchedule, DEFAULT_AMSGRAD_BETA1_MEAN_DECAY, DEFAULT_AMSGRAD_BETA2_VAR_DECAY, DEFAULT_AMSGRAD_EPSILON); }
    public AMSGrad(ISchedule learningRateSchedule, double beta1, double beta2, double epsilon) { lr = learningRateSchedule.valueAt(0, 0); b1 = beta1; b2 = beta2; eps = epsilon; schedule = learningRateSchedule; }
    public int kind() { return 8; } public float lr() { return (float) lr; } public float beta1() { return (float) b1; } public float beta2() { return (float) b2; } public float eps() { return (float) eps; }
    public ISchedule lrSchedule() { return schedule; }
}
