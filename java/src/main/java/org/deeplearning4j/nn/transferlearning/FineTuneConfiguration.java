// new FineTuneConfiguration.Builder()....build() (J:338-349): the hyper-parameters applied to the NEW (unfrozen) layers.
package org.deeplearning4j.nn.transferlearning;

import org.deeplearning4j.nn.api.OptimizationAlgorithm;
import org.deeplearning4j.nn.conf.GradientNormalization;
import org.deeplearning4j.nn.conf.WorkspaceMode;
import org.deeplearning4j.nn.weights.WeightInit;
import org.nd4j.linalg.activations.Activation;
import org.nd4j.linalg.learning.config.IUpdater;

public class FineTuneConfiguration {
    public float clip, l2, l1, l1Bias, l2Bias; public GradientNormalization gradNorm = GradientNormalization.None; public float gradNormThreshold = 1f; public Activation act = Activation.TANH; public IUpdater updater; public long seed = 666;
    public static class Builder {
        private final FineTuneConfiguration c = new FineTuneConfiguration();
        public Builder trainingWorkspaceMode(WorkspaceMode m) { return this; }
        public Builder inferenceWorkspaceMode(WorkspaceMode m) { return this; }
        public Builder optimizationAlgo(OptimizationAlgorithm a) { return this; }
        public Builder gradientNormalization(GradientNormalization g) {
            if (g.isL2()) { c.gradNorm = g; c.clip = 0f; return this; }
            c.gradNorm = GradientNormalization.None; if (c.clip == 0f && g != GradientNormalization.None) c.clip = 1f; return this;
        }
        public Builder gradientNormalizationThreshold(double t) { c.gradNormThreshold = (float) t; if (!c.gradNorm.isL2()) c.clip = (float) t; return this; }
        public Builder activation(Activation a) { c.act = a; return this; }
        public Builder l2(double v) { c.l2 = (float) v; return this; }
        public Builder l1(double v) { c.l1 = (float) v; return this; }
        public Builder l1Bias(double v) { c.l1Bias = (float) v; return this; }
        public Builder l2Bias(double v) { c.l2Bias = (float) v; return this; }
        public Builder weightInit(WeightInit w) { return this; }
        public Builder updater(IUpdater u) { c.updater = u; return this; }
        public Builder seed(long s) { c.seed = s; return this; }
        public FineTuneConfiguration build() { return c; }
    }
}
