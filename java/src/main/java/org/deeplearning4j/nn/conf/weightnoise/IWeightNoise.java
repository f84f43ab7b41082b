package org.deeplearning4j.nn.conf.weightnoise;
import org.deeplearning4j.nn.conf.distribution.Distribution;
/** Layer.Builder.weightNoise / NeuralNetConfiguration.Builder.weightNoise (b2g_weight_noise in include/b200gan.h): kind 1 DropConnect, 2 WeightNoise. */
public interface IWeightNoise {
    int kind();
    boolean applyToBias();
    /** DropConnect's retain probability, or its ISchedule (null: none). */
    default double p() { return 1.0; }
    default org.nd4j.linalg.schedule.ISchedule pSchedule() { return null; }
    /** WeightNoise's distribution, and whether the noise is added (true) or multiplied. */
    default Distribution distribution() { return null; }
    default boolean additive() { return true; }
}
