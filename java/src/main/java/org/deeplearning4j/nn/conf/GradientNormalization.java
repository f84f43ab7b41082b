package org.deeplearning4j.nn.conf;
// DL4J's order: the ordinals are the library's b2g_gradient_normalization values.  ClipElementWiseAbsoluteValue is b2g_net_config.grad_clip;
// the four L2 modes go through b2g_net_set_gradient_normalization (ComputationGraph.init).
public enum GradientNormalization {
    None, RenormalizeL2PerLayer, RenormalizeL2PerParamType, ClipElementWiseAbsoluteValue, ClipL2PerLayer, ClipL2PerParamType;
    /** RenormalizeL2* / ClipL2*: normalized on the device from the L2 norm of the layer's or the parameter's gradient. */
    public boolean isL2() { return this != None && this != ClipElementWiseAbsoluteValue; }
}
