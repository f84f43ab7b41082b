package org.nd4j.linalg.lossfunctions;
public final class LossFunctions {
    /** The losses the library runs; code = b2g_loss (include/b200gan.h), written into b2g_layer_desc.loss. */
    public enum LossFunction {
        XENT(0), MCXENT(1), MSE(2), L1(3), L2(4), MEAN_ABSOLUTE_ERROR(5), HINGE(6), SQUARED_HINGE(7), WASSERSTEIN(8);
        public final int code;
        LossFunction(int code) { this.code = code; }
    }
    private LossFunctions() {}
}
