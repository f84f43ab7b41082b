package org.deeplearning4j.nn.conf.layers;
public final class LossLayer {
    private LossLayer() {}
    public static final class Builder extends Layer.Builder<Builder> {
        // XENT implies the sigmoid; the losses other than XENT and MCXENT apply .activation(..), identity by default
        public Builder(org.nd4j.linalg.lossfunctions.LossFunctions.LossFunction f) { l.type = 8; l.loss = f.code; l.act = 0; }
        /** new LossMCXENT(weights), new LossMSE(weights), ...: the loss and its per-output weights. */
        public Builder(org.nd4j.linalg.lossfunctions.ILossFunction f) { this(f.lossFunction()); l.lossWeights = f.getWeights(); }
        
    }
}
