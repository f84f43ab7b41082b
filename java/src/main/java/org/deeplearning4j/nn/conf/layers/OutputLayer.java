package org.deeplearning4j.nn.conf.layers;
public final class OutputLayer {
    private OutputLayer() {}
    public static final class Builder extends Layer.Builder<Builder> {
        // XENT+sigmoid (J:159-163) and MCXENT+softmax (J:357-362) imply their activation; the other losses apply .activation(..), identity by default
        public Builder(org.nd4j.linalg.lossfunctions.LossFunctions.LossFunction f) { l.type = 7; l.loss = f.code; l.act = 0; }
        /** new LossMCXENT(weights), new LossMSE(weights), ...: the loss and its per-output weights. */
        public Builder(org.nd4j.linalg.lossfunctions.ILossFunction f) { this(f.lossFunction()); l.lossWeights = f.getWeights(); }
        
    }
}
