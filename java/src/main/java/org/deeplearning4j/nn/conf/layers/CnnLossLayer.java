package org.deeplearning4j.nn.conf.layers;
/** CnnLossLayer (B2G_LAYER_CNN_LOSS, type 14): the loss on every pixel of a [mb, C, H, W] map, labels [mb, C, H, W]; no parameters. */
public final class CnnLossLayer {
    public static final int TYPE = 14;
    private CnnLossLayer() {}
    public static final class Builder extends Layer.Builder<Builder> {
        // XENT implies a sigmoid per element and MCXENT a softmax over the channels of each pixel; the other losses apply .activation(..),
        // identity by default
        public Builder(org.nd4j.linalg.lossfunctions.LossFunctions.LossFunction f) { l.type = TYPE; l.loss = f.code; l.act = 0; }
        /** new LossMCXENT(weights), ...: the loss and its per-channel weights. */
        public Builder(org.nd4j.linalg.lossfunctions.ILossFunction f) { this(f.lossFunction()); l.lossWeights = f.getWeights(); }
    }
}
