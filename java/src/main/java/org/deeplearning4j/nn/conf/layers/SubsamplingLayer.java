package org.deeplearning4j.nn.conf.layers;
public final class SubsamplingLayer {
    private SubsamplingLayer() {}
    public static final class Builder extends Layer.Builder<Builder> {
        /** MAX: B2G_LAYER_MAXPOOL (type 5, J:141-144; unpadded).  AVG / SUM / PNORM: B2G_LAYER_SUBSAMPLING (type 12), the kind in act. */
        public Builder(PoolingType t) { l.type = t == PoolingType.MAX ? 5 : 12; l.act = t == PoolingType.MAX ? 0 : t.ordinal(); }
        /** PNORM's p, a whole number >= 1, carried in act_alpha (DL4J has no default: PNORM without it is refused at b2g_net_create). */
        public Builder pnorm(int p) { l.alpha = p; l.alphaSet = true; return this; }
    }
}
