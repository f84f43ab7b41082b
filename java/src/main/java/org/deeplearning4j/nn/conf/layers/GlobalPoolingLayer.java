package org.deeplearning4j.nn.conf.layers;
/** GlobalPoolingLayer (B2G_LAYER_GLOBAL_POOLING, type 13): [mb, C, H, W] -> [mb, C]; the kind in act, PNORM's p in act_alpha. */
public final class GlobalPoolingLayer {
    private GlobalPoolingLayer() {}
    public static final class Builder extends Layer.Builder<Builder> {
        /** DL4J's defaults: MAX, pnorm 2. */
        public Builder() { this(PoolingType.MAX); }
        public Builder(PoolingType t) { l.type = 13; l.act = t.ordinal(); l.alpha = 2; l.alphaSet = true; }
        public Builder pnorm(int p) { l.alpha = p; l.alphaSet = true; return this; }
        /** false keeps [mb, C, 1, 1]: the same bytes as [mb, C], so both are accepted and nothing changes in the desc. */
        public Builder collapseDimensions(boolean collapse) { return this; }
    }
}
