package org.deeplearning4j.nn.conf.layers;
public final class DropoutLayer {
    private DropoutLayer() {}
    public static final class Builder extends Layer.Builder<Builder> {
        /** p = the RETAIN probability, as in DL4J 1.0.0-beta3 (new DropoutLayer.Builder(1 - 0.5)); carried in the desc's act_alpha. */
        public Builder(double p) { l.type = 11; l.alpha = (float) p; l.act = 0; }
    }
}
