package org.deeplearning4j.nn.conf.layers;
public final class DropoutLayer {
    private DropoutLayer() {}
    public static final class Builder extends Layer.Builder<Builder> {
        /** p = the RETAIN probability, as in DL4J 1.0.0-beta3 (new DropoutLayer.Builder(1 - 0.5)); carried in the desc's act_alpha. */
        public Builder(double p) { l.type = 11; l.alpha = (float) p; l.act = 0; }
        /** DropoutLayer.Builder(IDropout): GaussianDropout, GaussianNoise, AlphaDropout, SpatialDropout or Dropout; the kind in act, its value in act_alpha. */
        public Builder(org.deeplearning4j.nn.conf.dropout.IDropout d) {
            l.type = 11; l.act = d.kind(); l.dropSchedule = d.schedule();
            l.alpha = (float) (d.schedule() != null ? d.schedule().valueAt(0, 0) : d.value());    // a schedule's value at 0, as for a scheduled lr
        }
    }
}
