package org.deeplearning4j.nn.conf.layers;
/** PReLULayer (B2G_LAYER_PRELU, include/b200gan.h): y = x < 0 ? alpha*x : x with learned slopes "W" (alpha), one per element of the input shape
 *  except along the shared axes.  Alpha starts at 0 (WeightInit.ZERO; the global weightInit is not inherited); weightInit(ZERO / ONES /
 *  DISTRIBUTION) on the layer redraws it at init().  Constraints and weight noise on alpha are not supported. */
public final class PReLULayer {
    private PReLULayer() {}
    public static final class Builder extends Layer.Builder<Builder> {
        public Builder() { l.type = 17; l.act = 0; l.alpha = 0f; }
        /** DL4J's inputShape: [C, H, W] or [F] (a feed-forward input); ComputationGraph.init fails with B2G_ERR_SHAPE when it is not the inferred input. */
        public Builder inputShape(long... shape) {
            if (shape.length != 1 && shape.length != 3) throw new IllegalArgumentException("PReLULayer inputShape is [C, H, W] or [F], got " + shape.length + " dimensions");
            l.preC = (int) shape[0]; l.preH = shape.length == 3 ? (int) shape[1] : 0; l.preW = shape.length == 3 ? (int) shape[2] : 0;
            return this;
        }
        /** DL4J's 1-based axes that share one slope: 1 = C (F), 2 = H, 3 = W; sharedAxes(2, 3) is one slope per channel.  Carried as a bit mask in the desc's act. */
        public Builder sharedAxes(long... axes) {
            int mask = 0;
            for (long a : axes) {
                if (a < 1 || a > 3) throw new IllegalArgumentException("PReLULayer shared axis " + a + ": DL4J's axes are 1 (C), 2 (H) and 3 (W)");
                mask |= 1 << (a - 1);
            }
            l.act = mask;
            return this;
        }
    }
}
