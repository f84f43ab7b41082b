// The fused adversarial iteration (b2g_gan_step): what J:408-510 computes when dis / gan / gen share storage.
// A driver that keeps the three-graph structure works unchanged through ComputationGraph.fit/output/getParam/setParam;
// a driver that wants the fast path replaces the loop body by GanTrainer.step(...).
package org.deeplearning4j.b200;

import java.nio.ByteBuffer;
import org.deeplearning4j.nn.graph.ComputationGraph;
import org.nd4j.linalg.api.ndarray.INDArray;

public final class GanTrainer implements AutoCloseable {
    private final long gan;
    private final long disOutputs;      // labels per example the native step reads: D's output size
    public GanTrainer(ComputationGraph gen, ComputationGraph dis, boolean fakeBnTrain, boolean cudaGraph) {
        ByteBuffer h = Native.direct(8); Native.check(Native.ganCreate(gen.handle(), dis.handle(), fakeBnTrain ? 1 : 0, cudaGraph ? 1 : 0, Native.address(h))); gan = h.getLong(0);
        disOutputs = dis.outputSize();
    }
    /** [mb, outputs of D per example] labels: [mb, 1] for an OutputLayer / LossLayer discriminator, [mb, C, H, W] (NCHW) for a CnnLossLayer
     *  one; per-image labels ([mb] or [mb, 1]) are broadcast over a patch map. */
    private float[] labels(INDArray y, long mb, String name) {
        if (y.length() == mb * disOutputs) return y.data;
        if (y.length() != mb) throw new IllegalArgumentException(name + ": " + y.length() + " labels for " + mb + " examples of " + disOutputs + " outputs each");
        float[] out = new float[(int) (mb * disOutputs)];
        for (int i = 0; i < mb; ++i) java.util.Arrays.fill(out, (int) (i * disOutputs), (int) ((i + 1) * disOutputs), y.data[i]);
        return out;
    }
    /** returns {mean D loss on real, mean D loss on fake, mean G loss} */
    public float[] step(INDArray xReal, INDArray zD, INDArray zG, INDArray yReal, INDArray yFake, INDArray yGen) {
        final long mb = xReal.shape()[0];
        float[] yr = labels(yReal, mb, "yReal"), yf = labels(yFake, mb, "yFake"), yg = labels(yGen, mb, "yGen");
        ByteBuffer l = Native.direct(12);
        Native.check(Native.ganStep(gan, Native.address(Native.floats(xReal.data)), Native.address(Native.floats(zD.data)), Native.address(Native.floats(zG.data)),
            Native.address(Native.floats(yr)), Native.address(Native.floats(yf)), Native.address(Native.floats(yg)), (int) mb, Native.address(l)));
        return new float[] { l.getFloat(0), l.getFloat(4), l.getFloat(8) };
    }
    /** Labels masks of the discriminator's loss for every later step ([mb, 1] per example, or [mb, 1 | C, H, W] on a CnnLossLayer
     *  discriminator; semantics at b2g_loss); all three null clears. */
    public void setLabelMasks(INDArray mReal, INDArray mFake, INDArray mGen) {
        if (mReal == null && mFake == null && mGen == null) { Native.check(Native.ganSetLabelMasks(gan, 0L, 0L, 0L, 0, 0)); return; }
        long[] sh = mReal.shape(); int width = sh.length > 1 ? (int) sh[1] : 1;
        java.nio.FloatBuffer r = Native.floats(mReal.data), f = Native.floats(mFake.data), g = Native.floats(mGen.data);
        Native.check(Native.ganSetLabelMasks(gan, Native.address(r), Native.address(f), Native.address(g), width, (int) sh[0]));
        java.lang.ref.Reference.reachabilityFence(r); java.lang.ref.Reference.reachabilityFence(f); java.lang.ref.Reference.reachabilityFence(g);
    }
    @Override public void close() { Native.ganDestroy(gan); }
}
