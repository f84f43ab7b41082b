// Base of the layer-configuration builders: collects exactly the fields of b2g_layer_desc (include/b200gan.h).
package org.deeplearning4j.nn.conf.layers;

import java.nio.ByteBuffer;
import java.util.List;
import org.deeplearning4j.nn.api.layers.LayerConstraint;
import org.nd4j.linalg.activations.Activation;
import org.nd4j.linalg.activations.IActivation;
import org.nd4j.linalg.learning.config.IUpdater;

public class Layer {
    public static final int DESC_BYTES = 4 + 64 + 4 * 2 + 4 * 6 + 4 + 4 + 4 + 4 + 4 * 4 + 4 + 4 * 2 + 4 * 3 + 4 * 2;   // == sizeof(b2g_layer_desc) = 164
    public int type, nIn, nOut, kH = 1, kW = 1, sH = 1, sW = 1, pH, pW, hasBias = 1, act = -1, preH, preW, preC, loss, frozen;
    public float alpha = 0.01f, l2 = Float.NaN, bnDecay = 0.9f, bnEps = 1e-5f;
    /** l1 (W), l1Bias and l2Bias (b); NaN: the global builder's.  Applied by ComputationGraph.init (l2 travels in the desc). */
    public float l1 = Float.NaN, l1Bias = Float.NaN, l2Bias = Float.NaN;
    public IUpdater updater; public String name = "";
    public org.nd4j.linalg.schedule.ISchedule dropSchedule;   // DropoutLayer.Builder(IDropout) with an ISchedule: applied by ComputationGraph.init
    public org.deeplearning4j.nn.conf.weightnoise.IWeightNoise weightNoise;   // Layer.Builder.weightNoise (null: the global builder's): applied by ComputationGraph.init
    /** Layer.Builder.weightInit / dist / biasInit (null: the global builder's): applied by ComputationGraph.init. */
    public org.deeplearning4j.nn.weights.WeightInit weightInit; public org.deeplearning4j.nn.conf.distribution.Distribution dist; public Double biasInit;
    /** constrainAllParameters / constrainWeights / constrainBias; all null: the global builder's lists apply. */
    public List<LayerConstraint> constrainAll, constrainW, constrainB;
    public boolean alphaSet;   // alpha given by leakyReluAlpha(..) or activation(IActivation); else ELU / ThresholdedReLU write DL4J's 1.0
    /** The loss's per-output weights of an OutputLayer / LossLayer / CnnLossLayer built from an ILossFunction (null: none): applied by ComputationGraph.init. */
    public org.nd4j.linalg.api.ndarray.INDArray lossWeights;

    /** Serialise into the C struct layout (little-endian, no padding: every field is 4-byte aligned). */
    public void write(ByteBuffer b, Activation globalAct, float globalL2) {
        b.putInt(type); byte[] nm = name.getBytes(java.nio.charset.StandardCharsets.US_ASCII); byte[] fixed = new byte[64]; System.arraycopy(nm, 0, fixed, 0, Math.min(63, nm.length)); b.put(fixed);
        b.putInt(nIn).putInt(nOut).putInt(kH).putInt(kW).putInt(sH).putInt(sW).putInt(pH).putInt(pW).putInt(hasBias);
        final int a = act >= 0 ? act : defaultAct(globalAct);
        b.putInt(a).putFloat(!alphaSet && (a == Activation.ELU.code || a == Activation.THRESHOLDEDRELU.code) ? 1.0f : alpha);
        b.putInt(updater == null ? 0 : updater.kind()).putFloat(updater == null ? 0f : updater.lr()).putFloat(updater == null ? 0f : updater.beta1()).putFloat(updater == null ? 0f : updater.beta2()).putFloat(updater == null ? 1e-8f : updater.eps());
        b.putFloat(Float.isNaN(l2) ? globalL2 : l2).putFloat(bnDecay).putFloat(bnEps).putInt(preH).putInt(preW).putInt(preC).putInt(loss).putInt(frozen);
    }
    public Layer copy() { Layer c = new Layer(); c.type = type; c.nIn = nIn; c.nOut = nOut; c.kH = kH; c.kW = kW; c.sH = sH; c.sW = sW; c.pH = pH; c.pW = pW; c.hasBias = hasBias; c.act = act;
        c.preH = preH; c.preW = preW; c.preC = preC; c.loss = loss; c.frozen = frozen; c.alpha = alpha; c.l2 = l2; c.l1 = l1; c.l1Bias = l1Bias; c.l2Bias = l2Bias; c.bnDecay = bnDecay; c.bnEps = bnEps; c.updater = updater; c.name = name; c.alphaSet = alphaSet;
        c.constrainAll = constrainAll; c.constrainW = constrainW; c.constrainB = constrainB; c.dropSchedule = dropSchedule; c.weightNoise = weightNoise;
        c.weightInit = weightInit; c.dist = dist; c.biasInit = biasInit; c.lossWeights = lossWeights; return c; }
    protected int defaultAct(Activation g) { return g.code; }   // conv / dense inherit the global .activation(..) (J:126)

    @SuppressWarnings("unchecked")
    public abstract static class Builder<T extends Builder<T>> {
        protected final Layer l = new Layer();
        public T nIn(int n) { l.nIn = n; return (T) this; }
        public T nOut(int n) { l.nOut = n; return (T) this; }
        public T stride(int h, int w) { l.sH = h; l.sW = w; return (T) this; }
        public T padding(int h, int w) { l.pH = h; l.pW = w; return (T) this; }
        public T kernelSize(int h, int w) { l.kH = h; l.kW = w; return (T) this; }
        public T hasBias(boolean b) { l.hasBias = b ? 1 : 0; return (T) this; }
        public T updater(IUpdater u) { l.updater = u; return (T) this; }
        public T activation(Activation a) { l.act = a.code; return (T) this; }
        public T activation(IActivation a) { l.act = a.code(); l.alpha = a.alpha(); l.alphaSet = true; return (T) this; }   // ActivationELU(alpha), ActivationThresholdedReLU(theta)
        public T leakyReluAlpha(double a) { l.alpha = (float) a; l.alphaSet = true; return (T) this; }
        public T l2(double v) { l.l2 = (float) v; return (T) this; }
        public T l1(double v) { l.l1 = (float) v; return (T) this; }
        public T l1Bias(double v) { l.l1Bias = (float) v; return (T) this; }
        public T l2Bias(double v) { l.l2Bias = (float) v; return (T) this; }
        public T constrainAllParameters(LayerConstraint... c) { l.constrainAll = List.of(c); return (T) this; }
        public T constrainWeights(LayerConstraint... c) { l.constrainW = List.of(c); return (T) this; }
        public T constrainBias(LayerConstraint... c) { l.constrainB = List.of(c); return (T) this; }
        public T weightNoise(org.deeplearning4j.nn.conf.weightnoise.IWeightNoise w) { l.weightNoise = w; return (T) this; }
        public T weightInit(org.deeplearning4j.nn.weights.WeightInit w) { l.weightInit = w; return (T) this; }
        public T dist(org.deeplearning4j.nn.conf.distribution.Distribution d) { l.dist = d; return (T) this; }
        public T biasInit(double b) { l.biasInit = b; return (T) this; }
        public Layer build() { return l; }
    }
}
