// ComputationGraph facade: init / summary / output / fit / getLayer(..).getParam/setParam / params  (J:166-170,420,429-510).
package org.deeplearning4j.nn.graph;

import java.nio.ByteBuffer;
import java.nio.FloatBuffer;
import java.util.List;
import org.deeplearning4j.b200.Native;
import org.deeplearning4j.nn.api.layers.LayerConstraint;
import org.deeplearning4j.nn.conf.GradientNormalization;
import org.deeplearning4j.nn.conf.NeuralNetConfiguration;
import org.deeplearning4j.nn.conf.NeuralNetConfiguration.ComputationGraphConfiguration;
import org.deeplearning4j.nn.conf.distribution.Distribution;
import org.deeplearning4j.nn.conf.layers.Layer;
import org.deeplearning4j.nn.weights.WeightInit;
import org.nd4j.linalg.api.ndarray.INDArray;
import org.nd4j.linalg.dataset.DataSet;
import org.nd4j.linalg.schedule.ISchedule;

public class ComputationGraph {
    private final ComputationGraphConfiguration conf; private long net; private List<Layer> layers; private int maxBatch = Integer.getInteger("b200gan.maxBatch", 1024);
    public ComputationGraph(ComputationGraphConfiguration conf) { this.conf = conf; }

    public void init() {
        layers = conf.resolved();
        ByteBuffer cfg = Native.direct(40);
        cfg.putInt(conf.b.in.h).putInt(conf.b.in.w).putInt(conf.b.in.c).putInt(maxBatch).putInt(conf.b.g.precision)
           .putFloat(conf.b.g.clip).putFloat(1e-5f).putInt(1).putLong(conf.b.g.seed);
        ByteBuffer desc = Native.direct(Layer.DESC_BYTES * layers.size());
        for (Layer l : layers) l.write(desc, conf.b.g.act, conf.b.g.l2);
        ByteBuffer h = Native.direct(8);
        Native.check(Native.netCreate(Native.context(), Native.address(cfg), Native.address(desc), layers.size(), Native.address(h)));
        net = h.getLong(0);
        NeuralNetConfiguration.Builder g = conf.b.g;     // weightInit / dist / biasInit, resolved per layer: its own, else the global builder's
        boolean global = g.weightInit != null || g.dist != null || g.biasInit != null;
        for (Layer l : layers) {
            boolean gemm = l.type == 0 || l.type == 1 || l.type == 3 || l.type == 7;
            if (gemm && (global || l.weightInit != null || l.dist != null || l.biasInit != null))
                initWeights(l.name, l.weightInit != null ? l.weightInit : g.weightInit, l.dist != null ? l.dist : g.dist, l.biasInit != null ? l.biasInit : g.biasInit);
            if (l.type == 17 && l.weightInit != null) preluSlopeInit(l);      // PReLU: its own weightInit only (ZERO otherwise)
        }
        for (Layer l : layers) {          // l1 / l1Bias / l2Bias, resolved per layer like l2: its own, else the global builder's
            boolean reg = l.type == 0 || l.type == 1 || l.type == 3 || l.type == 7 || l.type == 17;    // PReLU's slopes are a weight
            float l1 = Float.isNaN(l.l1) ? g.l1 : l.l1, l1b = Float.isNaN(l.l1Bias) ? g.l1Bias : l.l1Bias, l2b = Float.isNaN(l.l2Bias) ? g.l2Bias : l.l2Bias;
            if (reg && (l1 != 0f || l1b != 0f || l2b != 0f)) setRegularization(l.name, l1, Float.isNaN(l.l2) ? g.l2 : l.l2, l1b, l2b);
        }
        GradientNormalization gn = conf.b.g.gradNorm;      // RenormalizeL2* / ClipL2*: on-device norms before every update
        if (gn.isL2()) Native.check(Native.netSetGradientNormalization(net, gn.ordinal(), conf.b.g.gradNormThreshold));
        for (Layer l : layers)            // new Adam(ISchedule) / RmsProp(ISchedule) / Sgd(ISchedule): evaluated on the device at every update
            if (l.updater != null && l.updater.lrSchedule() != null && hasLearningRate(l)) setLearningRate(l.name, l.updater.lrSchedule());
        for (Layer l : layers) applyConstraints(l);
        Layer last = layers.get(layers.size() - 1);     // new LossMCXENT(weights), ...: device-resident, used by every later fit
        if (last.lossWeights != null)
            Native.check(Native.netSetLossWeights(net, 0L, Native.address(Native.floats(last.lossWeights.data)), (int) last.lossWeights.length()));
        for (Layer l : layers)            // new GaussianNoise(ISchedule) etc.: evaluated on the device at every train-mode forward
            if (l.type == 11 && l.dropSchedule != null) setDropoutSchedule(l.name, l.dropSchedule);
        for (Layer l : layers) {          // DropConnect / WeightNoise: drawn on the device at every train-mode pass
            boolean gemm = l.type == 0 || l.type == 1 || l.type == 3 || l.type == 7;
            org.deeplearning4j.nn.conf.weightnoise.IWeightNoise w = l.weightNoise != null ? l.weightNoise : (l.frozen == 0 ? conf.b.g.weightNoise : null);
            if (gemm && w != null) setWeightNoise(l.name, w);
        }
    }
    /** The parameters a constrainAllParameters / constrainWeights / constrainBias list reaches on a layer (the library's rule, include/b200gan.h
     *  b2g_constraint, and engine.py constraint_params): weights = W of conv, deconv, dense and output layers, nothing on BatchNorm; bias = b
     *  where the layer has one; all = every parameter, BatchNorm's gamma, beta, mean and var included. */
    static String[] constrainedParams(Layer l, String on) {
        boolean gemm = l.type == 0 || l.type == 1 || l.type == 3 || l.type == 7;
        if (gemm && on.equals("weights")) return new String[] { "W" };
        if (gemm && on.equals("bias")) return l.hasBias != 0 ? new String[] { "b" } : new String[0];
        if (gemm && on.equals("all")) return l.hasBias != 0 ? new String[] { "b", "W" } : new String[] { "W" };
        if (l.type == 2 && on.equals("all")) return new String[] { "gamma", "beta", "mean", "var" };
        return new String[0];
    }
    /** Each tensor's list runs all-parameter, then weight, then bias constraints.  A layer whose own lists reach none of its parameters takes
     *  the global builder's lists (DL4J's NeuralNetConfiguration.Builder fills them in when the layer's resolved constraints are empty). */
    private void applyConstraints(Layer l) {
        java.util.Map<String, List<LayerConstraint>> per = constraintsByParam(l, l.constrainAll, l.constrainW, l.constrainB);
        if (per.isEmpty()) per = constraintsByParam(l, conf.b.g.constrainAll, conf.b.g.constrainW, conf.b.g.constrainB);
        for (java.util.Map.Entry<String, List<LayerConstraint>> e : per.entrySet()) {
            List<LayerConstraint> cs = e.getValue();
            ByteBuffer b = Native.direct(32 * cs.size());          // b2g_constraint[]: kind, dims_mask, max_norm, min_norm, rate (32 bytes)
            for (int i = 0; i < cs.size(); ++i) {
                LayerConstraint c = cs.get(i);
                b.putInt(32 * i, c.kind()).putInt(32 * i + 4, c.dimsMask()).putDouble(32 * i + 8, c.maxNorm()).putDouble(32 * i + 16, c.minNorm())
                 .putDouble(32 * i + 24, c.rate());
            }
            ByteBuffer name = Native.cstr(l.name), param = Native.cstr(e.getKey());
            Native.check(Native.netSetConstraints(net, Native.address(name), Native.address(param), Native.address(b), cs.size()));
            java.lang.ref.Reference.reachabilityFence(b); java.lang.ref.Reference.reachabilityFence(name); java.lang.ref.Reference.reachabilityFence(param);
        }
    }
    private static java.util.Map<String, List<LayerConstraint>> constraintsByParam(Layer l, List<LayerConstraint> all, List<LayerConstraint> w,
                                                                                   List<LayerConstraint> b) {
        List<List<LayerConstraint>> lists = java.util.Arrays.asList(all, w, b);
        String[] on = { "all", "weights", "bias" };
        java.util.Map<String, List<LayerConstraint>> per = new java.util.LinkedHashMap<>();
        for (int k = 0; k < 3; ++k)
            if (lists.get(k) != null)
                for (String p : constrainedParams(l, on[k])) for (LayerConstraint c : lists.get(k)) per.computeIfAbsent(p, x -> new java.util.ArrayList<>()).add(c);
        return per;
    }
    /** Model.applyConstraints(iteration, epoch): every constraint once, now (fit applies them after each update by itself). */
    public void applyConstraints(int iteration, int epoch) { Native.check(Native.netApplyConstraints(net)); }
    /** The library's rule (include/b200gan.h, b2g_net_set_lr_schedule): parameters, not frozen, updater neither NoOp nor AdaDelta. */
    private static boolean hasLearningRate(Layer l) {
        boolean params = l.type == 0 || l.type == 1 || l.type == 2 || l.type == 3 || l.type == 7 || l.type == 17;    // conv, deconv, BatchNorm, dense, output, PReLU
        return params && l.frozen == 0 && l.updater.kind() != 3 && l.updater.kind() != 9;
    }

    /** setLearningRate(ISchedule): every layer whose updater has a learning rate, from the next update on (null: back to the constant lr). */
    public void setLearningRate(ISchedule s) { applySchedule(null, s); }
    public void setLearningRate(String layerName, ISchedule s) { applySchedule(layerName, s); }
    /** An IDropout's ISchedule for one DropoutLayer (layerName null: every non-frozen DropoutLayer; s null: back to its constant). */
    public void setDropoutSchedule(String layerName, ISchedule s) { applySchedule(layerName, s, true); }
    /** The value (p, rate or stddev) the DropoutLayer's next train-mode forward uses. */
    public double getDropoutValue(String layerName) {
        ByteBuffer o = Native.direct(4); ByteBuffer name = Native.cstr(layerName);
        Native.check(Native.netGetDropoutValue(net, Native.address(name), Native.address(o))); return o.getFloat(0);
    }
    private void applySchedule(String layerName, ISchedule s) { applySchedule(layerName, s, false); }
    /** b2g_lr_schedule (72 bytes) of s in buf[0], a MapSchedule's keys and values in buf[1], buf[2]; all null for s null. */
    private static ByteBuffer[] scheduleStruct(ISchedule s) {
        ByteBuffer st = null, keys = null, vals = null;
        if (s != null) {
            int[] k = s.mapKeys(); double[] v = s.mapValues(); double[] p = s.parameters();
            keys = Native.direct(4 * Math.max(1, k.length)); vals = Native.direct(8 * Math.max(1, v.length));
            for (int i = 0; i < k.length; ++i) { keys.putInt(4 * i, k[i]); vals.putDouble(8 * i, v[i]); }
            st = Native.direct(72);
            st.putInt(0, s.kind()).putInt(4, s.getScheduleType().ordinal());
            for (int i = 0; i < 5; ++i) st.putDouble(8 + 8 * i, p[i]);
            st.putInt(48, k.length).putLong(56, Native.address(keys)).putLong(64, Native.address(vals));
        }
        return new ByteBuffer[] { st, keys, vals };
    }
    private void applySchedule(String layerName, ISchedule s, boolean dropout) {
        ByteBuffer[] sb = scheduleStruct(s); ByteBuffer st = sb[0];
        ByteBuffer name = layerName == null ? null : Native.cstr(layerName);
        final long nameAddr = name == null ? 0 : Native.address(name), stAddr = st == null ? 0 : Native.address(st);
        Native.check(dropout ? Native.netSetDropoutSchedule(net, nameAddr, stAddr) : Native.netSetLrSchedule(net, nameAddr, stAddr));
        java.lang.ref.Reference.reachabilityFence(sb);
        java.lang.ref.Reference.reachabilityFence(name);   // the native side reads these buffers only through their addresses
    }
    /** Layer.Builder.weightNoise after init: DropConnect or WeightNoise on one layer (layerName null: every non-frozen conv, deconv, dense and
     *  output layer; w null: none). */
    public void setWeightNoise(String layerName, org.deeplearning4j.nn.conf.weightnoise.IWeightNoise w) {
        ByteBuffer b = null; ByteBuffer[] sb = scheduleStruct(w == null ? null : w.pSchedule());
        if (w != null) {                    // b2g_weight_noise: kind, apply_to_bias, p, (pad), p_schedule, dist, a, b, additive (40 bytes)
            b = Native.direct(40);
            b.putInt(0, w.kind()).putInt(4, w.applyToBias() ? 1 : 0).putFloat(8, (float) w.p()).putLong(16, sb[0] == null ? 0 : Native.address(sb[0]));
            if (w.distribution() != null) b.putInt(24, w.distribution().kind()).putFloat(28, (float) w.distribution().a()).putFloat(32, (float) w.distribution().b());
            b.putInt(36, w.additive() ? 1 : 0);
        }
        ByteBuffer name = layerName == null ? null : Native.cstr(layerName);
        Native.check(Native.netSetWeightNoise(net, name == null ? 0 : Native.address(name), b == null ? 0 : Native.address(b)));
        java.lang.ref.Reference.reachabilityFence(b); java.lang.ref.Reference.reachabilityFence(sb); java.lang.ref.Reference.reachabilityFence(name);
    }
    /** A PReLULayer's weightInit(ZERO / ONES / DISTRIBUTION) with its dist: the slopes redrawn at init(); the global builder's is not inherited. */
    private void preluSlopeInit(Layer l) { initWeights(l.name, l.weightInit, l.dist, null); }
    /** WeightInitUtil.initWeights at init(): redraws W and sets b on one layer (layerName null: every conv, deconv, dense and output layer).
     *  w null is DL4J's default XAVIER, biasInit null its 0; DISTRIBUTION draws from d. */
    public void initWeights(String layerName, WeightInit w, Distribution d, Double biasInit) {
        ByteBuffer b = Native.direct(20);   // b2g_weight_init: scheme, dist, a, b, bias_init (20 bytes)
        b.putInt(0, (w == null ? WeightInit.XAVIER : w).ordinal()).putInt(4, d == null ? -1 : d.kind()).putFloat(8, d == null ? 0f : (float) d.a())
         .putFloat(12, d == null ? 0f : (float) d.b()).putFloat(16, biasInit == null ? 0f : biasInit.floatValue());
        ByteBuffer name = layerName == null ? null : Native.cstr(layerName);
        Native.check(Native.netInitWeights(net, name == null ? 0 : Native.address(name), Native.address(b)));
        java.lang.ref.Reference.reachabilityFence(b); java.lang.ref.Reference.reachabilityFence(name);
    }
    /** l1 / l2 on W and l1Bias / l2Bias on b of one layer (layerName null: every non-frozen conv, deconv, dense and output layer), applied
     *  after the updater from the next update on; replaces all four. */
    public void setRegularization(String layerName, float l1, float l2, float l1Bias, float l2Bias) {
        ByteBuffer b = Native.direct(16);   // b2g_regularization: l1, l2, l1_bias, l2_bias (16 bytes)
        b.putFloat(0, l1).putFloat(4, l2).putFloat(8, l1Bias).putFloat(12, l2Bias);
        ByteBuffer name = layerName == null ? null : Native.cstr(layerName);
        Native.check(Native.netSetRegularization(net, name == null ? 0 : Native.address(name), Native.address(b)));
        java.lang.ref.Reference.reachabilityFence(b); java.lang.ref.Reference.reachabilityFence(name);
    }
    /** ComputationGraph.calcL1(true) / calcL2(true): the score's regularization terms over the current parameters. */
    public double calcL1(boolean backpropParamsOnly) { return calcRegularization()[0]; }
    public double calcL2(boolean backpropParamsOnly) { return calcRegularization()[1]; }
    private double[] calcRegularization() {
        ByteBuffer o = Native.direct(16);
        Native.check(Native.netCalcRegularization(net, Native.address(o), Native.address(o) + 8)); return new double[] { o.getDouble(0), o.getDouble(8) };
    }
    /** The learning rate the layer's next update uses (its schedule's value at the current iteration / epoch, or its constant lr). */
    public double getLearningRate(String layerName) {
        ByteBuffer o = Native.direct(4); ByteBuffer name = Native.cstr(layerName);
        Native.check(Native.netGetLearningRate(net, Native.address(name), Native.address(o))); return o.getFloat(0);
    }
    /** The epoch count EPOCH schedules read.  Nothing increments it but incrementEpochCount / setEpochCount: call one at each epoch's end. */
    public int getEpochCount() { ByteBuffer o = Native.direct(8); Native.check(Native.netGetEpoch(net, Native.address(o))); return (int) o.getLong(0); }
    public void setEpochCount(int epochCount) { Native.check(Native.netSetEpoch(net, epochCount)); }
    public void incrementEpochCount() { setEpochCount(getEpochCount() + 1); }
    public long handle() { return net; }
    public ComputationGraphConfiguration configuration() { return conf; }
    /** Outputs per example of the last layer (b2g_net_output_size): 1 for a one-logit discriminator, C*H*W after a CnnLossLayer. */
    public long outputSize() { ByteBuffer o = Native.direct(8); Native.check(Native.netOutputSize(net, Native.address(o))); return o.getLong(0); }
    public long numParams() { ByteBuffer o = Native.direct(8); Native.check(Native.netNumParams(net, Native.address(o))); return o.getLong(0); }
    public String summary() { StringBuilder s = new StringBuilder("b200gan ComputationGraph, params=" + numParams() + "\n"); for (Layer l : layers) s.append("  ").append(l.name).append(" type=").append(l.type).append(" nOut=").append(l.nOut).append("\n"); return s.toString(); }

    /** output(x)[0]: inference mode (BatchNormalization uses its mean/var parameters), J:420. */
    public INDArray[] output(INDArray... x) {
        int batch = (int) x[0].shape()[0]; FloatBuffer in = Native.floats(x[0].data);
        int per = outElems(); FloatBuffer out = Native.direct(4 * batch * per).asFloatBuffer();
        Native.check(Native.netOutput(net, Native.address(in), batch, 0, Native.address(out)));
        float[] d = new float[batch * per]; out.get(d); return new INDArray[] { new INDArray(d, batch, per) };
    }
    private int outElems() { Layer last = layers.get(layers.size() - 1); return last.type == 7 ? Math.max(1, last.nOut) : last.type == 8 ? 1 : Integer.getInteger("b200gan.outElems", 784); }

    /** fit(DataSet): one minibatch = computeGradientAndScore + updater + params.subi (what SparkComputationGraph.fit reaches, SURVEY.md 3.3). */
    public void fit(DataSet ds) {
        int batch = (int) ds.getFeatures().shape()[0]; ByteBuffer score = Native.direct(4);
        INDArray mask = ds.getLabelsMaskArray();
        if (mask == null)
            Native.check(Native.netFit(net, Native.address(Native.floats(ds.getFeatures().data)), Native.address(Native.floats(ds.getLabels().data)), batch, Native.address(score)));
        else                              // the mask's width is its second dimension: 1 (per example / pixel) or nOut / C (per output)
            Native.check(Native.netFitMasked(net, Native.address(Native.floats(ds.getFeatures().data)), Native.address(Native.floats(ds.getLabels().data)), batch,
                                             Native.address(score), Native.address(Native.floats(mask.data)), mask.shape().length > 1 ? (int) mask.shape()[1] : 1));
    }
    public INDArray params() { int n = (int) numParams(); FloatBuffer b = Native.direct(4 * n).asFloatBuffer(); Native.check(Native.netGetParams(net, Native.address(b), n)); float[] d = new float[n]; b.get(d); return new INDArray(d, 1, n); }
    /** Updater state in the library's [state0 | state1] order (RmsProp cache / Adam m, then Adam v), 2 x numParams values, plus | state2
     *  (AMSGrad's v-hat) on a graph with an AMSGrad layer; the slots of every updater kind are stated at b2g_updater in include/b200gan.h. */
    public long updaterStateSize() { ByteBuffer o = Native.direct(8); Native.check(Native.netUpdaterStateSize(net, Native.address(o))); return o.getLong(0); }
    public INDArray updaterState() { int n = (int) updaterStateSize(); FloatBuffer b = Native.direct(4 * n).asFloatBuffer(); Native.check(Native.netGetUpdaterState(net, Native.address(b), n)); float[] d = new float[n]; b.get(d); return new INDArray(d, 1, n); }
    /** The layer list as JSON (this library's specification, not DL4J's Jackson schema) -- ModelSerializer's configuration.json entry. */
    public void setUpdaterState(INDArray st) { Native.check(Native.netSetUpdaterState(net, Native.address(Native.floats(st.data)), st.length())); }
    /** BaseMultiLayerUpdater's iteration count (Adam's t - 1); part of a checkpoint and of the state a Spark worker starts from. */
    public long getIterationCount() { ByteBuffer o = Native.direct(8); Native.check(Native.netGetIteration(net, Native.address(o))); return o.getLong(0); }
    public void setIterationCount(long it) { Native.check(Native.netSetIteration(net, it)); }
    /** The DropoutLayer pass counter (one per train-mode forward that masks); save it with the parameters to resume the same mask sequence. */
    public long getDropoutPass() { ByteBuffer o = Native.direct(8); Native.check(Native.netGetDropoutPass(net, Native.address(o))); return o.getLong(0); }
    public void setDropoutPass(long pass) { Native.check(Native.netSetDropoutPass(net, pass)); }
    public String configurationJson() {
        StringBuilder s = new StringBuilder("{\"format\": \"b200gan layer specs\", \"layers\": [");
        for (int i = 0; i < layers.size(); ++i) { Layer l = layers.get(i); s.append(i == 0 ? "" : ", ").append("{\"name\": \"").append(l.name).append("\", \"type\": ").append(l.type).append(", \"nIn\": ").append(l.nIn).append(", \"nOut\": ").append(l.nOut).append("}"); }
        return s.append("]}").toString();
    }
    public void setParams(INDArray p) { Native.check(Native.netSetParams(net, Native.address(Native.floats(p.data)), p.length())); }

    public LayerView getLayer(String name) { return new LayerView(name); }
    /** Layer.getParam/setParam by DL4J name ("W","b","gamma","beta","mean","var"), DL4J flattened-view order (J:429-510). */
    public final class LayerView {
        private final String name; LayerView(String n) { name = n; }
        public INDArray getParam(String key) {
            int n = paramLength(key); FloatBuffer b = Native.direct(4 * n).asFloatBuffer();
            Native.check(Native.netGetParam(net, Native.address(Native.cstr(name)), Native.address(Native.cstr(key)), Native.address(b), n));
            float[] d = new float[n]; b.get(d); return new INDArray(d, 1, n);
        }
        public void setParam(String key, INDArray v) {
            Native.check(Native.netSetParam(net, Native.address(Native.cstr(name)), Native.address(Native.cstr(key)), Native.address(Native.floats(v.data)), v.length()));
        }
        private int paramLength(String key) {
            for (Layer l : layers) if (l.name.equals(name)) {
                if (key.equals("W")) return l.nIn * l.nOut * l.kH * l.kW;
                if (key.equals("b")) return l.nOut;
                return l.nOut;   // gamma / beta / mean / var
            }
            throw new IllegalArgumentException("no layer " + name);
        }
    }
}
