// new NeuralNetConfiguration.Builder()....graphBuilder().addInputs().setInputTypes().addLayer().inputPreProcessor().setOutputs().build()  (J:118-165)
// Collects the graph (a chain, or spine plus skip vertices) into b2g_net_config + b2g_layer_desc[]; CnnToFeedForward is auto-inserted before the first dense layer after
// a convolutional one, as setInputTypes does in DL4J (SURVEY.md 3.1).
package org.deeplearning4j.nn.conf;

import java.util.ArrayList;
import java.util.HashMap;
import java.util.List;
import java.util.Map;
import org.deeplearning4j.nn.api.OptimizationAlgorithm;
import org.deeplearning4j.nn.api.layers.LayerConstraint;
import org.deeplearning4j.nn.conf.inputs.InputType;
import org.deeplearning4j.nn.conf.layers.Layer;
import org.deeplearning4j.nn.conf.preprocessor.FeedForwardToCnnPreProcessor;
import org.deeplearning4j.nn.weights.WeightInit;
import org.nd4j.linalg.activations.Activation;

public class NeuralNetConfiguration {
    public static class Builder {
        long seed = 666; float clip = 0f, l2 = 0f; Activation act = Activation.SIGMOID; int precision = Integer.getInteger("b200gan.precision", 0);
        public Builder trainingWorkspaceMode(WorkspaceMode m) { return this; }
        public Builder inferenceWorkspaceMode(WorkspaceMode m) { return this; }
        public Builder seed(long s) { seed = s; return this; }
        public Builder optimizationAlgo(OptimizationAlgorithm a) { return this; }
        /** The L2 mode (RenormalizeL2* / ClipL2*) and its threshold (DL4J's default 1.0); ClipElementWiseAbsoluteValue lives in `clip`. */
        public GradientNormalization gradNorm = GradientNormalization.None; public float gradNormThreshold = 1f;
        public Builder gradientNormalization(GradientNormalization g) {
            if (g.isL2()) { gradNorm = g; clip = 0f; return this; }
            gradNorm = GradientNormalization.None;
            if (g == GradientNormalization.None) clip = 0f; else if (clip == 0f) clip = 1f;
            return this;
        }
        public Builder gradientNormalizationThreshold(double t) { gradNormThreshold = (float) t; if (!gradNorm.isL2()) clip = (float) t; return this; }
        public Builder l2(double v) { l2 = (float) v; return this; }
        /** The global l1 (W), l1Bias and l2Bias (b): every conv, deconv, dense and output layer takes each one it does not set itself. */
        public float l1 = 0f, l1Bias = 0f, l2Bias = 0f;
        public Builder l1(double v) { l1 = (float) v; return this; }
        public Builder l1Bias(double v) { l1Bias = (float) v; return this; }
        public Builder l2Bias(double v) { l2Bias = (float) v; return this; }
        public Builder activation(Activation a) { act = a; return this; }
        /** The global weightInit / dist / biasInit (null: not given): every conv, deconv, dense and output layer takes what it does not set
         *  itself.  With none of the three given anywhere a layer keeps the library's default draw. */
        public WeightInit weightInit; public org.deeplearning4j.nn.conf.distribution.Distribution dist; public Double biasInit;
        public Builder weightInit(WeightInit w) { weightInit = w; return this; }
        public Builder dist(org.deeplearning4j.nn.conf.distribution.Distribution d) { dist = d; return this; }
        public Builder biasInit(double b) { biasInit = b; return this; }
        /** The global constraints: a layer whose own lists reach none of its parameters takes these. */
        public List<LayerConstraint> constrainAll, constrainW, constrainB;
        public Builder constrainAllParameters(LayerConstraint... c) { constrainAll = List.of(c); return this; }
        public Builder constrainWeights(LayerConstraint... c) { constrainW = List.of(c); return this; }
        public Builder constrainBias(LayerConstraint... c) { constrainB = List.of(c); return this; }
        /** The global weight noise: every non-frozen conv, deconv, dense and output layer without its own takes it. */
        public org.deeplearning4j.nn.conf.weightnoise.IWeightNoise weightNoise;
        public Builder weightNoise(org.deeplearning4j.nn.conf.weightnoise.IWeightNoise w) { weightNoise = w; return this; }
        public GraphBuilder graphBuilder() { return new GraphBuilder(this); }
    }

    public static class GraphBuilder {
        final Builder g; final List<Layer> layers = new ArrayList<>(); final Map<String, FeedForwardToCnnPreProcessor> pre = new HashMap<>(); InputType in;
        GraphBuilder(Builder g) { this.g = g; }
        public GraphBuilder setInputTypes(InputType... t) { in = t[0]; return this; }
        public GraphBuilder inputPreProcessor(String layer, FeedForwardToCnnPreProcessor p) { pre.put(layer, p); return this; }
        final Map<String, String[]> inputsOf = new HashMap<>(); final List<String> graphInputs = new ArrayList<>(); boolean hasVertex = false;
        public GraphBuilder addInputs(String... names) { for (String n : names) graphInputs.add(n); return this; }
        /** A layer's input is the entry before it (the spine); in a graph with vertices that is checked at build(). */
        public GraphBuilder addLayer(String name, Layer l, String... inputs) { l.name = name; layers.add(l); inputsOf.put(name, inputs.clone()); return this; }
        /** ElementWiseVertex / MergeVertex: one input must be the entry right before the vertex, the other an earlier one (spine plus skip). */
        public GraphBuilder addVertex(String name, Layer v, String... inputs) { v.name = name; layers.add(v); inputsOf.put(name, inputs.clone()); hasVertex = true; return this; }
        public GraphBuilder setOutputs(String... names) { return this; }
        public ComputationGraphConfiguration build() { return new ComputationGraphConfiguration(this); }
    }

    public static class ComputationGraphConfiguration {
        public final GraphBuilder b;
        ComputationGraphConfiguration(GraphBuilder b) { this.b = b; }
        /** Final layer list with the preprocessors materialised as FF_TO_CNN / CNN_TO_FF pseudo-layers. */
        public List<Layer> resolved() {
            List<Layer> out = new ArrayList<>(); boolean cnn = b.in.h * b.in.w > 1;
            for (Layer l : b.layers) {
                FeedForwardToCnnPreProcessor p = b.pre.get(l.name);
                if (p != null) { Layer r = new Layer(); r.type = 9; r.name = l.name + "_ff2cnn"; r.preH = p.h; r.preW = p.w; r.preC = p.c; r.act = 0; out.add(r); cnn = true; }
                if (cnn && (l.type == 3 || l.type == 7)) { Layer r = new Layer(); r.type = 10; r.name = l.name + "_cnn2ff"; r.act = 0; out.add(r); cnn = false; }
                out.add(l);
            }
            // A graph with vertices is resolved and checked: every layer's input must be the layer added before it (the graph input for the
            // first), so nothing sits on a skip branch, and each vertex's inputs become (skip source index in preH, input order in preW).
            // IllegalStateException for anything but spine plus skip.  Graphs without vertices are the chains they always were.
            if (!b.hasVertex) return out;
            for (int k = 0; k < b.layers.size(); ++k) {
                Layer l = b.layers.get(k); String[] ins = b.inputsOf.get(l.name);
                if (l.type == 15 || l.type == 16) continue;
                String prev = k == 0 ? null : b.layers.get(k - 1).name;
                boolean ok = ins.length == 0 || (ins.length == 1 && (k == 0 ? b.graphInputs.contains(ins[0]) : ins[0].equals(prev)));
                if (!ok) throw new IllegalStateException("layer " + l.name + ": its input must be " + (k == 0 ? "the graph input" : prev)
                                                         + " (spine plus skip; layers on a skip branch are not supported)");
            }
            for (int i = 0; i < out.size(); ++i) {
                Layer v = out.get(i); String[] ins = b.inputsOf.get(v.name);
                if (v.type != 15 && v.type != 16) continue;
                if (ins == null || ins.length != 2 || i == 0) throw new IllegalStateException("vertex " + v.name + ": needs two inputs, one of them the layer before it");
                String spine = out.get(i - 1).name; int order; String other;
                if (ins[0].equals(spine)) { order = 0; other = ins[1]; } else if (ins[1].equals(spine)) { order = 1; other = ins[0]; }
                else throw new IllegalStateException("vertex " + v.name + ": one input must be " + spine + " (spine plus skip)");
                int j = -1;
                for (int k = 0; k < i; ++k) if (out.get(k).name.equals(other)) { if (j >= 0) throw new IllegalStateException("vertex " + v.name + ": " + other + " is ambiguous"); j = k; }
                if (j < 0) throw new IllegalStateException("vertex " + v.name + ": " + other + " is not an earlier layer");
                v.preH = j; v.preW = order;
            }
            return out;
        }
    }
}
