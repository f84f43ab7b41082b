// new TransferLearning.GraphBuilder(net).fineTuneConfiguration(..).setFeatureExtractor("dis_dense_layer_6")
//     .removeVertexKeepConnections("dis_output_layer_7").addLayer(..).addLayer(..).build()   (J:337-364)
// Layers up to and including the feature-extractor vertex are marked frozen (b2g_layer_desc.frozen: test-mode forward, no gradient, no
// update); the new graph is a fresh b2g_net whose trunk parameters the driver fills with getParam/setParam (J:516-542), as it does today.
package org.deeplearning4j.nn.transferlearning;

import java.util.ArrayList;
import java.util.List;
import org.deeplearning4j.nn.conf.NeuralNetConfiguration;
import org.deeplearning4j.nn.conf.layers.Layer;
import org.deeplearning4j.nn.graph.ComputationGraph;

public final class TransferLearning {
    private TransferLearning() {}
    public static class GraphBuilder {
        private final ComputationGraph src; private FineTuneConfiguration ft; private String frozenUpTo; private final List<String> removed = new ArrayList<>(); private final List<Layer> added = new ArrayList<>();
        public GraphBuilder(ComputationGraph origGraph) { src = origGraph; }
        public GraphBuilder fineTuneConfiguration(FineTuneConfiguration c) { ft = c; return this; }
        public GraphBuilder setFeatureExtractor(String... vertices) { frozenUpTo = vertices[vertices.length - 1]; return this; }
        public GraphBuilder removeVertexKeepConnections(String name) { removed.add(name); return this; }
        public GraphBuilder addLayer(String name, Layer l, String... inputs) { l.name = name; added.add(l); return this; }
        public ComputationGraph build() {
            NeuralNetConfiguration.Builder b = new NeuralNetConfiguration.Builder().seed(ft.seed).gradientNormalizationThreshold(ft.clip).l2(ft.l2).l1(ft.l1).l1Bias(ft.l1Bias).l2Bias(ft.l2Bias).activation(ft.act);
            if (ft.gradNorm.isL2()) b.gradientNormalization(ft.gradNorm).gradientNormalizationThreshold(ft.gradNormThreshold);
            NeuralNetConfiguration.GraphBuilder g = b.graphBuilder().setInputTypes(src.configuration().b.in);
            boolean frozen = frozenUpTo != null;
            for (Layer l : src.configuration().b.layers) {
                if (removed.contains(l.name)) continue;
                Layer c = l.copy(); c.frozen = frozen ? 1 : 0; g.addLayer(c.name, c);
                if (l.name.equals(frozenUpTo)) frozen = false;
            }
            for (Layer l : added) { if (l.updater == null) l.updater = ft.updater; g.addLayer(l.name, l); }
            ComputationGraph out = new ComputationGraph(g.build()); out.init(); return out;
        }
    }
}
