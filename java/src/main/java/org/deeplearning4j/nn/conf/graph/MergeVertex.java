// new MergeVertex(): B2G_LAYER_MERGE, the two inputs concatenated along dimension 1 in input order (GraphBuilder.addVertex).
package org.deeplearning4j.nn.conf.graph;

import org.deeplearning4j.nn.conf.layers.Layer;

public class MergeVertex extends Layer {
    public MergeVertex() { type = 16; act = 0; }
}
