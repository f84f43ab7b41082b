// new ElementWiseVertex(ElementWiseVertex.Op.Add): B2G_LAYER_ELEMENTWISE, the op in act (b2g_elementwise_op, DL4J's Op order).  Added with
// GraphBuilder.addVertex(name, vertex, inputs...): one input must be the layer right before it, the other an earlier layer.
package org.deeplearning4j.nn.conf.graph;

import org.deeplearning4j.nn.conf.layers.Layer;

public class ElementWiseVertex extends Layer {
    public enum Op { Add, Subtract, Product, Average, Max }
    public ElementWiseVertex(Op op) { type = 15; act = op.ordinal(); }
}
