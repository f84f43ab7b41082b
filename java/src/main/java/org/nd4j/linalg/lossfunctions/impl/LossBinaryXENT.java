package org.nd4j.linalg.lossfunctions.impl;
import org.nd4j.linalg.api.ndarray.INDArray;
import org.nd4j.linalg.lossfunctions.ILossFunction;
import org.nd4j.linalg.lossfunctions.LossFunctions;
/** LossBinaryXENT: sigmoid cross-entropy, with optional per-output weights (a row vector of nOut finite values; C on a CnnLossLayer). */
public class LossBinaryXENT implements ILossFunction {
    private final INDArray weights;
    public LossBinaryXENT() { this(null); }
    public LossBinaryXENT(INDArray weights) { this.weights = weights; }
    public LossFunctions.LossFunction lossFunction() { return LossFunctions.LossFunction.XENT; }
    public INDArray getWeights() { return weights; }
}
