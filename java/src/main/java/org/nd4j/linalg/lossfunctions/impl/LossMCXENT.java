package org.nd4j.linalg.lossfunctions.impl;
import org.nd4j.linalg.api.ndarray.INDArray;
import org.nd4j.linalg.lossfunctions.ILossFunction;
import org.nd4j.linalg.lossfunctions.LossFunctions;
/** LossMCXENT: softmax cross-entropy, with optional per-output weights (a row vector of nOut finite values; C on a CnnLossLayer). */
public class LossMCXENT implements ILossFunction {
    private final INDArray weights;
    public LossMCXENT() { this(null); }
    public LossMCXENT(INDArray weights) { this.weights = weights; }
    public LossFunctions.LossFunction lossFunction() { return LossFunctions.LossFunction.MCXENT; }
    public INDArray getWeights() { return weights; }
}
