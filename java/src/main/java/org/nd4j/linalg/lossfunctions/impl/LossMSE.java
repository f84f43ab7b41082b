package org.nd4j.linalg.lossfunctions.impl;
import org.nd4j.linalg.api.ndarray.INDArray;
import org.nd4j.linalg.lossfunctions.ILossFunction;
import org.nd4j.linalg.lossfunctions.LossFunctions;
/** LossMSE, with optional per-output weights (a row vector of nOut finite values; C on a CnnLossLayer). */
public class LossMSE implements ILossFunction {
    private final INDArray weights;
    public LossMSE() { this(null); }
    public LossMSE(INDArray weights) { this.weights = weights; }
    public LossFunctions.LossFunction lossFunction() { return LossFunctions.LossFunction.MSE; }
    public INDArray getWeights() { return weights; }
}
