package org.nd4j.linalg.lossfunctions.impl;
import org.nd4j.linalg.api.ndarray.INDArray;
import org.nd4j.linalg.lossfunctions.ILossFunction;
import org.nd4j.linalg.lossfunctions.LossFunctions;
/** LossMAE, with optional per-output weights (a row vector of nOut finite values; C on a CnnLossLayer). */
public class LossMAE implements ILossFunction {
    private final INDArray weights;
    public LossMAE() { this(null); }
    public LossMAE(INDArray weights) { this.weights = weights; }
    public LossFunctions.LossFunction lossFunction() { return LossFunctions.LossFunction.MEAN_ABSOLUTE_ERROR; }
    public INDArray getWeights() { return weights; }
}
