package org.nd4j.linalg.lossfunctions.impl;
import org.nd4j.linalg.api.ndarray.INDArray;
import org.nd4j.linalg.lossfunctions.ILossFunction;
import org.nd4j.linalg.lossfunctions.LossFunctions;
/** LossL2, with optional per-output weights (a row vector of nOut finite values; C on a CnnLossLayer). */
public class LossL2 implements ILossFunction {
    private final INDArray weights;
    public LossL2() { this(null); }
    public LossL2(INDArray weights) { this.weights = weights; }
    public LossFunctions.LossFunction lossFunction() { return LossFunctions.LossFunction.L2; }
    public INDArray getWeights() { return weights; }
}
