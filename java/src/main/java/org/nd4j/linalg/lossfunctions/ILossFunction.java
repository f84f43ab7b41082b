package org.nd4j.linalg.lossfunctions;
import org.nd4j.linalg.api.ndarray.INDArray;
/** A loss function object (new LossMCXENT(weights), ...): the loss it runs and its per-output weights (null: none); semantics at b2g_loss. */
public interface ILossFunction {
    LossFunctions.LossFunction lossFunction();
    INDArray getWeights();
}
