package org.nd4j.linalg.dataset;
import org.nd4j.linalg.api.ndarray.INDArray;
/** new DataSet(features, labels) (J:414-421,465-466), and new DataSet(features, labels, null, labelsMask): a labels mask [mb, 1] / [mb, nOut],
 *  or [mb, 1 | C, H, W] for a CnnLossLayer (semantics at b2g_loss).  Features masks are not supported. */
public class DataSet {
    private final INDArray features, labels, labelsMask;
    public DataSet(INDArray features, INDArray labels) { this(features, labels, null, null); }
    public DataSet(INDArray features, INDArray labels, INDArray featuresMask, INDArray labelsMask) {
        if (featuresMask != null) throw new UnsupportedOperationException("features masks are not supported");
        this.features = features; this.labels = labels; this.labelsMask = labelsMask;
    }
    public INDArray getFeatures() { return features; }
    public INDArray getLabels() { return labels; }
    public INDArray getLabelsMaskArray() { return labelsMask; }
}
