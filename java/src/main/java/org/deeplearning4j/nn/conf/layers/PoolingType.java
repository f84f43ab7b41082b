package org.deeplearning4j.nn.conf.layers;
/** The ordinal is the b2g_pooling code the layer builders write into the desc's act (include/b200gan.h). */
public enum PoolingType { MAX, AVG, SUM, PNORM }
