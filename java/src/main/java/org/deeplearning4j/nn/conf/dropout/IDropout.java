package org.deeplearning4j.nn.conf.dropout;
/** The IDropout of a DropoutLayer (b2g_dropout_kind in include/b200gan.h): the kind carried in the desc's act and its value in act_alpha. */
public interface IDropout {
    int kind();
    double value();
    /** The ISchedule given in place of the value (DL4J's ISchedule constructors), or null. */
    default org.nd4j.linalg.schedule.ISchedule schedule() { return null; }
}
