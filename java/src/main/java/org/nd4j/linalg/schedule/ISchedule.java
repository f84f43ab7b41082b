package org.nd4j.linalg.schedule;
/** A learning-rate schedule (DL4J 1.0.0-beta3 org.nd4j.linalg.schedule).  The library evaluates it on the device at every update
 *  (include/b200gan.h, b2g_lr_schedule); valueAt is the same arithmetic in Java.  kind() is the b2g_schedule_kind, parameters() the struct's
 *  {initial, gamma, power, step, decay_rate}. */
public interface ISchedule {
    double valueAt(int iteration, int epoch);
    ScheduleType getScheduleType();
    int kind();
    double[] parameters();
    default int[] mapKeys() { return new int[0]; }
    default double[] mapValues() { return new double[0]; }
}
