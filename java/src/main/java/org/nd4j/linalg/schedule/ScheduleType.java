package org.nd4j.linalg.schedule;
/** The counter a schedule reads: the updater's iteration count, or the epoch count (ComputationGraph.setEpochCount).  The ordinals are
 *  b2g_schedule_type. */
public enum ScheduleType { ITERATION, EPOCH }
