package org.nd4j.linalg.learning.config;
import org.nd4j.linalg.schedule.ISchedule;
/** lr() is the constant learning rate; an updater constructed with an ISchedule writes the schedule's value at 0 there and returns the schedule
 *  from lrSchedule(), which ComputationGraph.init applies per layer. */
public interface IUpdater { int kind(); float lr(); float beta1(); float beta2(); float eps(); default ISchedule lrSchedule() { return null; } }
