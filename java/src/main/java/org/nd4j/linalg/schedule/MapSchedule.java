package org.nd4j.linalg.schedule;
import java.util.Map;
import java.util.TreeMap;

/** The value at the largest key <= i; the map must contain key 0. */
public class MapSchedule implements ISchedule {
    private final ScheduleType type; private final TreeMap<Integer, Double> values;
    public MapSchedule(ScheduleType scheduleType, Map<Integer, Double> values) {
        if (!values.containsKey(0)) throw new IllegalArgumentException("Invalid set of values: must contain initial value (position 0)");
        type = scheduleType; this.values = new TreeMap<>(values);
    }
    public double valueAt(int iteration, int epoch) { int i = type == ScheduleType.ITERATION ? iteration : epoch; return values.floorEntry(i).getValue(); }
    public ScheduleType getScheduleType() { return type; }
    public int kind() { return 5; }
    public double[] parameters() { return new double[] { 0, 0, 0, 0, 0 }; }
    public int[] mapKeys() { return values.keySet().stream().mapToInt(Integer::intValue).toArray(); }
    public double[] mapValues() { return values.values().stream().mapToDouble(Double::doubleValue).toArray(); }
}
