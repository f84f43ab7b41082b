// Nd4j factory calls used by the driver (J:105,114-115,170,382-421): host-side only.
package org.nd4j.linalg.factory;

import java.util.Collection;
import java.util.Random;
import org.nd4j.linalg.api.buffer.DataBuffer;
import org.nd4j.linalg.api.ndarray.INDArray;

public final class Nd4j {
    private static final Random RNG = new Random(666);
    private Nd4j() {}
    public static void setDataType(DataBuffer.Type t) { if (t != DataBuffer.Type.FLOAT) throw new IllegalStateException("b200gan computes in fp32/bf16"); }
    public static String getBackend() { return "b200gan (sm_90a, libb200gan.so v" + org.deeplearning4j.b200.Native.version() + ")"; }
    public static MemoryManager getMemoryManager() { return new MemoryManager(); }
    public static final class MemoryManager { public void setAutoGcWindow(int ms) { /* device memory is one static arena per net */ } }
    private static long numel(long... s) { long n = 1; for (long v : s) n *= v; return n; }
    public static INDArray zeros(long... s) { return new INDArray(new float[(int) numel(s)], s); }
    public static INDArray ones(long... s) { INDArray a = zeros(s); java.util.Arrays.fill(a.data, 1f); return a; }
    public static INDArray rand(long... s) { INDArray a = zeros(s); for (int i = 0; i < a.data.length; i++) a.data[i] = RNG.nextFloat(); return a; }
    public static INDArray randn(long... s) { INDArray a = zeros(s); for (int i = 0; i < a.data.length; i++) a.data[i] = (float) RNG.nextGaussian(); return a; }
    public static INDArray linspace(double lo, double hi, long n) { INDArray a = zeros(1, n); for (int i = 0; i < n; i++) a.data[i] = (float) (lo + (hi - lo) * i / Math.max(1, n - 1)); return a; }
    public static INDArray create(float[] d, long... s) { return new INDArray(d, s); }
    public static INDArray vstack(Collection<INDArray> rows) {
        int n = 0, w = -1; for (INDArray r : rows) { n += r.shape()[0]; w = (int) (r.length() / r.shape()[0]); }
        float[] d = new float[n * w]; int o = 0; for (INDArray r : rows) { System.arraycopy(r.data, 0, d, o, r.data.length); o += r.data.length; }
        return new INDArray(d, n, w);
    }
}
