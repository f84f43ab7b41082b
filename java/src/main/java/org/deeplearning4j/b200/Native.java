// Native.java -- the ONLY class that touches JNI.  Every method is a 1:1 image of a C-ABI function in include/b200gan.h
// (see jni/b200gan_jni.cpp); arguments are primitives: handles and direct-buffer addresses travel as long.
// SOURCE ONLY: this image has no JDK (SURVEY.md section 8b/8f#2); the tested artefact is the same C-ABI driven through
// Python ctypes (gan_deeplearning4j_b200/_lib.py).
package org.deeplearning4j.b200;

import java.nio.ByteBuffer;
import java.nio.ByteOrder;
import java.nio.FloatBuffer;

public final class Native {
    static { System.loadLibrary("b200gan"); }
    private Native() {}

    public static native int version();
    public static native int ctxCreate(int device, long outHandleAddr);
    public static native int ctxDestroy(long ctx);
    public static native int sync(long ctx);
    public static native long lastErrorAddr();
    public static native int netCreate(long ctx, long cfgAddr, long layersAddr, int n, long outHandleAddr);
    public static native int netDestroy(long net);
    public static native int netNumParams(long net, long outAddr);
    public static native int netOutputSize(long net, long outAddr);
    public static native int netSetParam(long net, long layerNameAddr, long paramNameAddr, long hostAddr, long n);
    public static native int netGetParam(long net, long layerNameAddr, long paramNameAddr, long hostAddr, long n);
    public static native int netGetParams(long net, long hostAddr, long n);
    public static native int netSetParams(long net, long hostAddr, long n);
    public static native int netUpdaterStateSize(long net, long outAddr);
    public static native int netGetUpdaterState(long net, long hostAddr, long n);
    public static native int netSetUpdaterState(long net, long hostAddr, long n);
    public static native int netGetIteration(long net, long outAddr);
    public static native int netSetIteration(long net, long iteration);
    public static native int netGetDropoutPass(long net, long outAddr);
    public static native int netSetDropoutPass(long net, long pass);
    public static native int netSetGradientNormalization(long net, int mode, float threshold);
    public static native int netSetLrSchedule(long net, long layerNameAddr, long scheduleAddr);   // layerNameAddr 0: every layer; scheduleAddr 0: constant lr
    public static native int netSetConstraints(long net, long layerNameAddr, long paramNameAddr, long constraintsAddr, int n);   // b2g_constraint[n]
    public static native int netApplyConstraints(long net);
    public static native int netGetLearningRate(long net, long layerNameAddr, long outAddr);
    public static native int netSetDropoutSchedule(long net, long layerNameAddr, long scheduleAddr);   // layerNameAddr 0: every DropoutLayer; scheduleAddr 0: constant
    public static native int netGetDropoutValue(long net, long layerNameAddr, long outAddr);
    public static native int netSetWeightNoise(long net, long layerNameAddr, long weightNoiseAddr);   // b2g_weight_noise; layerNameAddr 0: every layer with a W
    public static native int netInitWeights(long net, long layerNameAddr, long weightInitAddr);   // b2g_weight_init; layerNameAddr 0: every layer with a W
    public static native int netSetRegularization(long net, long layerNameAddr, long regAddr);   // b2g_regularization; layerNameAddr 0: every non-frozen layer with a W
    public static native int netCalcRegularization(long net, long l1Addr, long l2Addr);          // two doubles: calcL1(true), calcL2(true)
    public static native int netGetEpoch(long net, long outAddr);
    public static native int netSetEpoch(long net, long epoch);
    public static native int netSimtGemmCalls(long net, long outAddr);
    public static native int netSetSyncBn(long net, int enabled);
    public static native int netSetGradPayloadBf16(long net, int enabled);
    public static native int netEnableP2pAllreduce(long net, long outEnabledAddr);   // collective over the communicator: b2g_net_enable_p2p_allreduce
    public static native int netOutput(long net, long xAddr, int batch, int train, long outAddr);
    public static native int netFit(long net, long xAddr, long yAddr, int batch, long scoreAddr);
    public static native int netFitMasked(long net, long xAddr, long yAddr, int batch, long scoreAddr, long maskAddr, int maskWidth);
    public static native int netSetLossWeights(long net, long layerNameAddr, long wAddr, int n);
    public static native int ganSetLabelMasks(long gan, long mReal, long mFake, long mGen, int maskWidth, int batch);
    public static native int ganCreate(long gen, long dis, int fakeBnTrain, int useGraph, long outHandleAddr);
    public static native int ganDestroy(long gan);
    public static native int ganStep(long gan, long xReal, long zD, long zG, long yReal, long yFake, long yGen, int batch, long lossesAddr);
    public static native int commUniqueId(long id128Addr);
    public static native int ctxCommInit(long ctx, int world, int rank, long id128Addr);

    // ---- helpers: direct buffers are the host side of every transfer (b2g copies during the call) ----
    public static ByteBuffer direct(int bytes) { return ByteBuffer.allocateDirect(bytes).order(ByteOrder.nativeOrder()); }
    public static long address(java.nio.Buffer b) {
        try {   // sun.nio.ch.DirectBuffer.address() without a compile-time dependency
            java.lang.reflect.Method m = b.getClass().getMethod("address"); m.setAccessible(true); return (Long) m.invoke(b);
        } catch (ReflectiveOperationException e) { throw new IllegalStateException(e); }
    }
    public static ByteBuffer cstr(String s) { byte[] a = s.getBytes(java.nio.charset.StandardCharsets.US_ASCII); ByteBuffer b = direct(a.length + 1); b.put(a).put((byte) 0); b.flip(); return b; }
    public static FloatBuffer floats(float[] a) { ByteBuffer b = direct(4 * a.length); FloatBuffer f = b.asFloatBuffer(); f.put(a); return f; }
    /** DL4J throws on failure; the C-ABI returns a status: map non-zero to IllegalStateException with b2g_last_error(). */
    public static void check(int status) {
        if (status != 0) throw new IllegalStateException("libb200gan error " + status);
    }

    private static long CTX = 0;
    public static synchronized long context() {
        if (CTX == 0) { ByteBuffer h = direct(8); check(ctxCreate(Integer.getInteger("b200gan.device", 0), address(h))); CTX = h.getLong(0); }
        return CTX;
    }
}
