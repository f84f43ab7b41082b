// b200gan_jni.cpp -- primitive-only JNI shim over the C-ABI (include/b200gan.h).
//
// The Java facade (java/org/deeplearning4j/b200/Native.java) declares these as
//   private static native int netFit(long net, long xAddr, long yAddr, int batch, long scoreAddr); ...
// Host tensors cross as raw addresses of direct ByteBuffers (jlong), handles as jlong, status as jint:
// no JNIEnv callbacks, no Java objects, no exceptions thrown from native code -- so this file needs no
// <jni.h> (this image has no JDK; SURVEY.md section 8b) and the exported symbols are exactly the ones a
// real JVM resolves.  A maintainer with a JDK may replace the typedefs below by #include <jni.h> unchanged.
#include <stdint.h>
#include "../include/b200gan.h"

typedef void JNIEnv_;            // opaque: never dereferenced
typedef void* jclass;
typedef int32_t jint;
typedef int64_t jlong;
typedef float jfloat;
#define JNIEXPORT __attribute__((visibility("default")))
#define JNICALL
#define FN(name) extern "C" JNIEXPORT jint JNICALL Java_org_deeplearning4j_b200_Native_##name
#define P(T, a) reinterpret_cast<T>(static_cast<intptr_t>(a))

FN(version)(JNIEnv_*, jclass) { return b2g_version(); }
FN(ctxCreate)(JNIEnv_*, jclass, jint device, jlong outHandleAddr) { return b2g_ctx_create(device, P(b2g_ctx**, outHandleAddr)); }
FN(ctxDestroy)(JNIEnv_*, jclass, jlong ctx) { return b2g_ctx_destroy(P(b2g_ctx*, ctx)); }
FN(sync)(JNIEnv_*, jclass, jlong ctx) { return b2g_sync(P(b2g_ctx*, ctx)); }
extern "C" JNIEXPORT jlong JNICALL Java_org_deeplearning4j_b200_Native_lastErrorAddr(JNIEnv_*, jclass) { return (jlong)(intptr_t)b2g_last_error(); }
// cfgAddr -> b2g_net_config, layersAddr -> b2g_layer_desc[n] laid out by the facade in a direct ByteBuffer
FN(netCreate)(JNIEnv_*, jclass, jlong ctx, jlong cfgAddr, jlong layersAddr, jint n, jlong outHandleAddr) {
  return b2g_net_create(P(b2g_ctx*, ctx), P(const b2g_net_config*, cfgAddr), P(const b2g_layer_desc*, layersAddr), n, P(b2g_net**, outHandleAddr));
}
FN(netDestroy)(JNIEnv_*, jclass, jlong net) { return b2g_net_destroy(P(b2g_net*, net)); }
FN(netNumParams)(JNIEnv_*, jclass, jlong net, jlong outAddr) { return b2g_net_num_params(P(b2g_net*, net), P(int64_t*, outAddr)); }
FN(netOutputSize)(JNIEnv_*, jclass, jlong net, jlong outAddr) { return b2g_net_output_size(P(b2g_net*, net), P(int64_t*, outAddr)); }
FN(netSetParam)(JNIEnv_*, jclass, jlong net, jlong layerNameAddr, jlong paramNameAddr, jlong hostAddr, jlong n) {
  return b2g_net_set_param(P(b2g_net*, net), P(const char*, layerNameAddr), P(const char*, paramNameAddr), P(const float*, hostAddr), n);
}
FN(netGetParam)(JNIEnv_*, jclass, jlong net, jlong layerNameAddr, jlong paramNameAddr, jlong hostAddr, jlong n) {
  return b2g_net_get_param(P(b2g_net*, net), P(const char*, layerNameAddr), P(const char*, paramNameAddr), P(float*, hostAddr), n);
}
FN(netGetParams)(JNIEnv_*, jclass, jlong net, jlong hostAddr, jlong n) { return b2g_net_get_params(P(b2g_net*, net), P(float*, hostAddr), n); }
FN(netSetParams)(JNIEnv_*, jclass, jlong net, jlong hostAddr, jlong n) { return b2g_net_set_params(P(b2g_net*, net), P(const float*, hostAddr), n); }
FN(netUpdaterStateSize)(JNIEnv_*, jclass, jlong net, jlong outAddr) { return b2g_net_updater_state_size(P(b2g_net*, net), P(int64_t*, outAddr)); }
FN(netGetUpdaterState)(JNIEnv_*, jclass, jlong net, jlong hostAddr, jlong n) { return b2g_net_get_updater_state(P(b2g_net*, net), P(float*, hostAddr), n); }
FN(netSetUpdaterState)(JNIEnv_*, jclass, jlong net, jlong hostAddr, jlong n) { return b2g_net_set_updater_state(P(b2g_net*, net), P(const float*, hostAddr), n); }
FN(netGetIteration)(JNIEnv_*, jclass, jlong net, jlong outAddr) { return b2g_net_get_iteration(P(b2g_net*, net), P(int64_t*, outAddr)); }
FN(netSetIteration)(JNIEnv_*, jclass, jlong net, jlong it) { return b2g_net_set_iteration(P(b2g_net*, net), it); }
FN(netGetDropoutPass)(JNIEnv_*, jclass, jlong net, jlong outAddr) { return b2g_net_get_dropout_pass(P(b2g_net*, net), P(int64_t*, outAddr)); }
FN(netSetDropoutPass)(JNIEnv_*, jclass, jlong net, jlong pass) { return b2g_net_set_dropout_pass(P(b2g_net*, net), pass); }
FN(netSetGradientNormalization)(JNIEnv_*, jclass, jlong net, jint mode, jfloat threshold) { return b2g_net_set_gradient_normalization(P(b2g_net*, net), mode, threshold); }
// scheduleAddr -> b2g_lr_schedule laid out by the facade in a direct ByteBuffer (0 = back to the constant lr); layerNameAddr 0 = every layer
FN(netSetLrSchedule)(JNIEnv_*, jclass, jlong net, jlong layerNameAddr, jlong scheduleAddr) {
  return b2g_net_set_lr_schedule(P(b2g_net*, net), P(const char*, layerNameAddr), P(const b2g_lr_schedule*, scheduleAddr));
}
// constraintsAddr -> b2g_constraint[n] laid out by the facade in a direct ByteBuffer; n = 0 clears the tensor's list
FN(netSetConstraints)(JNIEnv_*, jclass, jlong net, jlong layerNameAddr, jlong paramNameAddr, jlong constraintsAddr, jint n) {
  return b2g_net_set_constraints(P(b2g_net*, net), P(const char*, layerNameAddr), P(const char*, paramNameAddr), P(const b2g_constraint*, constraintsAddr), n);
}
FN(netApplyConstraints)(JNIEnv_*, jclass, jlong net) { return b2g_net_apply_constraints(P(b2g_net*, net)); }
FN(netGetLearningRate)(JNIEnv_*, jclass, jlong net, jlong layerNameAddr, jlong outAddr) {
  return b2g_net_get_learning_rate(P(b2g_net*, net), P(const char*, layerNameAddr), P(float*, outAddr));
}
// the DropoutLayer's IDropout schedule, laid out as for netSetLrSchedule (layerNameAddr 0: every non-frozen DropoutLayer; scheduleAddr 0: constant)
FN(netSetDropoutSchedule)(JNIEnv_*, jclass, jlong net, jlong layerNameAddr, jlong scheduleAddr) {
  return b2g_net_set_dropout_schedule(P(b2g_net*, net), P(const char*, layerNameAddr), P(const b2g_lr_schedule*, scheduleAddr));
}
FN(netGetDropoutValue)(JNIEnv_*, jclass, jlong net, jlong layerNameAddr, jlong outAddr) {
  return b2g_net_get_dropout_value(P(b2g_net*, net), P(const char*, layerNameAddr), P(float*, outAddr));
}
// b2g_weight_noise (40 bytes, its p_schedule laid out as for netSetLrSchedule); layerNameAddr 0: every non-frozen layer with a W; 0: none
FN(netSetWeightNoise)(JNIEnv_*, jclass, jlong net, jlong layerNameAddr, jlong wnAddr) {
  return b2g_net_set_weight_noise(P(b2g_net*, net), P(const char*, layerNameAddr), P(const b2g_weight_noise*, wnAddr));
}
// b2g_weight_init (20 bytes); layerNameAddr 0: every layer with a W
FN(netInitWeights)(JNIEnv_*, jclass, jlong net, jlong layerNameAddr, jlong wiAddr) {
  return b2g_net_init_weights(P(b2g_net*, net), P(const char*, layerNameAddr), P(const b2g_weight_init*, wiAddr));
}
// b2g_regularization (16 bytes); layerNameAddr 0: every non-frozen layer with a W
FN(netSetRegularization)(JNIEnv_*, jclass, jlong net, jlong layerNameAddr, jlong regAddr) {
  return b2g_net_set_regularization(P(b2g_net*, net), P(const char*, layerNameAddr), P(const b2g_regularization*, regAddr));
}
FN(netCalcRegularization)(JNIEnv_*, jclass, jlong net, jlong l1Addr, jlong l2Addr) {
  return b2g_net_calc_regularization(P(b2g_net*, net), P(double*, l1Addr), P(double*, l2Addr));
}
FN(netGetEpoch)(JNIEnv_*, jclass, jlong net, jlong outAddr) { return b2g_net_get_epoch(P(b2g_net*, net), P(int64_t*, outAddr)); }
FN(netSetEpoch)(JNIEnv_*, jclass, jlong net, jlong epoch) { return b2g_net_set_epoch(P(b2g_net*, net), epoch); }
FN(netSimtGemmCalls)(JNIEnv_*, jclass, jlong net, jlong outAddr) { return b2g_net_simt_gemm_calls(P(b2g_net*, net), P(uint64_t*, outAddr)); }
FN(netSetSyncBn)(JNIEnv_*, jclass, jlong net, jint enabled) { return b2g_net_set_sync_bn(P(b2g_net*, net), enabled); }
FN(netSetGradPayloadBf16)(JNIEnv_*, jclass, jlong net, jint enabled) { return b2g_net_set_grad_payload_bf16(P(b2g_net*, net), enabled); }
FN(netEnableP2pAllreduce)(JNIEnv_*, jclass, jlong net, jlong outAddr) { return b2g_net_enable_p2p_allreduce(P(b2g_net*, net), P(int32_t*, outAddr)); }
FN(netOutput)(JNIEnv_*, jclass, jlong net, jlong xAddr, jint batch, jint train, jlong outAddr) {
  return b2g_net_output(P(b2g_net*, net), P(const float*, xAddr), batch, train, P(float*, outAddr));
}
FN(netFit)(JNIEnv_*, jclass, jlong net, jlong xAddr, jlong yAddr, jint batch, jlong scoreAddr) {
  return b2g_net_fit(P(b2g_net*, net), P(const float*, xAddr), P(const float*, yAddr), batch, P(float*, scoreAddr));
}
FN(netFitMasked)(JNIEnv_*, jclass, jlong net, jlong xAddr, jlong yAddr, jint batch, jlong scoreAddr, jlong maskAddr, jint maskWidth) {
  return b2g_net_fit_masked(P(b2g_net*, net), P(const float*, xAddr), P(const float*, yAddr), batch, P(float*, scoreAddr), P(const float*, maskAddr), maskWidth);
}
FN(netSetLossWeights)(JNIEnv_*, jclass, jlong net, jlong layerNameAddr, jlong wAddr, jint n) {
  return b2g_net_set_loss_weights(P(b2g_net*, net), P(const char*, layerNameAddr), P(const float*, wAddr), n);
}
FN(ganSetLabelMasks)(JNIEnv_*, jclass, jlong gan, jlong mReal, jlong mFake, jlong mGen, jint maskWidth, jint batch) {
  return b2g_gan_set_label_masks(P(b2g_gan*, gan), P(const float*, mReal), P(const float*, mFake), P(const float*, mGen), maskWidth, batch);
}
FN(ganCreate)(JNIEnv_*, jclass, jlong gen, jlong dis, jint fakeBnTrain, jint useGraph, jlong outHandleAddr) {
  b2g_gan_config c{fakeBnTrain, useGraph};
  return b2g_gan_create(P(b2g_net*, gen), P(b2g_net*, dis), &c, P(b2g_gan**, outHandleAddr));
}
FN(ganDestroy)(JNIEnv_*, jclass, jlong gan) { return b2g_gan_destroy(P(b2g_gan*, gan)); }
FN(ganStep)(JNIEnv_*, jclass, jlong gan, jlong xReal, jlong zD, jlong zG, jlong yReal, jlong yFake, jlong yGen, jint batch, jlong lossesAddr) {
  return b2g_gan_step(P(b2g_gan*, gan), P(const float*, xReal), P(const float*, zD), P(const float*, zG), P(const float*, yReal), P(const float*, yFake),
                      P(const float*, yGen), batch, P(float*, lossesAddr));
}
FN(netSetGradAllreduce)(JNIEnv_*, jclass, jlong net, jint enabled) { return b2g_net_set_grad_allreduce(P(b2g_net*, net), enabled); }
FN(netAverageParameters)(JNIEnv_*, jclass, jlong net) { return b2g_net_average_parameters(P(b2g_net*, net)); }
FN(commUniqueId)(JNIEnv_*, jclass, jlong id128Addr) { return b2g_comm_unique_id(P(void*, id128Addr)); }
FN(ctxCommInit)(JNIEnv_*, jclass, jlong ctx, jint world, jint rank, jlong id128Addr) { return b2g_ctx_comm_init(P(b2g_ctx*, ctx), world, rank, P(const void*, id128Addr)); }
