# Build libb200gan.so (sm_90a, H100, only).  `make` here or __graft_entry__.build() -- same commands.
NVCC ?= /usr/local/cuda/bin/nvcc
ARCH := -gencode arch=compute_90a,code=sm_90a
NVFLAGS := $(ARCH) -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-Wall,-Wno-unused-function -Xptxas -v
SRC := gan_deeplearning4j_b200/csrc
OUT := gan_deeplearning4j_b200/lib
OBJS := $(OUT)/kernels_ew.o $(OUT)/kernels_dropout.o $(OUT)/kernels_act.o $(OUT)/kernels_pool.o $(OUT)/kernels_cnnloss.o $(OUT)/kernels_head.o $(OUT)/kernels_graph.o $(OUT)/kernels_prelu.o $(OUT)/kernels_gradnorm.o $(OUT)/kernels_constraint.o $(OUT)/kernels_init.o $(OUT)/kernels_simt.o $(OUT)/kernels_tc.o $(OUT)/kernels_edge.o $(OUT)/engine.o $(OUT)/jni_shim.o

all: $(OUT)/libb200gan.so

$(OUT)/%.o: $(SRC)/%.cu $(SRC)/kernels.h $(SRC)/common.cuh include/b200gan.h
	@mkdir -p $(OUT)
	$(NVCC) $(NVFLAGS) -c $< -o $@ 2> $(OUT)/$*.ptxas.log || (cat $(OUT)/$*.ptxas.log; exit 1)

$(OUT)/jni_shim.o: jni/b200gan_jni.cpp include/b200gan.h
	@mkdir -p $(OUT)
	g++ -O2 -fPIC -std=c++17 -Wall -c $< -o $@

$(OUT)/libb200gan.so: $(OBJS)
	$(NVCC) $(ARCH) -shared -o $@ $(OBJS) -lcudart_static -ldl -lrt -lpthread

clean:
	rm -rf $(OUT)
