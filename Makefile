# Builds libmpn_b200.so (hand-written CUDA for sm_90a, Hopper H100; C ABI in include/mpn_abi.h),
# plus the test oracle (oracle/). The reference's own Makefile:1-6 builds libnms.so the
# same way (a .so next to the sources, loaded by relative path).
NVCC ?= /usr/local/cuda/bin/nvcc
ARCH := -gencode arch=compute_90a,code=sm_90a
NVFLAGS := -O3 -std=c++17 $(ARCH) -lineinfo -Xcompiler -fPIC --expt-relaxed-constexpr -Xptxas -v
CSRC := multipathnet_b200/csrc
SRCS := $(CSRC)/abi.cu $(CSRC)/nms.cu $(CSRC)/roi.cu $(CSRC)/elementwise.cu $(CSRC)/preproc.cu $(CSRC)/post.cu $(CSRC)/dist.cu $(CSRC)/conv_simt.cu $(CSRC)/gemm_tc.cu $(CSRC)/model.cu $(CSRC)/fp8.cu $(CSRC)/coco_eval.cu $(CSRC)/train.cu $(CSRC)/roidb.cu
OBJS := $(SRCS:.cu=.o)
LIB := multipathnet_b200/libmpn_b200.so

all: $(LIB) oracle
# no flag flushes subnormals (no -use_fast_math / -ftz=true): train.cu's adamax update relies on epsilon 1e-38
$(CSRC)/%.o: $(CSRC)/%.cu $(CSRC)/common.cuh $(CSRC)/conv_gemm.cuh $(CSRC)/wgmma.cuh $(CSRC)/roi.cuh $(CSRC)/image_scale.cuh $(CSRC)/fp8_e4m3.cuh $(CSRC)/train_rule.cuh $(CSRC)/roidb_rule.cuh include/mpn_abi.h
	$(NVCC) $(NVFLAGS) -c $< -o $@ 2> $@.ptxas.log || (cat $@.ptxas.log; false)
# nms.cu must keep the reference's unfused fp32 op order: explicit *_rn intrinsics + -fmad=false
$(CSRC)/nms.o: NVFLAGS += -fmad=false
# preproc.cu reproduces image.scale's unfused fp32 arithmetic (image_scale.cuh uses *_rn intrinsics; belt and braces)
$(CSRC)/preproc.o: NVFLAGS += -fmad=false
# coco_eval.cu keeps pycocotools' unfused double op order (bbIou, linspace thresholds, precision / recall)
$(CSRC)/coco_eval.o: NVFLAGS += -fmad=false
# roidb.cu keeps Torch's unfused fp32 tensor ops and Lua's double arithmetic (roidb_rule.cuh)
$(CSRC)/roidb.o: NVFLAGS += -fmad=false
$(LIB): $(OBJS)
	$(NVCC) $(ARCH) -shared -o $@ $(OBJS) -lcudart -ldl
oracle:
	$(MAKE) -C oracle
clean:
	rm -f $(OBJS) $(CSRC)/*.ptxas.log $(LIB); $(MAKE) -C oracle clean
.PHONY: all oracle clean
