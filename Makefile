# libxsmm_b200 -- build of the C-ABI library (host C + sm_90a CUDA) and of the test oracles.
#   make lib      -> libxsmm_b200/lib/libxsmm_b200.so   (the product)
#   make oracle   -> oracle/liboracle.so                (C restatement, test infrastructure)
#   make ref      -> oracle/_ref/libxsmm_ref.so         (the unmodified reference, header-only build;
#                                                        only where /root/reference exists)
NVCC      ?= /usr/local/cuda/bin/nvcc
CC        := /usr/bin/gcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVFLAGS   := -O3 -std=c++17 $(ARCH) -lineinfo -Xcompiler -fPIC,-fvisibility=hidden -Xptxas -v --fmad=false
CFLAGS    := -O2 -std=gnu99 -fPIC -fvisibility=hidden -Wall -Wno-unused-function
CSRC      := libxsmm_b200/csrc
OBJDIR    := build/obj
LIB       := libxsmm_b200/lib/libxsmm_b200.so
HOST_C    := host_core.c host_thunks.c host_sparse.c host_meltw.c host_utils.c host_meqn.c
DEVICE_CU := runtime.cu gemm_simt.cu gemm_tc.cu sparse.cu bcsc_tc.cu meltw.cu
OBJS      := $(addprefix $(OBJDIR)/,$(HOST_C:.c=.o) $(DEVICE_CU:.cu=.o))
REFDIR    ?= /root/reference

.PHONY: all lib oracle ref clean
all: lib oracle

lib: $(LIB)

$(OBJDIR)/%.o: $(CSRC)/%.c $(CSRC)/xb_internal.h $(CSRC)/xb_device.cuh include/libxsmm.h include/libxsmm_typedefs.h include/libxsmm_b200.h include/libxsmm_utils.h
	@mkdir -p $(OBJDIR)
	$(CC) $(CFLAGS) -Iinclude -x c -c $< -o $@

$(OBJDIR)/%.o: $(CSRC)/%.cu $(CSRC)/xb_internal.h $(CSRC)/xb_device.cuh $(CSRC)/xb_tma.cuh $(CSRC)/xb_wgmma.cuh $(CSRC)/xb_epilogue.cuh include/libxsmm.h include/libxsmm_typedefs.h
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) -Iinclude -c $< -o $@ 2> $(OBJDIR)/$*.ptxas.log || (cat $(OBJDIR)/$*.ptxas.log; exit 1)

$(LIB): $(OBJS)
	@mkdir -p libxsmm_b200/lib
	$(NVCC) -shared $(ARCH) -cudart static -o $@ $(OBJS) -lpthread -ldl
	ln -sf libxsmm_b200.so libxsmm_b200/lib/libxsmm.so

oracle: oracle/liboracle.so
oracle/liboracle.so: oracle/oracle.c oracle/oracle_meltw.c
	$(CC) -O2 -std=gnu99 -fPIC -shared -ffp-contract=off -fopenmp -Iinclude -o $@ oracle/oracle.c oracle/oracle_meltw.c -lm

ref: oracle/_ref/libxsmm_ref.so
oracle/_ref/libxsmm_ref.so: oracle/ref_shim.c
	@mkdir -p oracle/_ref
	@if [ -d $(REFDIR)/include ]; then \
	  $(CC) -O2 -fPIC -shared -fvisibility=hidden -Wl,-Bsymbolic -fopenmp -ffp-contract=off -I$(REFDIR)/include -I$(REFDIR)/src -o $@ $< -lm -lpthread -ldl; \
	else echo "reference tree not present: keeping prebuilt $@"; fi

clean:
	rm -rf build $(LIB) oracle/liboracle.so
