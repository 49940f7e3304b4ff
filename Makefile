# Builds the C-ABI library (hand-written sm_90a CUDA) and the standalone GEMM self-test.
# `python -c "import __graft_entry__ as g; g.build()"` drives this.
NVCC      ?= /usr/local/cuda/bin/nvcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVFLAGS   := $(ARCH) -O3 -std=c++17 -lineinfo --use_fast_math -Xcompiler -fPIC,-Wall,-Wno-unused-function \
             -Xptxas -v --cudart static -Iinclude
CSRC      := xpretrain_b200/csrc
LIBDIR    := xpretrain_b200/lib
OBJDIR    := build/obj
SRCS      := $(wildcard $(CSRC)/*.cu)
OBJS      := $(patsubst $(CSRC)/%.cu,$(OBJDIR)/%.o,$(SRCS))
LIB       := $(LIBDIR)/libxpretrain_b200.so

all: $(LIB)

$(OBJDIR)/%.o: $(CSRC)/%.cu $(wildcard $(CSRC)/*.cuh) $(wildcard $(CSRC)/*.inc) $(wildcard $(CSRC)/*.h) include/xpretrain_b200.h
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) -c $< -o $@ 2> $(OBJDIR)/$*.ptxas.log || (cat $(OBJDIR)/$*.ptxas.log; exit 1)
	@grep -E "error|warning|spill" $(OBJDIR)/$*.ptxas.log | grep -v "0 bytes spill" | head -20 || true

# retrieval.cu feeds integer rank logic from float comparisons: IEEE exp / division and denormals (no flush-to-zero), so
# that tiny DSL weights stay distinct exactly as in the reference's numpy code
$(OBJDIR)/retrieval.o: NVFLAGS := $(filter-out --use_fast_math,$(NVFLAGS))
# lfvila_head.cu: IEEE division, sqrt, exp and log in the pooled means, the norms and the log-sum-exps
$(OBJDIR)/lfvila_head.o: NVFLAGS := $(filter-out --use_fast_math,$(NVFLAGS))

$(LIB): $(OBJS)
	@mkdir -p $(LIBDIR)
	$(NVCC) $(ARCH) -shared --cudart static -o $@ $(OBJS)

clean:
	rm -rf build $(LIB)

.PHONY: all clean

# standalone GPU self-tests (no torch); run on the GPU box
TOOLS := build/gemm_selftest
tools: $(LIB) $(TOOLS)
build/gemm_selftest: tools/gemm_selftest.cu $(LIB)
	$(NVCC) $(ARCH) -O2 -std=c++17 --cudart static -Iinclude $< -o $@ -L$(LIBDIR) -lxpretrain_b200 -Xlinker -rpath -Xlinker '$$ORIGIN/../$(LIBDIR)'
