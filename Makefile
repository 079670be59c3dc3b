# Builds the C-ABI library in-tree (lfm_quant_b200/_lfmq.so, for the H100: sm_90a).
NVCC      ?= nvcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVCCFLAGS := -O3 -Xptxas -v -std=c++17 -lineinfo $(ARCH) -Xcompiler -fPIC -Xcompiler -Wall -Xcompiler -Wno-unknown-pragmas --expt-relaxed-constexpr
CSRC      := lfm_quant_b200/csrc
SRCS      := $(CSRC)/lfmq_api.cu $(CSRC)/kernels_simt.cu $(CSRC)/lstm_tc.cu $(CSRC)/rnn_tc.cu $(CSRC)/tc_shared.cu
OBJS      := $(SRCS:.cu=.o)
LIB       := lfm_quant_b200/_lfmq.so

all: $(LIB)

$(CSRC)/%.o: $(CSRC)/%.cu $(wildcard $(CSRC)/*.h $(CSRC)/*.cuh) include/lfmq.h
	$(NVCC) $(NVCCFLAGS) -c $< -o $@

$(LIB): $(OBJS)
	$(NVCC) $(ARCH) -shared -o $@ $(OBJS) -lcudart

clean:
	rm -f $(OBJS) $(LIB)

# A/B builds of kernel variants: `make alt ALT_FLAGS="-D..."` -> lfm_quant_b200/_lfmq_alt.so (LFMQ_LIB_PATH selects it)
alt:
	mkdir -p build/alt
	for f in lfmq_api kernels_simt lstm_tc rnn_tc tc_shared; do $(NVCC) $(NVCCFLAGS) $(ALT_FLAGS) -c $(CSRC)/$$f.cu -o build/alt/$$f.o || exit 1; done
	$(NVCC) $(ARCH) -shared -o lfm_quant_b200/_lfmq_alt.so $(patsubst $(CSRC)/%.cu,build/alt/%.o,$(SRCS)) -lcudart
