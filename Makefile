# Builds libb200exec.so (the product: CUDA kernels + C-ABI host engine) for sm_90a, in-tree.
NVCC      ?= nvcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
PKG       := datafusion-ballista_b200
SRC       := $(PKG)/csrc
OUT       := $(PKG)/lib
# B200_PLAN_STAT_AGGREGATES: this library computes VAR / STDDEV / COVAR / CORR, regr_*, bool_* and bit_* (plan.hpp); set for every unit alike
# B200_PLAN_GROUPING_SETS: ... and grouping sets and the bitwise operators (plan.hpp)
# B200_PLAN_WINDOW: ... and window functions (plan.hpp)
# B200_PLAN_REGEX: ... and ILIKE, the regex operators and regexp_like (plan.hpp)
# B200_PLAN_STRINGS: ... and concat, ||, concat_ws, repeat and reverse (plan.hpp)
NVFLAGS   := $(ARCH) -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -Xcompiler -Wno-unused-function -DB200_PLAN_STAT_AGGREGATES=1 -DB200_PLAN_GROUPING_SETS=1 -DB200_PLAN_WINDOW=1 -DB200_PLAN_REGEX=1 -DB200_PLAN_STRINGS=1
OBJS      := $(OUT)/pipeline.o $(OUT)/kernels.o $(OUT)/shuffle.o $(OUT)/join.o $(OUT)/nlj.o $(OUT)/groupby.o $(OUT)/parquet.o $(OUT)/csv.o $(OUT)/json.o $(OUT)/filter.o $(OUT)/window.o $(OUT)/engine.o $(OUT)/host_narrow.o
CXX       ?= g++
COMMON    := $(wildcard $(SRC)/common/*.hpp) $(wildcard $(SRC)/device/*.h) $(wildcard $(SRC)/device/*.cuh) $(wildcard $(SRC)/host/*.hpp) include/b200exec.h include/b200_arrow_abi.h

all: $(OUT)/libb200exec.so oracle

$(OUT)/pipeline.o: $(SRC)/device/pipeline.cu $(COMMON)
	@mkdir -p $(OUT)
	$(NVCC) $(NVFLAGS) -c $< -o $@
$(OUT)/kernels.o: $(SRC)/device/kernels.cu $(COMMON)
	@mkdir -p $(OUT)
	$(NVCC) $(NVFLAGS) -c $< -o $@
$(OUT)/filter.o: $(SRC)/device/filter.cu $(COMMON)
	@mkdir -p $(OUT)
	$(NVCC) $(NVFLAGS) -c $< -o $@
$(OUT)/parquet.o: $(SRC)/device/parquet.cu $(COMMON)
	@mkdir -p $(OUT)
	$(NVCC) $(NVFLAGS) -c $< -o $@
$(OUT)/csv.o: $(SRC)/device/csv.cu $(COMMON)
	@mkdir -p $(OUT)
	$(NVCC) $(NVFLAGS) -c $< -o $@
$(OUT)/json.o: $(SRC)/device/json.cu $(COMMON)
	@mkdir -p $(OUT)
	$(NVCC) $(NVFLAGS) -c $< -o $@
$(OUT)/groupby.o: $(SRC)/device/groupby.cu $(COMMON)
	@mkdir -p $(OUT)
	$(NVCC) $(NVFLAGS) -c $< -o $@
$(OUT)/join.o: $(SRC)/device/join.cu $(COMMON)
	@mkdir -p $(OUT)
	$(NVCC) $(NVFLAGS) -c $< -o $@
$(OUT)/nlj.o: $(SRC)/device/nlj.cu $(COMMON)
	@mkdir -p $(OUT)
	$(NVCC) $(NVFLAGS) -c $< -o $@
$(OUT)/shuffle.o: $(SRC)/device/shuffle.cu $(COMMON)
	@mkdir -p $(OUT)
	$(NVCC) $(NVFLAGS) -c $< -o $@
$(OUT)/window.o: $(SRC)/device/window.cu $(COMMON)
	@mkdir -p $(OUT)
	$(NVCC) $(NVFLAGS) -c $< -o $@
$(OUT)/engine.o: $(SRC)/host/engine.cpp $(COMMON)
	@mkdir -p $(OUT)
	$(NVCC) $(NVFLAGS) -x cu -c $< -o $@
$(OUT)/host_narrow.o: $(SRC)/host/host_narrow.cpp
	@mkdir -p $(OUT)
	$(CXX) -O3 -std=c++17 -fPIC -c $< -o $@
$(OUT)/libb200exec.so: $(OBJS)
	$(NVCC) $(ARCH) -shared -o $@ $(OBJS) -lcudart_static -lpthread -ldl -lrt

oracle:
	$(MAKE) -C oracle

clean:
	rm -f $(OUT)/*.o $(OUT)/*.so
	$(MAKE) -C oracle clean
.PHONY: all oracle clean
