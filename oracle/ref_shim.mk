# oracle/ref_shim.mk -- builds the drop-in boundary harnesses (tests/shim/*.cu).  Not part of the product.
# (Unrelated to oracle/ref_shim.cpp, the host wrappers of the reference's templates in _ref/libnvbio_ref.so, which oracle/Makefile builds.)
#
# Each harness is a program written against nvbio's own types, compiled twice from one source against the reference headers:
#   _ref/shim/<harness>_ref    as is: nvbio's own templates and kernels, recompiled for sm_90a
#   _ref/shim/<harness>_b200   the same source with -DNVBIO_B200_SHIM (include/nvbio_b200/shim/*.h), linked against libnvbio_b200.so
#                              through an $ORIGIN-relative rpath (_ref/shim -> ../../../nvbio_b200)
# for <harness> = shim_harness, nvbowtie_harness, nvbowtie_score_harness; tests/test_gpu_shim.py runs and compares the pairs.
# nvBowtie's sources need its defs.h with the texture-reference path (removed in CUDA 12) switched off: a GENERATED overlay of that one
# header (a sed of the file where it lies, written under _ref/shim/overlay, never committed) comes first on their include path.
# Only built where the reference tree (REF) exists; elsewhere an _ref/shim built beside one is used as is.
#
#   make -C oracle -f ref_shim.mk [REF=...]
REF  ?= /root/reference
ROOT := $(abspath ..)
NVCC ?= /usr/local/cuda/bin/nvcc
SRC  := $(ROOT)/tests/shim
OUT  := _ref/shim
OBJ  := $(OUT)/obj
OVERLAY := $(OUT)/overlay
DEFS := $(OVERLAY)/nvBowtie/bowtie2/cuda/defs.h
LIB  := $(ROOT)/nvbio_b200/libnvbio_b200.so
SHIM_HEADERS := $(wildcard $(ROOT)/include/nvbio_b200/shim/*.h) $(ROOT)/include/nvbio_b200.h
ARCH := -gencode arch=compute_90a,code=sm_90a
FLAGS     := -O3 -std=c++17 $(ARCH) -use_fast_math -Xcompiler -fopenmp -w -I$(REF) -I$(REF)/contrib -I$(ROOT)/include
NVB_FLAGS := -O3 -std=c++17 $(ARCH) -use_fast_math -Xcompiler -fopenmp -w \
             -I$(OVERLAY) -I$(REF) -I$(REF)/contrib -I$(REF)/contrib/crc -I$(REF)/contrib/bamtools -I$(ROOT)/include -DPLATFORM_X86
LINK_B200 := -L$(ROOT)/nvbio_b200 -lnvbio_b200 -Xlinker -rpath -Xlinker '$$ORIGIN/../../../nvbio_b200'

BINS := $(addprefix $(OUT)/,shim_harness_ref shim_harness_b200 nvbowtie_harness_ref nvbowtie_harness_b200 nvbowtie_score_harness_ref nvbowtie_score_harness_b200)

all:
	@if [ -d $(REF)/nvbio ] && [ -d $(REF)/nvBowtie ]; then $(MAKE) -f ref_shim.mk $(BINS); \
	 else echo "oracle: $(REF) absent, keeping prebuilt $(OUT) (if any)"; fi

$(DEFS): $(REF)/nvBowtie/bowtie2/cuda/defs.h
	@mkdir -p $(dir $@)
	sed 's/^#define USE_TEX  *1/#define USE_TEX             0/; s/^#define USE_TEX_READS  *1/#define USE_TEX_READS       0/' $< > $@

# nvbio's console.cpp (log_error & co.), compiled where it lies: with the flags of the objects it is linked with
$(OBJ)/console.o: $(REF)/nvbio/basic/console.cpp
	@mkdir -p $(OBJ)
	$(NVCC) $(FLAGS) -c $< -o $@
$(OBJ)/console_nvb.o: $(REF)/nvbio/basic/console.cpp $(DEFS)
	@mkdir -p $(OBJ)
	$(NVCC) $(NVB_FLAGS) -c $< -o $@

# B-A1 / B-B1: fmmap and the batch programs (nvbio's FM-index filter, batched banded and full-matrix scoring)
$(OUT)/shim_harness_ref: $(SRC)/shim_harness.cu $(OBJ)/console.o
	$(NVCC) $(FLAGS) $(SRC)/shim_harness.cu $(OBJ)/console.o -o $@
$(OUT)/shim_harness_b200: $(SRC)/shim_harness.cu $(OBJ)/console.o $(SHIM_HEADERS) $(LIB)
	$(NVCC) $(FLAGS) -DNVBIO_B200_SHIM $(SRC)/shim_harness.cu $(OBJ)/console.o -o $@ $(LINK_B200)

# B-A2: one caller object linked once against nvBowtie's mapping.cu (compiled where it lies) and once against its replacement
$(OBJ)/nvbowtie_harness.o: $(SRC)/nvbowtie_harness.cu $(DEFS)
	@mkdir -p $(OBJ)
	$(NVCC) $(NVB_FLAGS) -c $< -o $@
$(OBJ)/nvbowtie_mapping_ref.o: $(REF)/nvBowtie/bowtie2/cuda/mapping.cu $(DEFS)
	@mkdir -p $(OBJ)
	$(NVCC) $(NVB_FLAGS) -c $< -o $@
$(OBJ)/nvbowtie_mapping_b200.o: $(SRC)/nvbowtie_mapping_b200.cu $(SHIM_HEADERS) $(DEFS)
	@mkdir -p $(OBJ)
	$(NVCC) $(NVB_FLAGS) -c $< -o $@
$(OUT)/nvbowtie_harness_ref: $(OBJ)/nvbowtie_harness.o $(OBJ)/nvbowtie_mapping_ref.o $(OBJ)/console_nvb.o
	$(NVCC) $(ARCH) -Xcompiler -fopenmp $^ -o $@
$(OUT)/nvbowtie_harness_b200: $(OBJ)/nvbowtie_harness.o $(OBJ)/nvbowtie_mapping_b200.o $(OBJ)/console_nvb.o $(LIB)
	$(NVCC) $(ARCH) -Xcompiler -fopenmp $(OBJ)/nvbowtie_harness.o $(OBJ)/nvbowtie_mapping_b200.o $(OBJ)/console_nvb.o -o $@ $(LINK_B200)

# B-B2: nvBowtie's best-score extension stage, with and without the shim
$(OUT)/nvbowtie_score_harness_ref: $(SRC)/nvbowtie_score_harness.cu $(OBJ)/console_nvb.o $(DEFS)
	$(NVCC) $(NVB_FLAGS) $(SRC)/nvbowtie_score_harness.cu $(OBJ)/console_nvb.o -o $@
$(OUT)/nvbowtie_score_harness_b200: $(SRC)/nvbowtie_score_harness.cu $(OBJ)/console_nvb.o $(SHIM_HEADERS) $(DEFS) $(LIB)
	$(NVCC) $(NVB_FLAGS) -DNVBIO_B200_SHIM $(SRC)/nvbowtie_score_harness.cu $(OBJ)/console_nvb.o -o $@ $(LINK_B200)

clean:
	rm -rf $(OUT)

.PHONY: all clean
