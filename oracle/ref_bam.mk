# oracle/ref_bam.mk -- builds the test-only BAM checkers.  Not part of the product.
#
#   _ref/libnvbio_ref_bam.so   htslib's UNMODIFIED library objects (the copy in the reference's contrib/htslib, compiled where they lie
#                              into _ref/htslib/, the tree being read-only) and ref_bam.c: SAM line -> bam_write1 bytes, .bam ->
#                              sam_format1 text, hts_reg2bin.
#   _ref/libnvbio_ref_bns.so   nvbio's own save_bns (nvbio/basic/bnt.cpp, compiled where it lies) behind ref_bns.cpp: the
#                              writer of the .ann files the .ann reader (nvbio_b200/io.py) is pinned against.
# Only built where the reference tree (REF) exists; elsewhere an _ref/ built beside one is used as is.
#
#   make -C oracle -f ref_bam.mk [REF=...]
REF  ?= /root/reference
CUDA ?= /usr/local/cuda
HTS  := $(REF)/contrib/htslib
OBJ  := _ref/htslib

HTS_SRC := kfunc knetfile kstring bgzf faidx hfile hfile_net hts sam synced_bcf_reader vcf_sweep tbx vcf vcfutils \
           cram/cram_codecs cram/cram_decode cram/cram_encode cram/cram_index cram/cram_io cram/cram_samtools cram/cram_stats \
           cram/files cram/mFILE cram/md5 cram/open_trace_file cram/pooled_alloc cram/sam_header cram/string_alloc cram/thread_pool \
           cram/vlen cram/zfio
HTS_OBJ := $(addprefix $(OBJ)/,$(addsuffix .o,$(HTS_SRC)))

all:
	@if [ -d $(HTS) ] && [ -d $(REF)/nvbio ]; then $(MAKE) -f ref_bam.mk _ref/libnvbio_ref_bam.so _ref/libnvbio_ref_bns.so; \
	 else echo "oracle: $(REF) absent, keeping prebuilt _ref/libnvbio_ref_bam.so / libnvbio_ref_bns.so (if any)"; fi

# htslib's own Makefile flags (-O2, -DSAMTOOLS=1, PIC), each object with an explicit -o so that nothing is written into the tree
$(OBJ)/%.o: $(HTS)/%.c
	@mkdir -p $(dir $@)
	gcc -O2 -fPIC -w -DSAMTOOLS=1 -I$(HTS) -c $< -o $@

_ref/libnvbio_ref_bam.so: ref_bam.c $(HTS_OBJ)
	gcc -O2 -fPIC -shared -w -I$(HTS) ref_bam.c $(HTS_OBJ) -o $@ -lz -lpthread -lm

_ref/libnvbio_ref_bns.so: ref_bns.cpp
	mkdir -p _ref
	g++ -O2 -std=c++14 -fPIC -shared -w -I$(REF) -I$(REF)/contrib -I$(CUDA)/include ref_bns.cpp $(REF)/nvbio/basic/bnt.cpp -o $@

clean:
	rm -rf _ref/libnvbio_ref_bam.so _ref/libnvbio_ref_bns.so $(OBJ)

.PHONY: all clean
