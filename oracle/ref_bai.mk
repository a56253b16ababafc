# oracle/ref_bai.mk -- builds the test-only BAI checkers.  Not part of the product.
#
#   _ref/libnvbio_ref_bai.so   htslib's UNMODIFIED library objects (as ref_bam.mk compiles them into _ref/htslib/) and ref_bai.c:
#                              bam_index_build and region queries through a given .bai.
# Only built where the reference tree (REF) exists; elsewhere an _ref/ built beside one is used as is.
#
#   make -C oracle -f ref_bai.mk [REF=...]
include ref_bam.mk
.DEFAULT_GOAL := bai

bai:
	@if [ -d $(HTS) ]; then $(MAKE) -f ref_bai.mk _ref/libnvbio_ref_bai.so; \
	 else echo "oracle: $(REF) absent, keeping prebuilt _ref/libnvbio_ref_bai.so (if any)"; fi

_ref/libnvbio_ref_bai.so: ref_bai.c $(HTS_OBJ)
	gcc -O2 -fPIC -shared -w -I$(HTS) ref_bai.c $(HTS_OBJ) -o $@ -lz -lpthread -lm

.PHONY: bai
