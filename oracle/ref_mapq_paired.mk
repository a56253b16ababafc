# oracle/ref_mapq_paired.mk -- builds the test-only paired MAPQ checker.  Not part of the product.
#
#   _ref/libnvbio_ref_mapq_paired.so   nvBowtie's UNMODIFIED BowtieMapq2 on paired alignments (ref_mapq_paired.cpp) compiled from an nvbio
#                                      source tree (REF) where it lies (header-only).  Only built when that tree exists; elsewhere an
#                                      _ref/ built beside one is used as is.  Same flags as ref_mapq.mk.
#
#   make -C oracle -f ref_mapq_paired.mk [REF=...]
REF  ?= /root/reference
CUDA ?= /usr/local/cuda

all:
	@if [ -d $(REF)/nvbio ]; then $(MAKE) -f ref_mapq_paired.mk _ref/libnvbio_ref_mapq_paired.so; else echo "oracle: $(REF) absent, keeping prebuilt _ref/libnvbio_ref_mapq_paired.so (if any)"; fi

_ref/libnvbio_ref_mapq_paired.so: ref_mapq_paired.cpp
	mkdir -p _ref
	g++ -O3 -msse4.2 -mpopcnt -funroll-loops -std=c++14 -fopenmp -fPIC -shared -w \
	    -I$(REF) -I$(REF)/contrib -I$(CUDA)/include ref_mapq_paired.cpp -o $@

clean:
	rm -f _ref/libnvbio_ref_mapq_paired.so

.PHONY: all clean
