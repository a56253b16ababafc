# oracle/ref_mapq.mk -- builds the test-only MAPQ checker.  Not part of the product.
#
#   _ref/libnvbio_ref_mapq.so   nvBowtie's UNMODIFIED BowtieMapq2 and SimpleFunc (ref_mapq.cpp) compiled from an nvbio source tree (REF)
#                               where they lie (header-only).  Only built when that tree exists; elsewhere an _ref/ built beside one is
#                               used as is.  Same flags as _ref/libnvbio_ref.so in oracle/Makefile.
#
#   make -C oracle -f ref_mapq.mk [REF=...]
REF  ?= /root/reference
CUDA ?= /usr/local/cuda

all:
	@if [ -d $(REF)/nvbio ]; then $(MAKE) -f ref_mapq.mk _ref/libnvbio_ref_mapq.so; else echo "oracle: $(REF) absent, keeping prebuilt _ref/libnvbio_ref_mapq.so (if any)"; fi

_ref/libnvbio_ref_mapq.so: ref_mapq.cpp
	mkdir -p _ref
	g++ -O3 -msse4.2 -mpopcnt -funroll-loops -std=c++14 -fopenmp -fPIC -shared -w \
	    -I$(REF) -I$(REF)/contrib -I$(CUDA)/include ref_mapq.cpp -o $@

clean:
	rm -f _ref/libnvbio_ref_mapq.so

.PHONY: all clean
