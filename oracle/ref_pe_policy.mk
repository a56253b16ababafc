# oracle/ref_pe_policy.mk -- builds the test-only paired-end framing checker.  Not part of the product.
#
#   _ref/libnvbio_ref_pe_policy.so   nvBowtie's UNMODIFIED frame_opposite_mate (ref_pe_policy.cpp) compiled from an nvbio source tree
#                                    (REF) where it lies (header-only).  Only built when that tree exists; elsewhere an _ref/ built
#                                    beside one is used as is.  Same flags as ref_mapq.mk.
#
#   make -C oracle -f ref_pe_policy.mk [REF=...]
REF  ?= /root/reference
CUDA ?= /usr/local/cuda

all:
	@if [ -d $(REF)/nvbio ]; then $(MAKE) -f ref_pe_policy.mk _ref/libnvbio_ref_pe_policy.so; else echo "oracle: $(REF) absent, keeping prebuilt _ref/libnvbio_ref_pe_policy.so (if any)"; fi

_ref/libnvbio_ref_pe_policy.so: ref_pe_policy.cpp
	mkdir -p _ref
	g++ -O3 -msse4.2 -mpopcnt -funroll-loops -std=c++14 -fopenmp -fPIC -shared -w \
	    -I$(REF) -I$(REF)/contrib -I$(CUDA)/include ref_pe_policy.cpp -o $@

clean:
	rm -f _ref/libnvbio_ref_pe_policy.so

.PHONY: all clean
