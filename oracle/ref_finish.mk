# oracle/ref_finish.mk -- builds the test-only finishing checker.  Not part of the product.
#
#   _ref/libnvbio_ref_finish.so   nvbio's UNMODIFIED io::analyze_md_string, io::count_symbols and io::reference_cigar_length (ref_finish.cpp)
#                                 compiled from an nvbio source tree (REF) where they lie (header-only).  Only built when that tree exists;
#                                 elsewhere an _ref/ built beside one is used as is.  Same flags as ref_mapq.mk.
#
#   make -C oracle -f ref_finish.mk [REF=...]
REF  ?= /root/reference
CUDA ?= /usr/local/cuda

all:
	@if [ -d $(REF)/nvbio ]; then $(MAKE) -f ref_finish.mk _ref/libnvbio_ref_finish.so; else echo "oracle: $(REF) absent, keeping prebuilt _ref/libnvbio_ref_finish.so (if any)"; fi

_ref/libnvbio_ref_finish.so: ref_finish.cpp
	mkdir -p _ref
	g++ -O3 -msse4.2 -mpopcnt -funroll-loops -std=c++14 -fopenmp -fPIC -shared -w \
	    -I$(REF) -I$(REF)/contrib -I$(CUDA)/include ref_finish.cpp -o $@

clean:
	rm -f _ref/libnvbio_ref_finish.so

.PHONY: all clean
