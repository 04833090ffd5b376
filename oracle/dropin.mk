# oracle/dropin.mk -- TEST INFRASTRUCTURE ONLY (never linked into the product library).  Run by build() (__graft_entry__.py) after the
# library and oracle/Makefile:
#
#   _ref/libbsc_dropin.so   the reference's block layer and host stages (libbsc.cpp, lzp, platform, adler32, filters -- unmodified, from
#                           $(REF)) as a shared library whose stage entry points (bsc_{bwt,st,coder}_*) come from libbsc_b200.so: the
#                           reference's own in-place bsc_compress on top of this library's stages (INTEGRATION.md option 1), what
#                           _ref/bsc_dropin is as a CLI.  Both libraries export bsc_compress, so a test loads this one only in a child
#                           process of its own (tests/test_gpu_large_st_encode.py).
#
# Built only where $(REF) and ../libbsc_b200/libbsc_b200.so exist; elsewhere `make -f dropin.mk` does nothing.  No reference source is
# copied into this repo.

REF      ?= /root/reference
CXX       = /usr/bin/g++
LIB_SRC   = libbsc/libbsc/libbsc.cpp libbsc/lzp/lzp.cpp libbsc/platform/platform.cpp libbsc/adler32/adler32.cpp \
            libbsc/filters/detectors.cpp libbsc/filters/preprocessing.cpp

.PHONY: all
all: $(if $(and $(wildcard $(REF)/libbsc/libbsc.h),$(wildcard ../libbsc_b200/libbsc_b200.so)),_ref/libbsc_dropin.so,)

_ref/libbsc_dropin.so: $(addprefix $(REF)/,$(LIB_SRC)) ../libbsc_b200/libbsc_b200.so
	mkdir -p _ref
	$(CXX) -O2 -fopenmp -mavx2 -w -fPIC -shared -DLIBBSC_OPENMP_SUPPORT -DLIBBSC_SORT_TRANSFORM_SUPPORT -DLIBBSC_ALLOW_UNALIGNED_ACCESS -I$(REF) \
	    $(addprefix $(REF)/,$(LIB_SRC)) -o $@ -L../libbsc_b200 -lbsc_b200 -Wl,-rpath,'$$ORIGIN/../../libbsc_b200'
