# oracle/bspgemm.mk -- the block SpGEMM checker (TEST INFRASTRUCTURE ONLY), built by `make -C oracle -f bspgemm.mk`.
#
#   libkkoracle_bspgemm.so      restatement of bspgemm_debug_numeric, -ffp-contract=off (kk_oracle_bspgemm.c)
#   _ref/libkkref_bspgemm.so    the REFERENCE's own bspgemm_debug_numeric
#                               (sparse/impl/KokkosSparse_bspgemm_impl_seq.hpp) and its GEMM
#                               (batched/dense/impl/KokkosBatched_Gemm_Serial_Internal.hpp), compiled where they lie over
#                               the stand-ins in oracle/kokkos_mock/bspgemm; the reference's blocked inner GEMM is skipped
#                               through its include guard.  Built only when the reference tree (REF) exists; elsewhere a prebuilt
#                               file is kept if there is one.
CC = gcc
CXX = g++
# the reference tree: the same default as oracle/Makefile (override with REF=...)
REF ?= $(shell sed -n 's/^REF ?= //p' Makefile)
CFLAGS = -O2 -fPIC -shared -fvisibility=hidden -std=gnu11 -Wall -Wno-unused-function

all: libkkoracle_bspgemm.so ref

libkkoracle_bspgemm.so: kk_oracle_bspgemm.c bspgemm.mk
	$(CC) $(CFLAGS) -ffp-contract=off -o $@.tmp.$$$$ kk_oracle_bspgemm.c && mv -f $@.tmp.$$$$ $@

REF_SRCS = kkref_bspgemm.cpp bspgemm.mk $(wildcard kokkos_mock/bspgemm/*.hpp)
ref:
	@if [ -f $(REF)/sparse/impl/KokkosSparse_bspgemm_impl_seq.hpp ]; then $(MAKE) --no-print-directory -f bspgemm.mk _ref/libkkref_bspgemm.so; \
	else echo "reference tree absent: keeping prebuilt oracle/_ref/libkkref_bspgemm.so (if any)"; fi

_ref/libkkref_bspgemm.so: $(REF_SRCS)
	@mkdir -p _ref && T=_ref/.tmp.bsp.$$$$ && mkdir -p $$T && \
	  $(CXX) -O2 -fPIC -std=c++17 -ffp-contract=off -I kokkos_mock/bspgemm -I $(REF)/batched/dense/impl \
	    -DKOKKOSBATCHED_INNER_GEMM_FIX_C_SERIAL_IMPL_HPP \
	    -DKKREF_BSPGEMM_SEQ='"$(REF)/sparse/impl/KokkosSparse_bspgemm_impl_seq.hpp"' \
	    -c -o $$T/kkref_bspgemm.o kkref_bspgemm.cpp && \
	  $(CXX) -shared -o $$T/libkkref_bspgemm.so $$T/kkref_bspgemm.o && \
	  mv -f $$T/libkkref_bspgemm.so _ref/libkkref_bspgemm.so && rm -rf $$T && echo "built oracle/_ref/libkkref_bspgemm.so"

.PHONY: all ref
