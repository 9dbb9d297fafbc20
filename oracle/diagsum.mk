# oracle/diagsum.mk -- builds the TEST-ONLY checker of the diagonal sums (make -C oracle -f diagsum.mk), next to those
# of oracle/Makefile, which must have run first:
#   _ref/bin/shim_diagsum_test   : tests/cpp/shim_diagsum_test.cpp with ref_diagsum.cpp, Evaluator::apply_galois_multiply_plain_add_inplace and diagonal_sum on CiphertextBatch
#                               against the chains of seal::Evaluator::apply_galois_inplace or rotate_rows_inplace / rotate_vector_inplace, multiply_plain_inplace and add_inplace.
# It needs the reference headers, so it is built where the reference sources are; elsewhere a prebuilt _ref/ is kept.
REF      ?= /root/reference
REFSRC   := $(REF)/native/src
OUT      := _ref
CXX      ?= g++

all: ref

ifneq ($(wildcard $(REFSRC)/seal/seal.h),)
ref: $(OUT)/bin/shim_diagsum_test

SHIM_HDR := $(wildcard ../include/seal_b200/*.hpp) ../include/seal_b200.h
$(OUT)/bin/shim_diagsum_test: ../tests/cpp/shim_diagsum_test.cpp ref_diagsum.cpp $(SHIM_HDR) $(OUT)/libseal.so ../seal_b200/libseal_b200.so
	@mkdir -p $(dir $@)
	$(CXX) -std=c++17 -O2 -Wall -pthread -I../include -I$(OUT)/include -I$(REFSRC) $< ref_diagsum.cpp -o $@ -L$(OUT) -lseal -L../seal_b200 -lseal_b200 \
	    -Wl,-rpath,'$$ORIGIN/..' -Wl,-rpath,'$$ORIGIN/../../../seal_b200' -Wl,-rpath,/usr/local/cuda/lib64
else
ref:
	@echo "reference sources not present; keeping prebuilt $(OUT)/ (if any)"
endif

.PHONY: all ref
