# oracle/multsum.mk -- builds the TEST-ONLY checker of the sums of ciphertext products (make -C oracle -f multsum.mk), next to those
# of oracle/Makefile, which must have run first:
#   _ref/bin/shim_multsum_test   : tests/cpp/shim_multsum_test.cpp with ref_multsum.cpp, Evaluator::multiply_sum and multiply_relinearize_sum on CiphertextBatch
#                                against the chain of seal::Evaluator::multiply_inplace, add_many and relinearize_inplace.
# It needs the reference headers, so it is built where the reference sources are; elsewhere a prebuilt _ref/ is kept.
REF      ?= /root/reference
REFSRC   := $(REF)/native/src
OUT      := _ref
CXX      ?= g++

all: ref

ifneq ($(wildcard $(REFSRC)/seal/seal.h),)
ref: $(OUT)/bin/shim_multsum_test

SHIM_HDR := $(wildcard ../include/seal_b200/*.hpp) ../include/seal_b200.h
$(OUT)/bin/shim_multsum_test: ../tests/cpp/shim_multsum_test.cpp ref_multsum.cpp $(SHIM_HDR) $(OUT)/libseal.so ../seal_b200/libseal_b200.so
	@mkdir -p $(dir $@)
	$(CXX) -std=c++17 -O2 -Wall -pthread -I../include -I$(OUT)/include -I$(REFSRC) $< ref_multsum.cpp -o $@ -L$(OUT) -lseal -L../seal_b200 -lseal_b200 \
	    -Wl,-rpath,'$$ORIGIN/..' -Wl,-rpath,'$$ORIGIN/../../../seal_b200' -Wl,-rpath,/usr/local/cuda/lib64
else
ref:
	@echo "reference sources not present; keeping prebuilt $(OUT)/ (if any)"
endif

.PHONY: all ref
