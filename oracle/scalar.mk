# oracle/scalar.mk -- builds the TEST-ONLY checkers of the scalar CKKS encoder (make -C oracle -f scalar.mk), next to those of
# oracle/Makefile, which must have run first:
#   _ref/libsealref_scalar.so  : oracle/ref_scalar.cpp, the reference's CKKSEncoder::encode of one double, complex number or int64.
#   _ref/bin/shim_scalar_test  : tests/cpp/shim_scalar_test.cpp, the scalar overloads of seal_b200::CKKSEncoder (Plaintext and
#                                PlaintextBatch) and the reference's example 5 on device-resident batches against seal::CKKSEncoder /
#                                seal::Evaluator.
# Both need the reference headers, so they are built where the reference sources are; elsewhere a prebuilt _ref/ is kept.
REF      ?= /root/reference
REFSRC   := $(REF)/native/src
OUT      := _ref
CXX      ?= g++

all: ref

ifneq ($(wildcard $(REFSRC)/seal/seal.h),)
ref: $(OUT)/libsealref_scalar.so $(OUT)/bin/shim_scalar_test

$(OUT)/libsealref_scalar.so: ref_scalar.cpp $(OUT)/libseal.so
	$(CXX) -std=c++17 -O2 -fPIC -shared -pthread -I$(OUT)/include -I$(REFSRC) ref_scalar.cpp -o $@ -L$(OUT) -lseal -Wl,-rpath,'$$ORIGIN'

SHIM_HDR := $(wildcard ../include/seal_b200/*.hpp) ../include/seal_b200.h
$(OUT)/bin/shim_scalar_test: ../tests/cpp/shim_scalar_test.cpp $(SHIM_HDR) $(OUT)/libseal.so ../seal_b200/libseal_b200.so
	@mkdir -p $(dir $@)
	$(CXX) -std=c++17 -O2 -Wall -pthread -I../include -I$(OUT)/include -I$(REFSRC) $< -o $@ -L$(OUT) -lseal -L../seal_b200 -lseal_b200 \
	    -Wl,-rpath,'$$ORIGIN/..' -Wl,-rpath,'$$ORIGIN/../../../seal_b200' -Wl,-rpath,/usr/local/cuda/lib64
else
ref:
	@echo "reference sources not present; keeping prebuilt $(OUT)/ (if any)"
endif

.PHONY: all ref
