# oracle/keyset.mk -- builds the TEST-ONLY checkers of the device key sets and batch streams (make -C oracle -f keyset.mk), next to
# those of oracle/Makefile, which must have run first:
#   _ref/libsealref_keyset.so  : oracle/ref_keyset.cpp, the reference's RelinKeys / GaloisKeys / Ciphertext saved with compr_mode none
#                                or zlib (or as seeded Serializable objects) under a seeded factory, and its load of such streams.
#   _ref/bin/shim_keyset_test  : tests/cpp/shim_keyset_test.cpp, the DeviceRelinKeys / DeviceGaloisKeys overloads of
#                                seal_b200::Evaluator and seal_b200::KeyGenerator and the CiphertextBatch load / save against the
#                                seal:: classes; --bench times a batch load against seal::Ciphertext::load plus upload.
# Both need the reference headers, so they are built where the reference sources are; elsewhere a prebuilt _ref/ is kept.
REF      ?= /root/reference
REFSRC   := $(REF)/native/src
OUT      := _ref
CXX      ?= g++

all: ref

ifneq ($(wildcard $(REFSRC)/seal/seal.h),)
ref: $(OUT)/libsealref_keyset.so $(OUT)/bin/shim_keyset_test

$(OUT)/libsealref_keyset.so: ref_keyset.cpp $(OUT)/libseal.so
	$(CXX) -std=c++17 -O2 -fPIC -shared -pthread -I$(OUT)/include -I$(REFSRC) ref_keyset.cpp -o $@ -L$(OUT) -lseal -Wl,-rpath,'$$ORIGIN'

SHIM_HDR := $(wildcard ../include/seal_b200/*.hpp) ../include/seal_b200.h
$(OUT)/bin/shim_keyset_test: ../tests/cpp/shim_keyset_test.cpp $(SHIM_HDR) $(OUT)/libseal.so ../seal_b200/libseal_b200.so
	@mkdir -p $(dir $@)
	$(CXX) -std=c++17 -O2 -Wall -pthread -I../include -I$(OUT)/include -I$(REFSRC) $< -o $@ -L$(OUT) -lseal -L../seal_b200 -lseal_b200 \
	    -Wl,-rpath,'$$ORIGIN/..' -Wl,-rpath,'$$ORIGIN/../../../seal_b200' -Wl,-rpath,/usr/local/cuda/lib64
else
ref:
	@echo "reference sources not present; keeping prebuilt $(OUT)/ (if any)"
endif

.PHONY: all ref
