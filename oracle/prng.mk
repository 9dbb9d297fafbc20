# oracle/prng.mk -- builds the TEST-ONLY checkers of the device's PRNG paths (make -C oracle -f prng.mk), next to those of
# oracle/Makefile, which must have run first:
#   libshake256.so             : oracle/shake256.c, SHAKE256 and the Shake256PRNG stream from FIPS 202; always buildable.
#   _ref/libsealref_prng.so    : oracle/ref_prng.cpp, a C wrapper around the reference library _ref/libseal.so.
#   _ref/bin/shim_prng_test    : tests/cpp/shim_prng_test.cpp, seal_b200::Encryptor against seal::Encryptor under a
#                                Shake256PRNGFactory.
# The last two need the reference headers, so they are built where the reference sources are; elsewhere a prebuilt _ref/ is kept.
REF      ?= /root/reference
REFSRC   := $(REF)/native/src
OUT      := _ref
CXX      ?= g++
CC       ?= gcc

all: libshake256.so ref

libshake256.so: shake256.c
	$(CC) -O2 -fPIC -shared -Wall -Wextra -o $@ shake256.c

ifneq ($(wildcard $(REFSRC)/seal/seal.h),)
ref: $(OUT)/libsealref_prng.so $(OUT)/bin/shim_prng_test

$(OUT)/libsealref_prng.so: ref_prng.cpp $(OUT)/libseal.so
	$(CXX) -std=c++17 -O2 -fPIC -shared -pthread -I$(OUT)/include -I$(REFSRC) ref_prng.cpp -o $@ -L$(OUT) -lseal -Wl,-rpath,'$$ORIGIN'

SHIM_HDR := $(wildcard ../include/seal_b200/*.hpp) ../include/seal_b200.h
$(OUT)/bin/shim_prng_test: ../tests/cpp/shim_prng_test.cpp $(SHIM_HDR) $(OUT)/libseal.so ../seal_b200/libseal_b200.so
	@mkdir -p $(dir $@)
	$(CXX) -std=c++17 -O2 -pthread -I../include -I$(OUT)/include -I$(REFSRC) $< -o $@ -L$(OUT) -lseal -L../seal_b200 -lseal_b200 \
	    -Wl,-rpath,'$$ORIGIN/..' -Wl,-rpath,'$$ORIGIN/../../../seal_b200' -Wl,-rpath,/usr/local/cuda/lib64
else
ref:
	@echo "reference sources not present; keeping prebuilt $(OUT)/ (if any)"
endif

.PHONY: all ref
