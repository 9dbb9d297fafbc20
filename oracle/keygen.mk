# oracle/keygen.mk -- builds the TEST-ONLY checkers of the device's key generation (make -C oracle -f keygen.mk), next to those of
# oracle/Makefile, which must have run first:
#   _ref/libsealref_keygen.so  : oracle/ref_keygen.cpp, a C wrapper around the reference library _ref/libseal.so
#                                (KeyGenerator under a seeded Blake2xb / Shake256 factory; also timed by tools/keygen_bench.py).
#   _ref/bin/shim_keygen_test  : tests/cpp/shim_keygen_test.cpp, seal_b200::KeyGenerator against seal::KeyGenerator.
# Both need the reference headers, so they are built where the reference sources are; elsewhere a prebuilt _ref/ is kept.
REF      ?= /root/reference
REFSRC   := $(REF)/native/src
OUT      := _ref
CXX      ?= g++

all: ref

ifneq ($(wildcard $(REFSRC)/seal/seal.h),)
ref: $(OUT)/libsealref_keygen.so $(OUT)/bin/shim_keygen_test

$(OUT)/libsealref_keygen.so: ref_keygen.cpp $(OUT)/libseal.so
	$(CXX) -std=c++17 -O2 -fPIC -shared -pthread -I$(OUT)/include -I$(REFSRC) ref_keygen.cpp -o $@ -L$(OUT) -lseal -Wl,-rpath,'$$ORIGIN'

SHIM_HDR := $(wildcard ../include/seal_b200/*.hpp) ../include/seal_b200.h
$(OUT)/bin/shim_keygen_test: ../tests/cpp/shim_keygen_test.cpp $(SHIM_HDR) $(OUT)/libseal.so ../seal_b200/libseal_b200.so
	@mkdir -p $(dir $@)
	$(CXX) -std=c++17 -O2 -pthread -I../include -I$(OUT)/include -I$(REFSRC) $< -o $@ -L$(OUT) -lseal -L../seal_b200 -lseal_b200 \
	    -Wl,-rpath,'$$ORIGIN/..' -Wl,-rpath,'$$ORIGIN/../../../seal_b200' -Wl,-rpath,/usr/local/cuda/lib64
else
ref:
	@echo "reference sources not present; keeping prebuilt $(OUT)/ (if any)"
endif

.PHONY: all ref
