# oracle/noise.mk -- builds the TEST-ONLY checkers of the device's invariant noise budget (make -C oracle -f noise.mk), next to
# those of oracle/Makefile, which must have run first:
#   _ref/libsealref_noise.so   : oracle/ref_noise.cpp, a C wrapper around the reference library _ref/libseal.so
#                                (Decryptor::invariant_noise_budget under a given secret key).
#   _ref/bin/shim_noise_test   : tests/cpp/shim_noise_test.cpp, seal_b200::Decryptor's noise budget and CiphertextBatch
#                                overloads against seal::Decryptor.
# Both need the reference headers, so they are built where the reference sources are; elsewhere a prebuilt _ref/ is kept.
REF      ?= /root/reference
REFSRC   := $(REF)/native/src
OUT      := _ref
CXX      ?= g++

all: ref

ifneq ($(wildcard $(REFSRC)/seal/seal.h),)
ref: $(OUT)/libsealref_noise.so $(OUT)/bin/shim_noise_test

$(OUT)/libsealref_noise.so: ref_noise.cpp $(OUT)/libseal.so
	$(CXX) -std=c++17 -O2 -fPIC -shared -pthread -I$(OUT)/include -I$(REFSRC) ref_noise.cpp -o $@ -L$(OUT) -lseal -Wl,-rpath,'$$ORIGIN'

SHIM_HDR := $(wildcard ../include/seal_b200/*.hpp) ../include/seal_b200.h
$(OUT)/bin/shim_noise_test: ../tests/cpp/shim_noise_test.cpp $(SHIM_HDR) $(OUT)/libseal.so ../seal_b200/libseal_b200.so
	@mkdir -p $(dir $@)
	$(CXX) -std=c++17 -O2 -pthread -I../include -I$(OUT)/include -I$(REFSRC) $< -o $@ -L$(OUT) -lseal -L../seal_b200 -lseal_b200 \
	    -Wl,-rpath,'$$ORIGIN/..' -Wl,-rpath,'$$ORIGIN/../../../seal_b200' -Wl,-rpath,/usr/local/cuda/lib64
else
ref:
	@echo "reference sources not present; keeping prebuilt $(OUT)/ (if any)"
endif

.PHONY: all ref
