# oracle/serial.mk -- builds the TEST-ONLY checkers of the device's seed-compressed streams (make -C oracle -f serial.mk), next to
# those of oracle/Makefile, which must have run first:
#   _ref/libsealref_serial.so  : oracle/ref_serial.cpp, the reference's Serializable<...>::save(none) bytes of KeyGenerator and
#                                Encryptor under a seeded factory, and its load of such streams (also timed by tools/keygen_bench.py).
#   _ref/bin/shim_serial_test  : tests/cpp/shim_serial_test.cpp, the Serializable overloads of seal_b200::KeyGenerator and
#                                seal_b200::Encryptor against the seal:: classes.
# Both need the reference headers, so they are built where the reference sources are; elsewhere a prebuilt _ref/ is kept.
REF      ?= /root/reference
REFSRC   := $(REF)/native/src
OUT      := _ref
CXX      ?= g++

all: ref

ifneq ($(wildcard $(REFSRC)/seal/seal.h),)
ref: $(OUT)/libsealref_serial.so $(OUT)/bin/shim_serial_test

$(OUT)/libsealref_serial.so: ref_serial.cpp $(OUT)/libseal.so
	$(CXX) -std=c++17 -O2 -fPIC -shared -pthread -I$(OUT)/include -I$(REFSRC) ref_serial.cpp -o $@ -L$(OUT) -lseal -Wl,-rpath,'$$ORIGIN'

SHIM_HDR := $(wildcard ../include/seal_b200/*.hpp) ../include/seal_b200.h
$(OUT)/bin/shim_serial_test: ../tests/cpp/shim_serial_test.cpp $(SHIM_HDR) $(OUT)/libseal.so ../seal_b200/libseal_b200.so
	@mkdir -p $(dir $@)
	$(CXX) -std=c++17 -O2 -Wall -pthread -I../include -I$(OUT)/include -I$(REFSRC) $< -o $@ -L$(OUT) -lseal -L../seal_b200 -lseal_b200 \
	    -Wl,-rpath,'$$ORIGIN/..' -Wl,-rpath,'$$ORIGIN/../../../seal_b200' -Wl,-rpath,/usr/local/cuda/lib64
else
ref:
	@echo "reference sources not present; keeping prebuilt $(OUT)/ (if any)"
endif

.PHONY: all ref
