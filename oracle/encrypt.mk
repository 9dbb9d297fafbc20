# oracle/encrypt.mk -- builds the TEST-ONLY checkers of encryption of device-resident plaintexts (make -C oracle -f encrypt.mk),
# next to those of oracle/Makefile, which must have run first:
#   _ref/libsealref_encrypt.so  : oracle/ref_encrypt.cpp, seal::Encryptor::encrypt / encrypt_symmetric under a seeded factory.
#   _ref/bin/shim_encrypt_test  : tests/cpp/shim_encrypt_test.cpp, the PlaintextBatch / CiphertextBatch members of
#                                 seal_b200::Encryptor, Decryptor and the encoders against the seal:: classes.
# Both need the reference headers, so they are built where the reference sources are; elsewhere a prebuilt _ref/ is kept.
REF      ?= /root/reference
REFSRC   := $(REF)/native/src
OUT      := _ref
CXX      ?= g++

all: ref

ifneq ($(wildcard $(REFSRC)/seal/seal.h),)
ref: $(OUT)/libsealref_encrypt.so $(OUT)/bin/shim_encrypt_test

$(OUT)/libsealref_encrypt.so: ref_encrypt.cpp $(OUT)/libseal.so
	$(CXX) -std=c++17 -O2 -fPIC -shared -pthread -I$(OUT)/include -I$(REFSRC) ref_encrypt.cpp -o $@ -L$(OUT) -lseal -Wl,-rpath,'$$ORIGIN'

SHIM_HDR := $(wildcard ../include/seal_b200/*.hpp) ../include/seal_b200.h
$(OUT)/bin/shim_encrypt_test: ../tests/cpp/shim_encrypt_test.cpp $(SHIM_HDR) $(OUT)/libseal.so ../seal_b200/libseal_b200.so
	@mkdir -p $(dir $@)
	$(CXX) -std=c++17 -O2 -Wall -pthread -I../include -I$(OUT)/include -I$(REFSRC) $< -o $@ -L$(OUT) -lseal -L../seal_b200 -lseal_b200 \
	    -Wl,-rpath,'$$ORIGIN/..' -Wl,-rpath,'$$ORIGIN/../../../seal_b200' -Wl,-rpath,/usr/local/cuda/lib64
else
ref:
	@echo "reference sources not present; keeping prebuilt $(OUT)/ (if any)"
endif

.PHONY: all ref
