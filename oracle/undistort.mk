# TEST INFRASTRUCTURE.  Builds oracle/_ref/undistort_harness: oracle/undistort_harness.cc, our driver around the
# reference's unmodified mve::image::image_undistort_k2k4<uint8_t>, compiled with the reference flags of oracle/Makefile
# and linked like oracle/_ref/ref_harness (no -funsafe-math-optimizations on the link line) against the libmve.a /
# libmve_util.a that `make ref` builds there.  Run after `make ref`:
#     make -f undistort.mk
# Skipped when $(REF) does not exist (GPU box: the prebuilt binary is used).
REF    ?= /root/reference
OUT    := _ref
CXX    := /usr/bin/g++
REFFLAGS := -O3 -g -march=x86-64-v3 -funsafe-math-optimizations -fno-math-errno -std=c++17 -pthread -fPIC -w \
            -DMVE_NO_PNG_SUPPORT -DMVE_NO_JPEG_SUPPORT -DMVE_NO_TIFF_SUPPORT -I$(REF)/libs

.PHONY: all
ifneq ($(wildcard $(REF)/libs/mve/image_tools.h),)
all: $(OUT)/undistort_harness
else
all:
	@echo "oracle/undistort.mk: $(REF) not present - using prebuilt oracle/_ref/undistort_harness if any"
endif

$(OUT)/obj/undistort_harness.o: undistort_harness.cc
	@mkdir -p $(dir $@)
	$(CXX) $(REFFLAGS) -c undistort_harness.cc -o $@

$(OUT)/undistort_harness: $(OUT)/obj/undistort_harness.o $(OUT)/libmve.a $(OUT)/libmve_util.a
	$(CXX) $^ -pthread -static-libstdc++ -static-libgcc -o $@
