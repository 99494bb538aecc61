# TEST INFRASTRUCTURE.  Builds oracle/_ref/scene2pset: the UNMODIFIED reference app apps/scene2pset/scene2pset.cc,
# compiled where it lies with the reference flags of oracle/Makefile and -fopenmp, linked like oracle/_ref/dmrecon
# against the libmve.a / libmve_util.a that `make ref` builds there.  Run after `make ref`:
#     make -f scene2pset.mk
# Skipped when $(REF) does not exist (GPU box: the prebuilt binary is used).
REF    ?= /root/reference
OUT    := _ref
CXX    := /usr/bin/g++
REFFLAGS := -O3 -g -march=x86-64-v3 -funsafe-math-optimizations -fno-math-errno -std=c++17 -pthread -fPIC -w \
            -DMVE_NO_PNG_SUPPORT -DMVE_NO_JPEG_SUPPORT -DMVE_NO_TIFF_SUPPORT -I$(REF)/libs

.PHONY: all
ifneq ($(wildcard $(REF)/apps/scene2pset/scene2pset.cc),)
all: $(OUT)/scene2pset
else
all:
	@echo "oracle/scene2pset.mk: $(REF) not present - using prebuilt oracle/_ref/scene2pset if any"
endif

$(OUT)/obj/app_scene2pset/scene2pset.o: $(REF)/apps/scene2pset/scene2pset.cc
	@mkdir -p $(dir $@)
	$(CXX) $(REFFLAGS) -fopenmp -c $< -o $@

$(OUT)/scene2pset: $(OUT)/obj/app_scene2pset/scene2pset.o $(OUT)/libmve.a $(OUT)/libmve_util.a
	$(CXX) $^ -fopenmp -pthread -static-libstdc++ -static-libgcc -o $@
