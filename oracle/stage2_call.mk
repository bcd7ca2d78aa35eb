# ORACLE — TEST INFRASTRUCTURE ONLY.
# _ref/stage2_call_test: the reference's own FindOverlapsAndRepetetiveRegions (RavenLib
# construct.cc and friends, compiled IN PLACE from $(REF), never copied) over the
# product's ram::MinimizerEngine facade, next to raven_b200::FindOverlapsAndRepetetiveRegions
# on rvn_find_overlaps_and_repetitive_regions (tests/test_gpu_stage2.py; driver source
# tests/cpp/stage2_call_test.cc).
# _ref/stage2_time: that fast route timed against the route it replaced
# (profiles/stage2.py; source profiles/stage2_time.cc).
# _ref/overlap_clip_test: the __host__ __device__ OverlapClip and IdentityBound
# (include/raven_b200/overlap_clip.hpp) against the reference's overlap_utils.cc on the
# host (tests/test_overlap_clip_host.py; source tests/cpp/overlap_clip_test.cc).
# Built only where $(REF) exists; elsewhere a prebuilt _ref/ (if any) is kept. Point REF
# at a checkout of lbcb-sci/raven v1.8.3.
#   make -C oracle -f stage2_call.mk
REF ?= /root/reference
CXX := /usr/bin/g++
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
ROOT := $(abspath $(HERE)..)
CPP := $(ROOT)/tests/cpp
FLAGS := -O2 -std=c++17 -pthread -w -I$(ROOT)/include -I$(REF)/RavenLib/include
LIBS := -L$(ROOT)/raven_b200 -lraven_b200 -Wl,-rpath,'$$ORIGIN/../../raven_b200'
SRCS := $(REF)/RavenLib/src/construct.cc $(REF)/RavenLib/src/pile.cc \
        $(REF)/RavenLib/src/overlap_utils.cc $(REF)/RavenLib/src/graph.cc
FACADE_SRCS := $(ROOT)/raven_b200/host/minimizer_engine.cc $(ROOT)/raven_b200/host/edlib.cc

ifneq ($(wildcard $(REF)/RavenLib/src/construct.cc),)
all: _ref/stage2_call_test _ref/overlap_clip_test _ref/stage2_time
_ref/stage2_call_test: $(CPP)/stage2_call_test.cc $(FACADE_SRCS) \
    $(ROOT)/include/ram/minimizer_engine.hpp $(ROOT)/include/raven_b200/construct_b200.hpp \
    $(ROOT)/include/raven_b200/overlap_clip.hpp $(ROOT)/raven_b200/libraven_b200.so
	mkdir -p _ref
	$(CXX) $(FLAGS) -o $@ $< $(FACADE_SRCS) $(SRCS) $(LIBS)
_ref/stage2_time: $(ROOT)/profiles/stage2_time.cc $(FACADE_SRCS) \
    $(ROOT)/include/ram/minimizer_engine.hpp $(ROOT)/include/raven_b200/construct_b200.hpp \
    $(ROOT)/include/raven_b200/overlap_clip.hpp $(ROOT)/raven_b200/libraven_b200.so
	mkdir -p _ref
	$(CXX) $(FLAGS) -O3 -o $@ $< $(FACADE_SRCS) $(SRCS) $(LIBS)
_ref/overlap_clip_test: $(CPP)/overlap_clip_test.cc $(ROOT)/include/raven_b200/overlap_clip.hpp
	mkdir -p _ref
	$(CXX) $(FLAGS) -o $@ $< $(REF)/RavenLib/src/overlap_utils.cc $(REF)/RavenLib/src/pile.cc
else
all:
	@echo "reference tree not present: keeping prebuilt oracle/_ref (if any)"
endif
.PHONY: all
