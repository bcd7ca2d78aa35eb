# ORACLE — TEST INFRASTRUCTURE ONLY.
# _ref/facade_batch_test: the reference's own stage 1 and stage 2 (RavenLib
# construct.cc and friends, compiled IN PLACE from $(REF), never copied) over the
# product's ram::MinimizerEngine facade and libraven_b200.so, printing the facade's
# Map counters (tests/test_gpu_facade_batch.py; driver source
# tests/cpp/facade_batch_test.cc). Built only where $(REF) exists; elsewhere a
# prebuilt _ref/ (if any) is kept. Point REF at a checkout of lbcb-sci/raven v1.8.3.
#   make -C oracle -f facade_batch.mk
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
all: _ref/facade_batch_test
_ref/facade_batch_test: $(CPP)/facade_batch_test.cc $(FACADE_SRCS) \
    $(ROOT)/include/ram/minimizer_engine.hpp $(ROOT)/include/raven_b200/construct_b200.hpp \
    $(ROOT)/raven_b200/libraven_b200.so
	mkdir -p _ref
	$(CXX) $(FLAGS) -o $@ $< $(FACADE_SRCS) $(SRCS) $(LIBS)
else
all:
	@echo "reference tree not present: keeping prebuilt oracle/_ref (if any)"
endif
.PHONY: all
