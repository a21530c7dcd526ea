# Build libgoleft_b200.so (sm_90a only), the goleft CLI and the test oracle.
#   make            -> lib + cli + oracle
#   make lib        -> goleft_b200/libgoleft_b200.so
#   make cli        -> bin/goleft   (C++ host over the C ABI; links the .so)
#   make oracle     -> oracle/_build/liboracle.so  (TEST INFRASTRUCTURE, never linked into the product)
NVCC      ?= nvcc
CXX       ?= g++
CC        ?= gcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVFLAGS   := $(ARCH) -O3 -std=c++17 -lineinfo -Xcompiler -fPIC,-Wall,-Wno-unused-function -Xptxas -v --fmad=false
CXXFLAGS  := -O2 -std=c++17 -fPIC -Wall
CSRC      := goleft_b200/csrc
BUILD     := build
LIB       := goleft_b200/libgoleft_b200.so

CU_SRCS   := $(wildcard $(CSRC)/*.cu)
CPP_SRCS  := $(wildcard $(CSRC)/host/*.cpp)
CU_OBJS   := $(patsubst $(CSRC)/%.cu,$(BUILD)/%.o,$(CU_SRCS))
CPP_OBJS  := $(patsubst $(CSRC)/host/%.cpp,$(BUILD)/host_%.o,$(CPP_SRCS))
HDRS      := $(wildcard $(CSRC)/*.cuh) $(wildcard $(CSRC)/host/*.h) include/goleft_b200.h Makefile

NCCL_INC  ?= /usr/include
NCCL_LIB  ?= /usr/lib/x86_64-linux-gnu

all: lib cli oracle synth

lib: $(LIB)

$(BUILD)/%.o: $(CSRC)/%.cu $(HDRS)
	@mkdir -p $(BUILD)
	$(NVCC) $(NVFLAGS) -I$(NCCL_INC) -c $< -o $@ 2> $(BUILD)/$*.ptxas.log || (cat $(BUILD)/$*.ptxas.log; exit 1)

$(BUILD)/host_%.o: $(CSRC)/host/%.cpp $(HDRS)
	@mkdir -p $(BUILD)
	$(CXX) $(CXXFLAGS) -c $< -o $@

$(LIB): $(CU_OBJS) $(CPP_OBJS)
	$(NVCC) $(ARCH) -shared -o $@ $^ -lz -lpthread -ldl

CLI_SRCS := $(wildcard cli/*.cpp)
ifneq ($(CLI_SRCS),)
cli: bin/goleft
else
cli:
endif

bin/goleft: $(CLI_SRCS) $(LIB)
	@mkdir -p bin
	$(CXX) $(CXXFLAGS) -o $@ $(CLI_SRCS) -Iinclude -Lgoleft_b200 -lgoleft_b200 -Wl,-rpath,'$$ORIGIN/../goleft_b200' -lz -lpthread

oracle: oracle/_build/liboracle.so

oracle/_build/liboracle.so: $(wildcard oracle/*.c)
	@mkdir -p oracle/_build
	$(CC) -O3 -march=x86-64-v2 -fPIC -shared -Wall -ffp-contract=off -o $@ $^ -lm -lpthread

# bench workload generator (both bench arms load it; not part of the product library)
synth: tools/synth/libglsynth.so

tools/synth/libglsynth.so: tools/synth/glsynth.c tools/synth/bamsynth.c tools/synth/glsynth_core.h
	$(CC) -O2 -fPIC -shared -Wall -o $@ tools/synth/glsynth.c tools/synth/bamsynth.c -lpthread -lz

clean:
	rm -rf $(BUILD) $(LIB) bin oracle/_build tools/synth/libglsynth.so

.PHONY: all lib cli oracle synth clean
