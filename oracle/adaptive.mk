# oracle/adaptive.mk -- build the adaptive signal checker.  TEST INFRASTRUCTURE ONLY.
#
#   make -f adaptive.mk : where the reference sources lie under $(REF), compile its UNMODIFIED lab-tasks units
#                         SignalResamplingTask.cpp and TraceStorageTask.cpp with the rt-lang runtime, hw-dev's SignalBuffer,
#                         lab-data's RawFrame, microtar and zlib, together with oracle/ref_adaptive.cpp, into
#                         oracle/_ref/libnfcref_adaptive.so.  Elsewhere it does nothing and the tests use the recorded output
#                         (tests/golden/ref_adaptive.npz.xz).
# Flags mirror the reference's release flags (CMakeLists.txt:22-23,36-40): -O3 -msse -msse3 -mno-avx, no FMA; lab-tasks
# adds -msse2 -DUSE_SSE2 on x86 (lab-tasks/CMakeLists.txt:17-19).  No -fopenmp: processLogicSignal's channels run in order.

HERE     := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT      := $(HERE)_ref
REF      ?= /root/reference
LIB      := $(REF)/src/nfc-lib
LT       := $(LIB)/lib-lab/lab-tasks/src/main
LD       := $(LIB)/lib-lab/lab-data/src/main
HW       := $(LIB)/lib-hw/hw-dev/src/main
RT       := $(LIB)/lib-rt/rt-lang/src/main
JSON     := $(LIB)/lib-ext/nlohmann/src/main/cpp
MTAR     := $(LIB)/lib-ext/microtar/src/main/c

CXX      ?= g++
CC       ?= gcc
FLAGS    := -O3 -fno-math-errno -msse -msse3 -mno-avx -pthread -fPIC -w
INCS     := -I$(LT)/include -I$(LT)/cpp/tasks -I$(LD)/include -I$(RT)/include -I$(HW)/include -I$(JSON) -I$(MTAR)
SRC      := $(LT)/cpp/tasks/SignalResamplingTask.cpp $(LT)/cpp/tasks/TraceStorageTask.cpp \
            $(LD)/cpp/RawFrame.cpp $(HW)/cpp/hw/SignalBuffer.cpp \
            $(RT)/cpp/Logger.cpp $(RT)/cpp/Format.cpp $(RT)/cpp/Map.cpp $(RT)/cpp/Worker.cpp $(RT)/cpp/Package.cpp \
            $(RT)/cpp/FileSystem.cpp $(RT)/cpp/Tokenizer.cpp

.PHONY: all

all: $(if $(wildcard $(LT)/cpp/tasks/SignalResamplingTask.cpp),$(OUT)/libnfcref_adaptive.so,)

$(OUT)/libnfcref_adaptive.so: $(HERE)ref_adaptive.cpp $(HERE)adaptive.mk
	@mkdir -p $(OUT)/adobj
	$(CC) -std=gnu99 $(FLAGS) -c $(MTAR)/microtar.c -o $(OUT)/adobj/microtar.o
	$(CXX) -std=c++17 $(FLAGS) -msse2 -DUSE_SSE2 -shared -Wl,-Bsymbolic $(INCS) $(SRC) $(HERE)ref_adaptive.cpp $(OUT)/adobj/microtar.o -o $@ -lz
	rm -rf $(OUT)/adobj
