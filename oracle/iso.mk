# oracle/iso.mk -- build the ISO 7816 checker.  TEST INFRASTRUCTURE ONLY.
#
#   make -f iso.mk : where the reference sources lie under $(REF), compile its UNMODIFIED logic decoder (lab-logic:
#                    IsoDecoder.cpp, IsoTech.cpp, tech/Iso7816.cpp) with the rt-lang / hw-dev / lab-data units the radio
#                    oracle already uses, together with oracle/ref_iso.cpp, into oracle/_ref/libnfcref_iso.so.  Elsewhere
#                    it does nothing and the tests use the recorded output (tests/golden/ref_iso7816.json.xz).
# Flags mirror the reference's release flags (CMakeLists.txt:22-23,36-40): -O3 -msse -msse3 -mno-avx, no FMA.

HERE     := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT      := $(HERE)_ref
REF      ?= /root/reference
LIB      := $(REF)/src/nfc-lib
LL       := $(LIB)/lib-lab/lab-logic/src/main
LD       := $(LIB)/lib-lab/lab-data/src/main
HW       := $(LIB)/lib-hw/hw-dev/src/main
RT       := $(LIB)/lib-rt/rt-lang/src/main
JSON     := $(LIB)/lib-ext/nlohmann/src/main/cpp

CXX      ?= g++
REFFLAGS := -std=c++17 -O3 -fno-math-errno -msse -msse3 -mno-avx -pthread -fPIC -w
INCS     := -I$(LL)/include -I$(LL)/cpp -I$(LD)/include -I$(RT)/include -I$(HW)/include -I$(JSON)
ISOSRC   := $(LL)/cpp/IsoDecoder.cpp $(LL)/cpp/IsoTech.cpp $(LL)/cpp/tech/Iso7816.cpp \
            $(LD)/cpp/Crc.cpp $(LD)/cpp/RawFrame.cpp \
            $(HW)/cpp/hw/SignalBuffer.cpp $(HW)/cpp/hw/RecordDevice.cpp \
            $(RT)/cpp/Logger.cpp $(RT)/cpp/FileSystem.cpp $(RT)/cpp/Format.cpp $(RT)/cpp/Map.cpp $(RT)/cpp/Tokenizer.cpp

.PHONY: all

all: $(if $(wildcard $(LL)/cpp/IsoDecoder.cpp),$(OUT)/libnfcref_iso.so,)

$(OUT)/libnfcref_iso.so: $(HERE)ref_iso.cpp $(HERE)iso.mk
	@mkdir -p $(OUT)
	$(CXX) $(REFFLAGS) -shared -Wl,-Bsymbolic $(INCS) -I$(HERE)../include $(ISOSRC) $(HERE)ref_iso.cpp -o $@
