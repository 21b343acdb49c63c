# oracle/logic_replay.mk -- build the checkers of the reference's 8-bit logic capture files.  TEST INFRASTRUCTURE ONLY.
#
#   make -f logic_replay.mk : where the reference sources lie under $(REF), compile oracle/ref_logic_replay.cpp (write /
#                             read a logic WAV with hw::RecordDevice, replay one into lab::IsoDecoder as
#                             SignalStorageTask::readLogic streams it) twice, as oracle/iso_stream.mk does:
#     _ref/libnfcref_logic_replay.so  with the reference's UNMODIFIED logic decoder;
#     _ref/libnfcref_logic_b200.so    with the drop-in nfc_laboratory_b200/shim/IsoDecoderB200.cpp and libnfcb200.so.
#   Elsewhere it does nothing and the tests use the recorded output (tests/golden/ref_iso7816_u8.json.xz).
# Flags mirror the reference's release flags (CMakeLists.txt:22-23,36-40): -O3 -msse -msse3 -mno-avx, no FMA.

HERE     := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT      := $(HERE)_ref
REF      ?= /root/reference
ROOT     := $(abspath $(HERE)..)
LIB      := $(REF)/src/nfc-lib
LL       := $(LIB)/lib-lab/lab-logic/src/main
LD       := $(LIB)/lib-lab/lab-data/src/main
HW       := $(LIB)/lib-hw/hw-dev/src/main
RT       := $(LIB)/lib-rt/rt-lang/src/main
JSON     := $(LIB)/lib-ext/nlohmann/src/main/cpp
SHIM     := $(ROOT)/nfc_laboratory_b200/shim/IsoDecoderB200.cpp

CXX      ?= g++
REFFLAGS := -std=c++17 -O3 -fno-math-errno -msse -msse3 -mno-avx -pthread -fPIC -w
INCS     := -I$(LL)/include -I$(LL)/cpp -I$(LD)/include -I$(RT)/include -I$(HW)/include -I$(JSON)
LOGICSRC := $(LL)/cpp/IsoDecoder.cpp $(LL)/cpp/IsoTech.cpp $(LL)/cpp/tech/Iso7816.cpp
BASESRC  := $(LD)/cpp/Crc.cpp $(LD)/cpp/RawFrame.cpp \
            $(HW)/cpp/hw/SignalBuffer.cpp $(HW)/cpp/hw/RecordDevice.cpp \
            $(RT)/cpp/Logger.cpp $(RT)/cpp/FileSystem.cpp $(RT)/cpp/Format.cpp $(RT)/cpp/Map.cpp $(RT)/cpp/Tokenizer.cpp

.PHONY: all

all: $(if $(wildcard $(LL)/cpp/IsoDecoder.cpp),$(OUT)/libnfcref_logic_replay.so $(OUT)/libnfcref_logic_b200.so,)

$(OUT)/libnfcref_logic_replay.so: $(HERE)ref_logic_replay.cpp $(HERE)logic_replay.mk
	@mkdir -p $(OUT)
	$(CXX) $(REFFLAGS) -shared -Wl,-Bsymbolic $(INCS) -I$(ROOT)/include $(LOGICSRC) $(BASESRC) $(HERE)ref_logic_replay.cpp -o $@

# needs libnfcb200.so (nfc_laboratory_b200/csrc) built first; found at run time relative to the library
$(OUT)/libnfcref_logic_b200.so: $(HERE)ref_logic_replay.cpp $(HERE)logic_replay.mk $(SHIM) $(ROOT)/include/nfcb200.h
	@mkdir -p $(OUT)
	$(CXX) $(REFFLAGS) -shared -Wl,-Bsymbolic $(INCS) -I$(ROOT)/include $(SHIM) $(BASESRC) $(HERE)ref_logic_replay.cpp \
	   -L$(ROOT)/nfc_laboratory_b200 -lnfcb200 -Wl,-rpath,'$$ORIGIN/../../nfc_laboratory_b200' -o $@
