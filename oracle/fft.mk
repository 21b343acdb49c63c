# oracle/fft.mk -- build the spectrum checker.  TEST INFRASTRUCTURE ONLY.
#
#   make -f fft.mk : where the reference sources lie under $(REF), compile its UNMODIFIED FFT library mufft
#                    (lib-ext/mufft: fft.c kernel.c cpu.c, -DMUFFT_HAVE_X86 as lib-ext/mufft/CMakeLists.txt gives that
#                    target) together with oracle/ref_fft.cpp into oracle/_ref/libnfcref_fft.so.  Elsewhere it does
#                    nothing and the tests use the recorded output (tests/golden/ref_spectrum.npz.xz).
#
# mufft's CMakeLists.txt gives MUFFT_HAVE_SSE / SSE3 / AVX only to the SIMD kernel targets, not to fft.c, so the library
# the reference links registers the plain C kernels alone; the SIMD kernel files are therefore not compiled here.
# Flags mirror the reference's release flags (CMakeLists.txt:22-23,36-40): -O3 -msse -msse3 -mno-avx, no FMA.

HERE     := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT      := $(HERE)_ref
REF      ?= /root/reference
MUFFT    := $(REF)/src/nfc-lib/lib-ext/mufft/src/main/c

CXX      ?= g++
CC       ?= gcc
FLAGS    := -O3 -fno-math-errno -msse -msse3 -mno-avx -pthread -fPIC -w

.PHONY: all

all: $(if $(wildcard $(MUFFT)/fft.c),$(OUT)/libnfcref_fft.so,)

$(OUT)/libnfcref_fft.so: $(HERE)ref_fft.cpp
	@mkdir -p $(OUT)/fftobj
	for f in fft kernel cpu; do $(CC) -std=gnu99 $(FLAGS) -DMUFFT_HAVE_X86 -I$(MUFFT) -c $(MUFFT)/$$f.c -o $(OUT)/fftobj/$$f.o || exit 1; done
	$(CXX) -std=c++17 $(FLAGS) -shared -I$(MUFFT) $(HERE)ref_fft.cpp $(OUT)/fftobj/*.o -o $@ -lm
	rm -rf $(OUT)/fftobj
