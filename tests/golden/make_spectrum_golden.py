#!/usr/bin/env python3
"""Generate tests/golden/ref_spectrum.npz.xz: the reference's FFT spectrum frames (oracle/_ref/libnfcref_fft.so, built by
oracle/fft.mk where the reference sources are present) of the seeded inputs of tests/spectrum_ref.py CASES, keyed by a
hash of input and parameters.  The spectrum tests read it where the oracle cannot be built.

Usage: python tests/golden/make_spectrum_golden.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import spectrum_ref  # noqa: E402


def main():
    assert spectrum_ref.oracle_lib() is not None, "oracle/_ref/libnfcref_fft.so is missing: make -C oracle -f fft.mk"
    spectrum_ref.record()
    print("%-40s %d inputs" % (os.path.basename(spectrum_ref.RECORDED), len(spectrum_ref.CASES)))


if __name__ == "__main__":
    main()
