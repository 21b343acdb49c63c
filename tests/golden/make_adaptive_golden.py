#!/usr/bin/env python3
"""Generate tests/golden/ref_adaptive.npz.xz: the reference's adaptive signal points (oracle/_ref/libnfcref_adaptive.so,
built by oracle/adaptive.mk where the reference sources are present) of the inputs of tests/adaptive_ref.py RADIO_CASES
and LOGIC_CASES, keyed by a hash of input and buffer, and the members of the .trz files its TraceStorageTask writes for
TRZ_RADIO and TRZ_LOGIC.  The adaptive signal tests read it where the oracle cannot be built.

Usage: python tests/golden/make_adaptive_golden.py
"""
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import adaptive_ref  # noqa: E402


def main():
    assert adaptive_ref.oracle_lib() is not None, "oracle/_ref/libnfcref_adaptive.so is missing: make -C oracle -f adaptive.mk"
    with tempfile.TemporaryDirectory() as tmp:
        n = adaptive_ref.record(tmp)
    print("%-40s %d arrays" % (os.path.basename(adaptive_ref.RECORDED), n))


if __name__ == "__main__":
    main()
