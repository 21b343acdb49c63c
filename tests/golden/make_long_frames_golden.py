"""Write tests/golden/ref_long_frames.json.xz: for every input of tests/long_frames.py golden_inputs() -- the long-frame
cases, the streams of the dense batch and the two pool-overflow captures -- a hash of the input and every field of the
reference's frames (one lab::NfcDecoder fed 65 536-sample buffers, then nextFrames({})); the two overflow captures as a
count and a digest of those records.  Needs oracle/_ref/libnfcref.so (oracle/Makefile builds it from the
reference sources); run from the repository root:

    python3 tests/golden/make_long_frames_golden.py
"""
import json
import lzma
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import long_frames as L  # noqa: E402
import nfc_stream_ref as T  # noqa: E402


def main():
    if T.ref_lib() is None:
        sys.exit("oracle/_ref/libnfcref.so is missing: run make -C oracle where the reference sources are")
    out = {}
    for name, build in L.golden_inputs().items():
        out[name] = L.golden_entry(name, build())
        print("%-40s %6d frames" % (name, out[name].get("count", len(out[name].get("frames", [])))))
    with lzma.open(L.GOLDEN, "wt", preset=9) as f:
        json.dump(out, f, sort_keys=True, separators=(",", ":"))


if __name__ == "__main__":
    main()
