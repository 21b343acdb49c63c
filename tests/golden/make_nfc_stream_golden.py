"""Write tests/golden/ref_nfc_stream.json.xz: every field of the reference's frames for every run of
tests/nfc_stream_ref.py golden_entries() -- the fixture captures pushed whole and flushed, the settings matrix, IQ inputs,
the synthetic workloads, the flush sequences and the sample-rate changes -- one lab::NfcDecoder per run, its settings set
before the first buffer.  Needs oracle/_ref/libnfcref.so (oracle/Makefile builds it from the reference sources); run from
the repository root:

    python3 tests/golden/make_nfc_stream_golden.py
"""
import json
import lzma
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import nfc_stream_ref as T  # noqa: E402


def main():
    if T.ref_lib() is None:
        sys.exit("oracle/_ref/libnfcref.so is missing: run make -C oracle where the reference sources are")
    out = {}
    for name, steps, s in T.golden_entries():
        frames = T.ref_run(steps, s)
        out[name] = {"key": T.steps_key(steps, s), "frames": frames}
        print("%-60s %5d frames" % (name, len(frames)))
    with lzma.open(T.GOLDEN, "wt", preset=9) as f:
        json.dump(out, f, sort_keys=True, separators=(",", ":"))


if __name__ == "__main__":
    main()
