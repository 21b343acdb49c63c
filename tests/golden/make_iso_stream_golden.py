"""Write tests/golden/ref_iso7816_stream.json.xz: the reference's frames for every case of tests/iso_stream_ref.py pushed by
every one of its seeded chunk plans (one lab::IsoDecoder, one nextFrames per chunk, then nextFrames({})).  Needs the
checker oracle/iso_stream.mk builds from the reference sources; run from the repository root:

    python3 tests/golden/make_iso_stream_golden.py
"""
import json
import lzma
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import iso_stream_ref as T  # noqa: E402


def main():
    lib = T.ref_lib()
    if lib is None:
        sys.exit("oracle/_ref/libnfcref_iso_stream.so is missing: run make -C oracle -f iso_stream.mk where the reference sources are")
    out = {}
    for case in T.CASES:
        for plan, (x, chunks, rates) in T.plans(case).items():
            frames = T.chunked(lib, x, chunks, rates)
            out["%s/%s" % (T.case_id(case), plan)] = {"key": T.plan_key(x, chunks, rates), "chunks": len(chunks), "frames": frames}
            print("%-28s %-10s %6d chunks %4d frames" % (T.case_id(case), plan, len(chunks), len(frames)))
    with lzma.open(T.GOLDEN, "wt", preset=9) as f:
        json.dump(out, f, sort_keys=True, separators=(",", ":"))


if __name__ == "__main__":
    main()
