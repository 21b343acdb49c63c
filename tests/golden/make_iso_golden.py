"""Write tests/golden/ref_iso7816.json.xz: the reference ISO 7816 decoder's frames (oracle/_ref/libnfcref_iso.so) for the
seeded logic captures of nfc_laboratory_b200.synth.iso7816_capture (and of some of them with a CLK channel of more than
two levels, tests/iso_ref.py multilevel_clock), keyed by a hash of the input.  Run from the repository
root after building the oracle (oracle/iso.mk)."""
import json
import lzma
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import iso_ref as R  # noqa: E402

if __name__ == "__main__":
    assert R.ref_lib() is not None, "build the oracle first: make -C oracle -f iso.mk"
    out = {}
    for sc, rate in R.CASES:
        x = R.capture(sc, rate)
        out[R.key(x, rate)] = R.ref(x, rate)
        print(sc, rate, len(out[R.key(x, rate)]), "frames")
    for sc, rate, kind in R.CLOCK_CASES:
        x = R.clock_capture(sc, rate, kind)
        out[R.key(x, rate)] = R.ref(x, rate)
        print(sc, rate, kind, "clock", len(out[R.key(x, rate)]), "frames")
    with lzma.open(R.GOLDEN, "wt", preset=9) as f:
        json.dump(out, f, separators=(",", ":"))
