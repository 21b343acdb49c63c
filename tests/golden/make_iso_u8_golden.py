"""Write tests/golden/ref_iso7816_u8.json.xz: for every case of tests/logic_ref.py, the SHA-256 of the 8-bit logic WAV the
reference's hw::RecordDevice writes for it and the reference's frames when that file is replayed as
SignalStorageTask::readLogic streams it (65 536-sample buffers into one lab::IsoDecoder, then nextFrames({})).  Needs the
checker oracle/logic_replay.mk builds from the reference sources; run from the repository root:

    python3 tests/golden/make_iso_u8_golden.py
"""
import json
import lzma
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import logic_ref as L  # noqa: E402


def main():
    lib = L.ref_lib()
    if lib is None:
        sys.exit("oracle/_ref/libnfcref_logic_replay.so is missing: run make -C oracle -f logic_replay.mk where the reference sources are")
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "logic.wav")
        for case in L.CASES:
            L.ref_write(lib, path, case)
            frames = L.replay(lib, path)
            out[L.case_id(case)] = {"sha256": L.sha256(path), "samples": len(L.samples(case)), "frames": frames}
            print("%-30s %9d samples %4d frames" % (L.case_id(case), len(L.samples(case)), len(frames)))
    with lzma.open(L.GOLDEN, "wt", preset=9) as f:
        json.dump(out, f, sort_keys=True, separators=(",", ":"))


if __name__ == "__main__":
    main()
