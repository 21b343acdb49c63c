"""Random ISO 7816 logic captures through the host build of the device decoder (tests/native/iso_host.cpp) and the
compiled reference (oracle/_ref/libnfcref_iso.so); prints every capture whose frames differ and a summary line.

Each capture is a generator scenario at a random rate from 4 to 60 MS/s with a random seed, optionally with random
one-sample pulses on any channel and, for some, a random high level per channel in place of 1 (the decoder only sees
signs)."""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import iso_ref as R  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100)
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()
    assert R.ref_lib() is not None, "build the oracle first: make -C oracle -f iso.mk"
    rng = np.random.default_rng(a.seed)
    bad = 0
    frames = 0
    for i in range(a.n):
        sc = R.S.ISO_SCENARIOS[rng.integers(len(R.S.ISO_SCENARIOS))]
        rate = int(rng.integers(4, 61)) * 1_000_000
        x = R.S.iso7816_capture(sc, rate, seed=int(rng.integers(1 << 30)), glitches=bool(rng.integers(2)))
        for _ in range(int(rng.integers(0, 6))):
            x[rng.integers(len(x)), rng.integers(4)] = 1 - x[rng.integers(len(x)), rng.integers(4)]
        if rng.integers(4) == 0:
            x = (x * rng.uniform(0.25, 1.0, size=4)).astype(np.float32)
        st = int(rng.integers(0, 1 << 31))
        h, r = R.host(x, rate, stream_time=st), R.ref(x, rate, stream_time=st)
        frames += len(r)
        if h != r:
            bad += 1
            print("DIFF capture %d: %s at %d S/s, %d host frames, %d reference frames" % (i, sc, rate, len(h), len(r)))
    print("%d captures, %d reference frames, %d differ" % (a.n, frames, bad))


if __name__ == "__main__":
    main()
