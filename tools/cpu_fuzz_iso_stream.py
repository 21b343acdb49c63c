"""Random ISO 7816 logic captures pushed buffer by buffer through the host build of the stream push
(tests/native/iso_stream_host.cpp) and through one reference lab::IsoDecoder fed the same buffers
(oracle/_ref/libnfcref_iso_stream.so); prints every case whose frames differ and a summary line.

Each case is a generator scenario at a random rate from 4 to 60 MS/s with a random seed (the captures of
tools/cpu_fuzz_iso.py: random one-sample pulses, random high levels), optionally followed in the same stream by a second
capture at another random rate, cut into buffers by a random plan: tiny (1-63 samples) around a random point, random
1 000-300 000, fixed 65 536, or one split at a random point inside a window where RST is low."""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import iso_ref as R  # noqa: E402
import iso_stream_ref as T  # noqa: E402


def capture(rng):
    sc = R.S.ISO_SCENARIOS[rng.integers(len(R.S.ISO_SCENARIOS))]
    rate = int(rng.integers(4, 61)) * 1_000_000
    x = R.S.iso7816_capture(sc, rate, seed=int(rng.integers(1 << 30)), glitches=bool(rng.integers(2)))
    for _ in range(int(rng.integers(0, 6))):
        x[rng.integers(len(x)), rng.integers(4)] = 1 - x[rng.integers(len(x)), rng.integers(4)]
    if rng.integers(4) == 0:
        x = (x * rng.uniform(0.25, 1.0, size=4)).astype(np.float32)
    return sc, rate, x


def chunk_plan(rng, x):
    n = len(x)
    kind = ("tiny", "random", "p65536", "split")[rng.integers(4)]
    if kind == "tiny":
        a = int(rng.integers(0, max(1, n - 20_000)))
        w = min(20_000, n - a)
        tiny = []
        while sum(tiny) < w:
            tiny.append(int(min(rng.integers(1, 64), w - sum(tiny))))
        return kind, [c for c in [a] + tiny + [n - a - w] if c]
    if kind == "random":
        return kind, T._random_chunks(rng, n, 1_000, 300_000)
    if kind == "p65536":
        return kind, [65_536] * (n // 65_536) + ([n % 65_536] if n % 65_536 else [])
    windows = [(b, e) for b, e in T.rst_low_windows(x) if e - b > 1]
    b, e = windows[rng.integers(len(windows))] if windows else (1, n)
    m = int(rng.integers(b, e))
    return kind, [m, n - m] if 0 < m < n else [n]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100)
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()
    assert T.ref_lib() is not None, "build the oracle first: make -C oracle -f iso_stream.mk"
    rng = np.random.default_rng(a.seed)
    bad = frames = 0
    for i in range(a.n):
        sc, rate, x = capture(rng)
        kind, chunks = chunk_plan(rng, x)
        rates = [rate] * len(chunks)
        if rng.integers(3) == 0:  # a second capture at another rate in the same stream
            sc2, rate2, y = capture(rng)
            kind2, chunks2 = chunk_plan(rng, y)
            x = np.concatenate([x, y])
            chunks += chunks2
            rates += [rate2] * len(chunks2)
            sc, kind = sc + "+" + sc2, kind + "+" + kind2
        st = int(rng.integers(0, 1 << 31))
        h, r = T.host(x, chunks, rates, stream_time=st), T.chunked(T.ref_lib(), x, chunks, rates, stream_time=st)
        frames += len(r)
        if h != r:
            bad += 1
            print("DIFF case %d: %s, plan %s (%d buffers), %d host frames, %d reference frames" % (i, sc, kind, len(chunks), len(h), len(r)))
    print("%d cases, %d reference frames, %d differ" % (a.n, frames, bad))


if __name__ == "__main__":
    main()
