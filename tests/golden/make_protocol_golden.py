"""Write tests/golden/ref_protocol.json.xz: the edge delays of every window-edge context of tests/protocol_sessions.py,
measured on the reference by bisection (guard: the first delay at which the response decodes; wait: the last one), then
for every input of golden_inputs() -- the edge sweeps, the chunk-alignment shifts, the late responses, the encrypted
sessions, the error cases, each of those padded as its batch family holds it, and the long captures -- a hash of the input and every field of the reference's frames (one
lab::NfcDecoder fed 65 536-sample buffers, then nextFrames({})).  Needs oracle/_ref/libnfcref.so (oracle/Makefile
builds it from the reference sources); run from the repository root:

    python3 tests/golden/make_protocol_golden.py
"""
import json
import lzma
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import protocol_sessions as P  # noqa: E402
import nfc_stream_ref as T  # noqa: E402


def decodes(ctx, d):
    return P.responds(T.ref_run(P.steps(P.edge_capture(ctx, d))), ctx)


def bisect(ctx, good, bad):
    """the delay next to `good` on its side of the edge between a decoding delay `good` and a failing delay `bad`"""
    while abs(bad - good) > 1:
        mid = (good + bad) // 2
        if decodes(ctx, mid):
            good = mid
        else:
            bad = mid
    return good


def edge_delays(ctx):
    c = P.contexts()[ctx]
    # a delay that decodes: the nominal one, or the first of a downward scan (a window shorter than the nominal delay)
    good = c.nominal
    while not decodes(ctx, good):
        good -= 100
        assert good > 0, ctx
    # None: the response decodes at the earliest delay the context can build (NFC-V), no guard edge within reach
    guard = None if decodes(ctx, c.min_delay) else bisect(ctx, good, c.min_delay)
    wait = bisect(ctx, good, int(1.2 * c.fwt) + 2000)
    return {"guard": guard, "wait": wait}


def main():
    if T.ref_lib() is None:
        sys.exit("oracle/_ref/libnfcref.so is missing: run make -C oracle where the reference sources are")
    edges = {}
    for ctx in P.CONTEXTS:
        edges[ctx] = edge_delays(ctx)
        print("%-14s guard %7s  wait %8d  (nominal %d, window %d)" % (ctx, edges[ctx]["guard"], edges[ctx]["wait"], P.contexts()[ctx].nominal,
                                                                       P.contexts()[ctx].fwt))
    # the case list depends on the edges
    P.golden.cache_clear()
    P._builders.cache_clear()
    P.golden = lambda: {"edges": edges}
    out = {"edges": edges, "runs": {}}
    for name, build in P.golden_inputs().items():
        x = build()
        out["runs"][name] = P.golden_entry(name, x)
    print("%d runs" % len(out["runs"]))
    with lzma.open(P.GOLDEN, "wt", preset=9) as f:
        json.dump(out, f, sort_keys=True, separators=(",", ":"))


if __name__ == "__main__":
    main()
