"""Write tests/golden/ref_iso_protocol.json.xz: the edge delays of every context of tests/iso_sessions.py at every rate,
measured on the reference by bisection (guard: the first delay at which the swept character decodes; wait: the last
one, T=1 only), then for every case a hash of the capture and every field of the reference's frames
(oracle/_ref/libnfcref_iso.so), the frames of the capture padded as its batch family holds it, and for the edge sweeps and
the clock-batch cases the chunked reference's frames (libnfcref_iso_stream.so) for each chunk plan.  Every case is
decoded a second time in a fresh process; a case whose answers differ is dropped and named.  Run from the repository
root:

    python3 tests/golden/make_iso_protocol_golden.py
"""
import json
import lzma
import multiprocessing as mp
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import iso_ref as R  # noqa: E402
import iso_sessions as P  # noqa: E402
import iso_stream_ref as T  # noqa: E402


def ref(x, rate):
    return R.ref(x, rate, stream_time=P.STREAM_TIME)


def decodes(ctx, rate, d):
    return P.responds(ref(P.contexts()[ctx].capture(rate, d), rate), ctx)


def bisect(ctx, rate, good, bad):
    while abs(bad - good) > 1:
        mid = (good + bad) // 2
        if decodes(ctx, rate, mid):
            good = mid
        else:
            bad = mid
    return good


def edge_delays(ctx, rate):
    c = P.contexts()[ctx]
    etu = c.etu(rate)
    good = int(round(12 * etu))
    assert decodes(ctx, rate, good), (ctx, rate)
    early = int(round((9.6 if c.t1 else 10.6) * etu))
    guard = None if decodes(ctx, rate, early) else bisect(ctx, rate, good, early)
    wait = None
    if c.t1:
        cwi = int(ctx[6:]) if ctx.startswith("t1_cwi") else 5
        late = int(round((11 + 2 ** cwi + 3) * etu))
        assert not decodes(ctx, rate, late), (ctx, rate)
        wait = bisect(ctx, rate, good, late)
    return {"guard": guard, "wait": wait}


def entry(name, x, n_pad, stream):
    rate = P.rate_of(name)
    e = {"key": P.key(x, rate), "frames": ref(x, rate)}
    if n_pad > len(x):
        e["padded"] = ref(P.padded(x, n_pad), rate)
    if stream:
        plans = P.chunk_plans(name, x)
        e["plans"] = {k: T.chunked(T.ref_lib(), x, c, [rate] * len(c), stream_time=P.STREAM_TIME) for k, c in plans.items() if k != "whole"}
    return e


def wants_stream(name):
    return name.startswith("edge/") or name.startswith("clk/batch")


def family_entries(args):
    fam, names, edges = args
    keep = P.golden
    P.golden = lambda: {"edges": edges}   # the chunk plans of the edge sweeps cut at these edges
    try:
        b = P.builders(edges)
        xs = {n: b[n]() for n in names}
        n_pad = max(len(x) for x in xs.values())
        return {n: entry(n, xs[n], n_pad, wants_stream(n)) for n in names}
    finally:
        P.golden = keep


def main():
    if R.ref_lib() is None or T.ref_lib() is None:
        sys.exit("oracle/_ref/libnfcref_iso*.so are missing: run make -C oracle -f iso.mk / iso_stream.mk where the reference sources are")
    edges = {}
    for ctx, c in P.contexts().items():
        for rate in c.rates:
            k = "%s/r%d" % (ctx, rate // 1_000_000)
            edges[k] = edge_delays(ctx, rate)
            print("%-22s guard %7s  wait %8s  (ETU %.1f)" % (k, edges[k]["guard"], edges[k]["wait"], c.etu(rate)), flush=True)
    P.golden = lambda: {"edges": edges}
    P.names.cache_clear()
    fams = {}
    for n in sorted(P.builders(edges)):
        fams.setdefault(P.family(n), []).append(n)
    jobs = [(f, ns, edges) for f, ns in sorted(fams.items())]
    # one long run in this process, and each family again in a fresh process
    long_run = {}
    for j in jobs:
        long_run.update(family_entries(j))
    fresh = {}
    with mp.get_context("spawn").Pool(8, maxtasksperchild=1) as pool:
        for r in pool.imap_unordered(family_entries, jobs):
            fresh.update(r)
    dropped = sorted(n for n in long_run if json.dumps(long_run[n]) != json.dumps(fresh[n]))
    for n in dropped:
        print("dropped (the reference answers differently in a fresh process):", n)
        del long_run[n]
    out = {"edges": edges, "runs": long_run, "dropped": dropped}
    print("%d runs, %d dropped" % (len(long_run), len(dropped)))
    with lzma.open(P.GOLDEN, "wt", preset=9) as f:
        json.dump(out, f, sort_keys=True, separators=(",", ":"))


if __name__ == "__main__":
    main()
