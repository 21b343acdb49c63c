#!/usr/bin/env python3
"""Time nfcb200_spectrum (NfcDecoder.spectrum) on the benchmark's default batch: 512 streams x 1e7 float2 IQ at 10 MS/s,
generated on the device like bench.py, input and output resident.

For each hop it prints one JSON line:
  ms_call         median host time of a call, which ends in a device synchronise (the call returns complete output)
  ms_kernel       the spectrum kernels' device time in one call, from torch.profiler in a run of its own
  frames_per_s    frames / ms_call
  bytes           algorithmic traffic: 256 gathered 32-byte sectors + 4 096 output bytes per frame
  tb_s, of_peak   bytes / ms_kernel, and that over the H100 SXM data sheet's 3.35 TB/s of HBM3
plus the card's name, power limit and max SM clock, read in the same run (nvidia-smi query).

Usage: python tools/spectrum_bench.py [--streams 512] [--samples 10000000] [--hops span,4096] [--calls 7] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

RATE = 10_000_000
PEAK_TBS = 3.35


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        row = subprocess.check_output(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], text=True).splitlines()[0]
        return dict(zip(q.split(","), [v.strip() for v in row.split(",")]))
    except (OSError, subprocess.CalledProcessError, IndexError):
        return {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=512)
    ap.add_argument("--samples", type=int, default=10_000_000)
    ap.add_argument("--workload", default="nfca106")
    ap.add_argument("--seed", type=int, default=2024)
    ap.add_argument("--hops", default="span,4096")
    ap.add_argument("--calls", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", help="directory for the JSON lines (spectrum_bench.jsonl)")
    args = ap.parse_args()

    import torch
    import nfc_laboratory_b200 as N
    from nfc_laboratory_b200 import synth

    if not torch.cuda.is_available():
        sys.exit("spectrum_bench: no CUDA device")
    S, n = args.streams, args.samples
    iq = torch.empty((S, n, 2), dtype=torch.float32, device="cuda")
    synth.synth_batch(args.workload, S, n, seed=args.seed, device="cuda", out=iq)
    torch.cuda.synchronize()
    dec = N.NfcDecoder()
    info = card()
    lines = []

    for h in args.hops.split(","):
        span = 1024 * N.spectrum_shape(n, RATE)[1]
        hop = span if h == "span" else int(h)
        nf, _ = N.spectrum_shape(n, RATE, hop)
        frames = S * nf
        out = torch.empty((S, nf, 1024), dtype=torch.float32, device="cuda")

        def call():
            dec.spectrum_ptr(iq.data_ptr(), True, N.SIG_IQ_F32, S, n, RATE, hop, out.data_ptr(), True, out.numel())

        for _ in range(args.warmup):
            call()
        times = []
        for _ in range(args.calls):
            t0 = time.perf_counter()
            call()
            times.append((time.perf_counter() - t0) * 1e3)

        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        kern = [e for e in prof.events() if "spectrum_kernel" in e.name]
        ms_kernel = sum(e.device_time for e in kern) / 1e3

        nbytes = frames * (256 * 32 + 1024 * 4)
        ms = statistics.median(times)
        rec = {"hop": hop, "streams": S, "samples": n, "frames": frames, "calls": args.calls, "ms_call": round(ms, 3),
               "ms_call_min": round(min(times), 3), "ms_call_max": round(max(times), 3), "ms_kernel": round(ms_kernel, 3),
               "kernel_launches": len(kern), "frames_per_s": round(frames / ms * 1e3), "bytes": nbytes,
               "tb_s": round(nbytes / ms_kernel / 1e9, 3) if ms_kernel else None,
               "of_peak": round(nbytes / ms_kernel / 1e9 / PEAK_TBS, 3) if ms_kernel else None, "gpu": info}
        print(json.dumps(rec), flush=True)
        lines.append(rec)
        del out

    dec.close()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "spectrum_bench.jsonl"), "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
