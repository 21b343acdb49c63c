"""Benchmark of the streaming ISO 7816 decode (nfcb200_iso7816_stream_push) on one GPU: one live logic capture pushed
buffer by buffer from host memory, as lab::IsoDecoder is fed by LogicDecoderTask.

The capture is a seeded synthetic T=1 session (nfc_laboratory_b200.synth.iso7816_capture) repeated back to back into
24 x 2^20 samples (about 1 s at 25 MS/s), and the stream runs through it again and again.  Reports, as one JSON line:
  - push latency: host clock around each push (the call returns with its frames on the host), median and 90th
    percentile over --pushes pushes after --warmup, for pushes of 2^14, 2^16, 2^18 and 2^20 samples, float and int16;
  - sustained rate: samples per second over --seconds of capture pushed back to back, against the real-time rate;
  - what one push runs: kernels launched, copies and memsets, and stream synchronisations, from torch.profiler in a
    run of its own;
  - the card's name, power limit and SM clocks, read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import nfc_laboratory_b200 as N  # noqa: E402
from nfc_laboratory_b200 import synth as S  # noqa: E402

SIZES = (1 << 14, 1 << 16, 1 << 18, 1 << 20)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=60).stdout
        return out.strip().splitlines()[0]
    except Exception as e:  # the numbers are still reported, without the card line
        return "unavailable: %s" % e


def push_all(d, x, sigtype, rate, size, first, count):
    """pushes count buffers of `size` samples from x (cyclic) starting at buffer `first`; returns (seconds per push, frames)"""
    per = len(x) // size
    times, frames = [], 0
    for k in range(first, first + count):
        j = k % per
        t0 = time.perf_counter()
        frames += len(d.iso7816_push(x[j * size:(j + 1) * size], sigtype, rate, raw=True))
        times.append(time.perf_counter() - t0)
    return times, frames


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rate", type=int, default=25_000_000)
    ap.add_argument("--pushes", type=int, default=400)
    ap.add_argument("--warmup", type=int, default=40)
    ap.add_argument("--seconds", type=float, default=10.0)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"

    one = S.iso7816_capture("t1_lrc", a.rate, seed=11)
    n = 24 << 20
    x32 = np.ascontiguousarray(np.resize(one, (n, 4)), dtype=np.float32)
    x16 = np.ascontiguousarray(np.round(x32 * 32767), dtype=np.int16)
    inputs = {"f32": (x32, N.SIG_LOGIC_F32), "s16": (x16, N.SIG_LOGIC_S16)}

    d = N.NfcDecoder(device=0)
    latency, sustained = {}, {}
    for name, (x, sig) in inputs.items():
        for size in SIZES:
            d.iso7816_reset()
            push_all(d, x, sig, a.rate, size, 0, a.warmup)
            t, _ = push_all(d, x, sig, a.rate, size, a.warmup, a.pushes)
            latency["%s/%d" % (name, size)] = {"median_us": float(np.median(t)) * 1e6, "p90_us": float(np.percentile(t, 90)) * 1e6}
            # sustained: --seconds of capture back to back from a fresh stream, frames drained as they come
            d.iso7816_reset()
            count = int(a.seconds * a.rate) // size
            t0 = time.perf_counter()
            _, frames = push_all(d, x, sig, a.rate, size, 0, count)
            frames += len(d.iso7816_flush(raw=True))
            wall = time.perf_counter() - t0
            sps = count * size / wall
            sustained["%s/%d" % (name, size)] = {"samples": count * size, "seconds": wall, "samples_per_s": sps, "x_real_time": sps / a.rate,
                                                 "frames": frames}

    # what one push runs (2^16 float samples, in the middle of a stream)
    from torch.profiler import ProfilerActivity, profile
    d.iso7816_reset()
    push_all(d, x32, N.SIG_LOGIC_F32, a.rate, 1 << 16, 0, 8)
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        push_all(d, x32, N.SIG_LOGIC_F32, a.rate, 1 << 16, 8, 1)
        torch.cuda.synchronize()
    kernels, runtime = [], {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and "kernel" in e.name:
            kernels.append(e.name)
        elif e.name.startswith("cuda") and e.name != "cudaDeviceSynchronize":
            runtime[e.name] = runtime.get(e.name, 0) + 1
    d.close()

    print(json.dumps({
        "card": card(), "rate": a.rate, "capture_samples": n,
        "push_latency": latency, "sustained": sustained,
        "one_push": {"kernels": sorted(kernels), "runtime_calls": runtime},
    }))


if __name__ == "__main__":
    main()
