"""Benchmark of the ISO 7816 decoder (nfcb200_iso7816_decode_batch, nfcb200_iso7816_decode_batch_ch) on one GPU.

Default batch: 128 streams of 2.5e7 LOGIC_F32 samples (1 s at 25 MS/s each, 51.2 GB), assembled on the device from a
seeded synthetic session (nfc_laboratory_b200.synth.iso7816_capture, T=1, repeated back to back: every repetition is a
full power-up, ATR, PPS and block exchange).  --sigtype f32 / s16 / u8 (or the number) picks the sample format,
--channels 4-8 the stride (the channels past VCC are seeded noise); u8 samples are the capture clipped to [0, 1] as
RecordDevice writes it.  Reports, as one JSON line:
  - the whole call's time and rate (host clock around a synchronised call, median of --reps after a warm-up), with the
    frames converted to Python tuples and without (raw ctypes records: the C entry point alone),
  - kernel times of the edge pass and the walk from torch.profiler, in a run of their own,
  - the edge pass's input bytes over its kernel time, as a share of the H100 SXM's 3.35 TB/s,
  - with --pinned, the C entry point again from a pinned host copy of the batch (the input is copied in ~1 GB groups),
  - the card's name, power limit and SM clocks, read in the same run.
Writes the profiler trace under --out when given."""
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

HBM_BYTES_PER_S = 3.35e12
SIGTYPES = {"f32": N.SIG_LOGIC_F32, "s16": N.SIG_LOGIC_S16, "u8": N.SIG_LOGIC_U8}


def sigtype(v):
    return SIGTYPES[v] if v in SIGTYPES else int(v)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=60).stdout
        return out.strip().splitlines()[0]
    except Exception as e:  # the numbers are still reported, without the card line
        return "unavailable: %s" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=128)
    ap.add_argument("--samples", type=int, default=25_000_000)
    ap.add_argument("--rate", type=int, default=25_000_000)
    ap.add_argument("--sigtype", type=sigtype, default=N.SIG_LOGIC_F32)
    ap.add_argument("--channels", type=int, default=4)
    ap.add_argument("--pinned", action="store_true")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    dev = torch.device("cuda:0")
    one = S.iso7816_capture("t1_lrc", a.rate, seed=11)
    if a.channels > 4:
        extra = np.random.default_rng(a.channels).random((len(one), a.channels - 4), dtype=np.float32)
        one = np.concatenate([one, extra], axis=1)
    if a.sigtype == N.SIG_LOGIC_S16:
        one = (one * 32767).astype(np.int16)
    elif a.sigtype == N.SIG_LOGIC_U8:
        one = N.logic_wav.logic_bytes(np.clip(one, 0, 1))
    base = torch.from_numpy(one).to(dev)
    reps = -(-a.samples // base.shape[0])
    stream = base.repeat(reps, 1)[:a.samples]
    batch = torch.empty((a.streams, a.samples, a.channels), dtype=base.dtype, device=dev)
    for s in range(a.streams):
        batch[s].copy_(stream)
    del stream
    torch.cuda.synchronize()
    in_bytes = batch.numel() * batch.element_size()

    d = N.NfcDecoder(device=0)
    frames = d.iso7816_decode(batch, a.sigtype, a.rate)  # warm-up: allocations, module load
    per_stream = len(d.iso7816_decode(batch[:1], a.sigtype, a.rate))
    times = []
    for _ in range(a.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        got = d.iso7816_decode(batch, a.sigtype, a.rate)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
        assert got == frames
    call = float(np.median(times))
    # the entry point alone: frames stay ctypes records (no conversion to Python tuples)
    raw = []
    for _ in range(a.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        d.iso7816_decode(batch, a.sigtype, a.rate, raw=True)
        torch.cuda.synchronize()
        raw.append(time.perf_counter() - t0)
    entry = float(np.median(raw))
    pinned = None
    if a.pinned:
        host = torch.empty(batch.shape, dtype=batch.dtype, pin_memory=True)
        host.copy_(batch)
        d.iso7816_decode(host, a.sigtype, a.rate, raw=True)
        ph = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            d.iso7816_decode(host, a.sigtype, a.rate, raw=True)
            ph.append(time.perf_counter() - t0)
        pinned = float(np.median(ph))
        del host

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        d.iso7816_decode(batch, a.sigtype, a.rate)
        torch.cuda.synchronize()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        prof.export_chrome_trace(os.path.join(a.out, "iso_bench.pt.trace.json"))
    kt = {"edges": 0.0, "walk": 0.0}
    for e in prof.events():
        name = e.name
        dt = e.device_time_total
        if "iso_edges" in name:
            kt["edges"] += dt / 1e3
        elif "iso_walk_kernel" in name:
            kt["walk"] += dt / 1e3
    d.close()

    res = {
        "card": card(),
        "streams": a.streams, "samples_per_stream": a.samples, "sigtype": a.sigtype, "channels": a.channels, "input_bytes": in_bytes,
        "frames": len(frames), "frames_per_stream": per_stream,
        "call_ms_median": call * 1e3, "call_ms_all": [t * 1e3 for t in times],
        "call_gsps": a.streams * a.samples / call / 1e9,
        "entry_ms_median": entry * 1e3, "entry_gsps": a.streams * a.samples / entry / 1e9,
        "pinned_entry_ms_median": pinned * 1e3 if pinned else None,
        "pinned_entry_gsps": a.streams * a.samples / pinned / 1e9 if pinned else None,
        "edges_kernel_ms": kt["edges"], "walk_kernel_ms": kt["walk"],
        "edges_bytes_per_s": in_bytes / (kt["edges"] / 1e3) if kt["edges"] else None,
        "edges_share_of_3.35TBps": in_bytes / (kt["edges"] / 1e3) / HBM_BYTES_PER_S if kt["edges"] else None,
    }
    print(json.dumps(res))


if __name__ == "__main__":
    main()
