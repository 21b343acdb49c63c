#!/usr/bin/env python3
"""Measure nfcb200_adaptive_radio / nfcb200_adaptive_logic on the GPU (NfcDecoder.adaptive_radio / adaptive_logic).

Workloads, device-resident input:
  radio  512 x 10^7 float2 IQ at buffer 65 536 (the bench.py workload's shape)
  logic  128 x 2.5 x 10^7 4-channel float32 logic (the ISO 7816 bench workload's shape)

Reports per workload: call time (host clock around the whole call, which ends in a device synchronise), kernel time (CUDA
activity of the adaptive kernels from torch.profiler, in a run of its own), points emitted, and the algorithmic bytes
(the input read once plus the 24-byte points written) over kernel time as a share of the H100 SXM's 3.35 TB/s, with the
card's name and power limit read in the same run.  Prints one JSON line, and with --out also writes it to that file.

Usage: python tools/adaptive_bench.py [--reps 3] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import nfc_laboratory_b200 as N  # noqa: E402

HBM_TBS = 3.35


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def radio_input(streams, n):
    # a carrier with ASK bursts and a little noise: quiet stretches keep one sample in 255, bursts keep more
    g = torch.Generator(device="cuda").manual_seed(1)
    t = torch.arange(n, device="cuda", dtype=torch.float32)
    env = 0.5 + 0.1 * ((t // 4096) % 8 == 0).float() * ((t // 50) % 2)
    iq = torch.empty((streams, n, 2), device="cuda", dtype=torch.float32)
    for s in range(streams):
        noise = 1e-3 * torch.randn((n, 2), device="cuda", generator=g)
        iq[s, :, 0] = env + noise[:, 0]
        iq[s, :, 1] = noise[:, 1]
    return iq


def logic_input(streams, n):
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.zeros((streams, n, 4), device="cuda", dtype=torch.float32)
    t = torch.arange(n, device="cuda")
    x[:, :, 1] = ((t // 3) % 2).float()                       # CLK
    x[:, :, 3] = 1.0                                          # VCC
    x[:, :, 2] = (t > 1000).float()                           # RST
    for s in range(streams):
        x[s, :, 0] = (torch.rand(n // 372 + 1, device="cuda", generator=g) < 0.5).float().repeat_interleave(372)[:n]  # IO at 372 clocks / bit
    return x


def measure(name, call, in_bytes, reps):
    call()  # warm-up: modules, buffers
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        pts = call()
        times.append(time.perf_counter() - t0)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    ks = [e for e in prof.key_averages() if "adaptive" in e.key]
    kern = sum(e.device_time_total for e in ks) / 1e3  # ms
    launches = sum(e.count for e in ks)
    per_kernel = {}
    for e in ks:  # kernel names end in <..., true> for the emit pass, <..., false> for the count pass
        k = "emit" if "true>" in e.key else "count"
        per_kernel[k] = round(per_kernel.get(k, 0.0) + e.device_time_total / 1e3, 2)
    alg = in_bytes + len(pts) * N.SIGNAL_POINT_DTYPE.itemsize
    return {"workload": name, "call_ms": [round(1e3 * t, 2) for t in times], "kernel_ms": round(kern, 2), "kernel_launches": launches, "kernel_ms_by_pass": per_kernel,
            "points": int(len(pts)), "alg_bytes": int(alg), "alg_TBps": round(alg / (kern * 1e-3) / 1e12, 3),
            "share_of_3.35TBps": round(alg / (kern * 1e-3) / 1e12 / HBM_TBS, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--radio", default="512x10000000")
    ap.add_argument("--logic", default="128x25000000")
    ap.add_argument("--out", help="file for the JSON line")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: the adaptive signal is measured on the GPU only")
    d = N.NfcDecoder(device=0)
    res = {"card": card(), "results": []}
    rs, rn = (int(v) for v in a.radio.split("x"))
    iq = radio_input(rs, rn)
    res["results"].append(measure("radio %dx%d IQ_F32 buffer 65536" % (rs, rn), lambda: d.adaptive_radio(iq, N.SIG_IQ_F32, 10_000_000),
                                  iq.numel() * 4, a.reps))
    del iq
    torch.cuda.empty_cache()
    ls, ln = (int(v) for v in a.logic.split("x"))
    lg = logic_input(ls, ln)
    res["results"].append(measure("logic %dx%d x4 LOGIC_F32 buffer 65536" % (ls, ln), lambda: d.adaptive_logic(lg, N.SIG_LOGIC_F32, 10_000_000),
                                  lg.numel() * 4, a.reps))
    d.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
