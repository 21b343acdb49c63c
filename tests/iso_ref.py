"""ISO 7816 checkers: the host build of the device decoder (tests/native/iso_host.cpp), the live oracle
(oracle/_ref/libnfcref_iso.so, where it was built) and the recorded oracle output (tests/golden/ref_iso7816.json.xz)."""
import ctypes as C
import functools
import hashlib
import json
import lzma
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from nfc_laboratory_b200 import synth as S  # noqa: E402
from nfc_laboratory_b200.binding import CFrame  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_iso7816.json.xz")
RATES = (10_000_000, 25_000_000, 50_000_000)
STREAM_TIME = 1000
CASES = [(sc, rate) for sc in S.ISO_SCENARIOS for rate in RATES]
# CLK channels with more than two levels: a falling edge (clk - last < 0) can then come on consecutive samples
CLOCKS = ("noise", "staircase", "ramp")
CLOCK_CASES = [("t0_direct", 10_000_000, kind) for kind in CLOCKS] + [("t1_lrc", 25_000_000, "noise")]


def capture(scenario, rate, seed=1):
    return S.iso7816_capture(scenario, rate, seed=seed)


def multilevel_clock(x, kind, seed=1):
    """x with its CLK channel replaced: Gaussian noise (sigma 0.2) on the clock, a 1 / 0.5 / 0 staircase (falls on 2
    samples in 3), or a falling ramp over 1000 samples (falls on every sample but one in 1000)"""
    y = x.copy()
    n = len(y)
    if kind == "noise":
        y[:, 1] += np.random.default_rng(seed).normal(0.0, 0.2, n).astype(np.float32)
    elif kind == "staircase":
        y[:, 1] = 1.0 - 0.5 * (np.arange(n) % 3)
    else:
        y[:, 1] = 1.0 - (np.arange(n) % 1000) / 1000.0
    return np.clip(y, -1.0, 32767 / 32768).astype(np.float32)


def clock_capture(scenario, rate, kind):
    return multilevel_clock(capture(scenario, rate), kind)


def key(x, rate, stream_time=STREAM_TIME):
    """hash of one input: samples, rate and stream time"""
    h = hashlib.sha256(np.ascontiguousarray(x, dtype=np.float32).tobytes())
    h.update(b"%d/%d" % (rate, stream_time))
    return h.hexdigest()[:24]


def rows(buf, n):
    """every field of the frames, the payload as hex"""
    out = []
    for f in buf[:n]:
        out.append([f.stream, f.tech_type, f.frame_type, f.frame_flags, f.frame_phase, f.frame_rate, f.length, f.sample_start, f.sample_end,
                    f.sample_rate, f.time_start, f.time_end, f.date_time, bytes(f.data[:min(f.length, 512)]).hex()])
    return out


@functools.lru_cache(maxsize=None)
def host_lib():
    """the host build of iso_core.h, compiled like tests/native/host_sim.cpp"""
    src = os.path.join(ROOT, "tests", "native", "iso_host.cpp")
    hdr = os.path.join(ROOT, "nfc_laboratory_b200", "csrc", "iso_core.h")
    so = os.path.join(ROOT, "build", "libisohost.so")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        os.makedirs(os.path.dirname(so), exist_ok=True)
        tmp = so + ".tmp%d" % os.getpid()
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-msse2", "-mfpmath=sse", "-ffp-contract=off", "-shared", "-fPIC", src, "-o", tmp])
        os.replace(tmp, so)
    lib = C.CDLL(so)
    lib.iso_host_decode.restype = C.c_long
    lib.iso_host_decode.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint32, C.c_void_p, C.c_long]
    return lib


def s16(x):
    """float samples in [-1, 1) as the int16 samples that read back as them (s / 32768.f) where they are multiples of 2^-15"""
    return np.round(np.asarray(x, dtype=np.float64) * 32768).clip(-32768, 32767).astype(np.int16)


def host(x, rate, sigtype=5, stream_time=STREAM_TIME):
    """host build: x [n, 4] or [streams, n, 4] (float32 for sigtype 5, int16 for 6)"""
    a = np.ascontiguousarray(x, dtype=np.float32 if sigtype == 5 else np.int16)
    a = a[None] if a.ndim == 2 else a
    cap = 4096
    while True:
        buf = (CFrame * cap)()
        n = host_lib().iso_host_decode(a.ctypes.data, sigtype, a.shape[0], a.shape[1], rate, stream_time, buf, cap)
        if n <= cap:
            return rows(buf, n)
        cap = n


def ref_lib():
    so = os.path.join(ROOT, "oracle", "_ref", "libnfcref_iso.so")
    if not os.path.exists(so):
        return None
    lib = C.CDLL(so)
    lib.ref_iso_decode.restype = C.c_long
    lib.ref_iso_decode.argtypes = [C.c_void_p, C.c_ulong, C.c_uint, C.c_uint, C.c_void_p, C.c_long]
    return lib


def ref(x, rate, stream_time=STREAM_TIME):
    """the live oracle on one capture [n, 4] float32"""
    lib = ref_lib()
    a = np.ascontiguousarray(x, dtype=np.float32)
    cap = 4096
    while True:
        buf = (CFrame * cap)()
        n = lib.ref_iso_decode(a.ctypes.data, a.shape[0], rate, stream_time, buf, cap)
        if n <= cap:
            return rows(buf, n)
        cap = n


@functools.lru_cache(maxsize=None)
def golden():
    with lzma.open(GOLDEN, "rt") as f:
        return json.load(f)


def expected(x, rate):
    """the recorded oracle frames of one capture"""
    return golden()[key(x, rate)]
