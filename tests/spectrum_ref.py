"""What the spectrum tests compare against (nfcb200_spectrum, include/nfcb200.h): the reference's FFT spectrum frames from
oracle/_ref/libnfcref_fft.so (oracle/ref_fft.cpp over the reference's own mufft) or their recording, a float64 numpy
model of the same frame, and the host build of the device transform (tests/native/spectrum_host.cpp).

Nothing here is imported by the product package.  tests/golden/make_spectrum_golden.py writes the recording.
"""
import ctypes as C
import functools
import hashlib
import io
import lzma
import os
import struct
import subprocess

import numpy as np

import nfcutil as U

FFT_SO = os.path.join(U.ORACLE, "_ref", "libnfcref_fft.so")
RECORDED = os.path.join(U.GOLDEN, "ref_spectrum.npz.xz")
BINS = 1024
# max_k |a_k - b_k| <= TOL * max_k b_k per frame: two float32 FFTs of 1024 points with different summation orders
TOL = 2e-5

# the recorded input set: name -> (synth config or "carrier", sample rate, hop, frames, int16 grid).  nfcb106, the 4 MS/s
# workload and the carrier use hops that are not multiples of 4, so frames start inside a run of the selection pattern.
# Inputs on the int16 grid are multiples of 1 / 32768, so the same recording checks int16 ingest (s / 32768.f is exact)
CASES = {
    "nfca106": ("nfca106", 10_000_000, 16384, 20, False),
    "nfcb106": ("nfcb106", 10_000_000, 12345, 24, False),
    "mixed": ("mixed", 10_000_000, 16384, 20, False),
    "nfca106_4M": ("nfca106", 4_000_000, 5001, 30, True),
    "carrier": ("carrier", 10_000_000, 7777, 20, True),
}
S16_CASES = [name for name in CASES if CASES[name][4]]


def decimation(rate):
    return rate // 625000


def frames_of(n_samples, rate, hop):
    span = BINS * decimation(rate)
    return 0 if n_samples < span else (n_samples - span) // hop + 1


@functools.lru_cache(maxsize=None)
def case_input(name):
    """(float32 IQ [n, 2], sample rate, hop) of one recorded case"""
    config, rate, hop, frames, s16 = CASES[name]
    n = BINS * decimation(rate) + (frames - 1) * hop
    if config == "carrier":
        # a carrier 150 kHz above the tuned frequency, with a little noise
        t = np.arange(n, dtype=np.float64)
        noise = 1e-3 * np.random.default_rng(5).standard_normal((n, 2))
        iq = (0.3 * np.stack([np.cos(2 * np.pi * 150e3 / rate * t), np.sin(2 * np.pi * 150e3 / rate * t)], axis=1) + noise).astype(np.float32)
    else:
        from nfc_laboratory_b200 import synth
        iq = synth.synth_batch(config, 1, n, seed=11, fs=rate, iq=True)[0].numpy()
    iq = np.ascontiguousarray(iq, dtype=np.float32)
    if s16:
        iq = to_s16(iq).astype(np.float32) / np.float32(32768.0)
    iq.setflags(write=False)
    return iq, rate, hop


def to_s16(iq):
    return np.clip(np.rint(np.asarray(iq, dtype=np.float64) * 32768.0), -32768, 32767).astype(np.int16)


def key(iq, rate, hop):
    h = hashlib.sha256(np.ascontiguousarray(iq, dtype=np.float32).tobytes())
    h.update(struct.pack("<QIQ", iq.shape[0], rate, hop))
    return h.hexdigest()


@functools.lru_cache(maxsize=None)
def oracle_lib():
    if not os.path.exists(FFT_SO):
        return None
    lib = C.CDLL(FFT_SO)
    lib.nfcref_fft.restype = C.c_long
    lib.nfcref_fft.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint64, C.c_void_p, C.c_long]
    return lib


def oracle(iq, rate, hop):
    """the live oracle: float32 [frames, 1024]"""
    iq = np.ascontiguousarray(iq, dtype=np.float32)
    nf = frames_of(iq.shape[0], rate, hop)
    out = np.zeros((nf, BINS), dtype=np.float32)
    n = oracle_lib().nfcref_fft(iq.ctypes.data, iq.shape[0], rate, hop, out.ctypes.data, nf)
    assert n == nf
    return out


@functools.lru_cache(maxsize=None)
def recording():
    if not os.path.exists(RECORDED):
        return {}
    with lzma.open(RECORDED, "rb") as f:
        z = np.load(io.BytesIO(f.read()))
        return {k: z[k] for k in z.files}


def reference(iq, rate, hop):
    """the reference's frames: the live oracle where oracle/_ref/ has it, else the recording of this exact input"""
    if oracle_lib() is not None:
        return oracle(iq, rate, hop)
    rec = recording().get(key(iq, rate, hop))
    assert rec is not None, "no recorded spectrum for this input: rebuild oracle/_ref/ and run tests/golden/make_spectrum_golden.py"
    return rec


def record(path=RECORDED):
    """write the live oracle's frames of every case, keyed by input and parameters"""
    arrays = {}
    for name in CASES:
        iq, rate, hop = case_input(name)
        arrays[key(iq, rate, hop)] = oracle(iq, rate, hop)
    buf = io.BytesIO()
    np.savez(buf, **arrays)
    with lzma.open(path, "wb", preset=9 | lzma.PRESET_EXTREME) as f:
        f.write(buf.getvalue())


def window():
    """the reference's window (FourierProcessTask.cpp:126-127) in float32: sin(float(pi n / 1024))^2"""
    n = np.arange(BINS)
    s = np.sin(np.float32(np.pi * n / BINS)).astype(np.float64)
    return (s * s).astype(np.float32)


def selection(rate):
    """sample offset of every window position from the frame's first sample (the reference's SSE2 loop, :250-263)"""
    k = np.arange(BINS)
    return 4 * decimation(rate) * (k // 4) + k % 4


def model(iq, rate, hop, streams_axis=False):
    """float64 model of the frames: the selection, the float32 window product, a float64 FFT, magnitudes, the shift.
    iq [n, 2] -> [frames, 1024]; with streams_axis, [streams, n, 2] -> [streams, frames, 1024]"""
    iq = np.asarray(iq, dtype=np.float32)
    if not streams_axis:
        return model(iq[None], rate, hop, True)[0]
    nf = frames_of(iq.shape[1], rate, hop)
    idx = (np.arange(nf) * hop)[:, None] + selection(rate)[None, :]
    w = window()
    x = iq[:, idx]                                   # [streams, frames, 1024, 2]
    z = (x[..., 0] * w).astype(np.float64) + 1j * (x[..., 1] * w).astype(np.float64)
    m = np.abs(np.fft.fft(z, axis=-1))
    return np.concatenate([m[..., BINS // 2:], m[..., :BINS // 2]], axis=-1)


def worst(a, b):
    """max over frames of max_k |a_k - b_k| / max_k b_k"""
    a = np.asarray(a, dtype=np.float64).reshape(-1, BINS)
    b = np.asarray(b, dtype=np.float64).reshape(-1, BINS)
    return float(np.max(np.max(np.abs(a - b), axis=1) / np.max(b, axis=1))) if a.size else 0.0


@functools.lru_cache(maxsize=None)
def host_lib():
    """the host build of the device transform, compiled like tests/native/host_sim.cpp"""
    src = os.path.join(U.ROOT, "tests", "native", "spectrum_host.cpp")
    hdr = os.path.join(U.ROOT, "nfc_laboratory_b200", "csrc", "nfc_spectrum.cuh")
    so = os.path.join(U.ROOT, "build", "libspectrumhost.so")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        os.makedirs(os.path.dirname(so), exist_ok=True)
        tmp = so + ".tmp%d" % os.getpid()
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-msse2", "-mfpmath=sse", "-ffp-contract=off", "-shared", "-fPIC", src, "-o", tmp])
        os.replace(tmp, so)
    lib = C.CDLL(so)
    lib.spectrum_host.restype = C.c_long
    lib.spectrum_host.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint64, C.c_void_p]
    lib.spectrum_host_window.argtypes = [C.c_void_p]
    return lib


def host(samples, sigtype, rate, hop):
    """host build: IQ [streams, n, 2] (float32 for sigtype 1, int16 for 4) -> float32 [streams, frames, 1024]"""
    a = np.ascontiguousarray(samples, dtype=np.float32 if sigtype == 1 else np.int16)
    nf = frames_of(a.shape[1], rate, hop)
    out = np.zeros((a.shape[0], nf, BINS), dtype=np.float32)
    assert host_lib().spectrum_host(a.ctypes.data, sigtype, a.shape[0], a.shape[1], rate, hop, out.ctypes.data) == nf
    return out
