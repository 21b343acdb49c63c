"""What the adaptive signal tests compare against (nfcb200_adaptive_radio / nfcb200_adaptive_logic, include/nfcb200.h): the
reference's lab::SignalResamplingTask and lab::TraceStorageTask from oracle/_ref/libnfcref_adaptive.so (oracle/ref_adaptive.cpp)
or their recording, and the host build of the device steps (tests/native/adaptive_host.cpp).

Nothing here is imported by the product package.  tests/golden/make_adaptive_golden.py writes the recording.
"""
import ctypes as C
import functools
import hashlib
import io
import lzma
import os
import subprocess
import tarfile

import numpy as np

import nfcutil as U

SO = os.path.join(U.ORACLE, "_ref", "libnfcref_adaptive.so")
RECORDED = os.path.join(U.GOLDEN, "ref_adaptive.npz.xz")
BUFFER = 65536
RATE = 10_000_000
IQ_F32, MAG_F32, MAG_S16, IQ_S16 = 1, 2, 3, 4
LOGIC_F32, LOGIC_S16, LOGIC_U8 = 5, 6, 7

# radio cases: name -> (magnitude source, buffer).  Fixture captures as the reference replays them; synthetic IQ whose last
# buffer is shorter than 65 536 samples (but holds the 26 the initial sum reads), as float and on the int16 grid
FIXTURES = ["test_NFC-A_106kbps_001", "test_NFC-B_106kbps_001", "test_NFC-F_212kbps_001", "test_NFC-V_26kbps_002", "test_POLL_AB_001"]
SYNTH = {"nfca106": ("nfca106", 3 * BUFFER + 1000), "nfcb106": ("nfcb106", 2 * BUFFER + 3000)}
RADIO_CASES = [("fixture", f, BUFFER) for f in FIXTURES] + [(kind, s, BUFFER) for s in SYNTH for kind in ("iq_f32", "iq_s16")] + \
              [("iq_f32", "nfca106", 4096)]
# logic cases: ISO 7816 captures as float, int16 and 8-bit values at 4 and 8 channels
LOGIC_CASES = [(sc, fmt, ch) for sc in ("t0_direct", "t1_crc") for fmt in (LOGIC_F32, LOGIC_S16, LOGIC_U8) for ch in (4, 8)]


def case_id(case):
    return "/".join(str(c) for c in case)


def to_s16(x):
    return np.clip(np.rint(np.asarray(x, dtype=np.float64) * 32768.0), -32768, 32767).astype(np.int16)


def magnitude(iq):
    """sqrtf(I * I + Q * Q) in float32, one IEEE operation at a time (RadioDeviceTask / K1)"""
    iq = np.asarray(iq, dtype=np.float32)
    return np.sqrt(iq[..., 0] * iq[..., 0] + iq[..., 1] * iq[..., 1])


@functools.lru_cache(maxsize=None)
def synth_iq(name):
    from nfc_laboratory_b200 import synth
    config, n = SYNTH[name]
    return np.ascontiguousarray(synth.synth_batch(config, 1, n, seed=23, fs=RATE, iq=True)[0].numpy(), dtype=np.float32)


@functools.lru_cache(maxsize=None)
def radio_input(case):
    """(device input, its sigtype, the magnitude the reference is fed, buffer) of a radio case"""
    kind, src, buf = case
    if kind == "fixture":
        mag = np.ascontiguousarray(U.fixture_wav(src)[0], dtype=np.float32)
        return mag, MAG_F32, mag, buf
    iq = synth_iq(src)
    if kind == "iq_s16":
        s = to_s16(iq)
        return s, IQ_S16, magnitude(s.astype(np.float32) / np.float32(32768.0)), buf
    return iq, IQ_F32, magnitude(iq), buf


@functools.lru_cache(maxsize=None)
def logic_input(case):
    """(device input, sigtype, the float values the reference is fed [n, ch]) of a logic case.  Channels 4-7 of the
    8-channel captures are IO delayed by 3, 40, 300 and 5000 samples."""
    from nfc_laboratory_b200 import synth
    sc, fmt, ch = case
    x = synth.iso7816_capture(sc, RATE, seed=1).astype(np.float32)
    if ch == 8:
        extra = [np.concatenate([np.zeros(d, np.float32), x[:-d, 0]]) for d in (3, 40, 300, 5000)]
        x = np.concatenate([x, np.stack(extra, axis=1)], axis=1)
    x = np.ascontiguousarray(x)
    if fmt == LOGIC_S16:
        s = to_s16(x * np.float32(0.75))
        return s, fmt, s.astype(np.float32) / np.float32(32768.0)
    if fmt == LOGIC_U8:
        u = np.clip(np.rint(x * 200.0), 0, 255).astype(np.uint8)
        return u, fmt, u.astype(np.float32) / np.float32(255.0)
    return x, fmt, x


def key(values, buf, offset=0):
    h = hashlib.sha256(np.ascontiguousarray(values, dtype=np.float32).tobytes())
    h.update(b"%d/%d/%d" % (values.shape[-1] if values.ndim == 2 else 0, buf, offset))
    return h.hexdigest()[:24]


POINTS = [("channel", "<u4"), ("sample", "<u8"), ("value", "<f4")]


def _points(val, sample, channel, n):
    p = np.empty(n, dtype=POINTS)
    p["value"], p["sample"], p["channel"] = val[:n], sample[:n], channel[:n]
    return p


@functools.lru_cache(maxsize=None)
def oracle_lib():
    if not os.path.exists(SO):
        return None
    lib = C.CDLL(SO)
    lib.nfcref_adaptive.restype = C.c_long
    lib.nfcref_adaptive.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_long, C.c_char_p, C.c_int, C.c_double, C.c_double]
    return lib


def oracle(values, buf, offset=0, trz=None, time_range=None):
    """the live oracle: points (channel, sample, value) in the order the resampler publishes them (buffer, channel);
    values [n] magnitudes or [n, ch] logic"""
    x = np.ascontiguousarray(values, dtype=np.float32)
    ch = x.shape[1] if x.ndim == 2 else 0
    cap = 2 * x.size + 4 * (x.shape[0] // buf + 1)
    val, sample, channel = np.zeros(cap, np.float32), np.zeros(cap, np.uint64), np.zeros(cap, np.uint32)
    t0, t1 = time_range or (0.0, 0.0)
    n = oracle_lib().nfcref_adaptive(x.ctypes.data, ch, x.shape[0], RATE, buf, offset, val.ctypes.data, sample.ctypes.data, channel.ctypes.data,
                                     cap, trz.encode() if trz else None, 1 if time_range else 0, t0, t1)
    assert 0 <= n <= cap
    return _points(val, sample, channel, n)


def by_channel(points):
    """the resampler's order (buffer, channel) -> the ABI's (channel, buffer): a stable sort by channel"""
    return points[np.argsort(points["channel"], kind="stable")]


@functools.lru_cache(maxsize=None)
def recording():
    if not os.path.exists(RECORDED):
        return {}
    with lzma.open(RECORDED, "rb") as f:
        z = np.load(io.BytesIO(f.read()))
        return {k: z[k] for k in z.files}


def reference(values, buf, offset=0):
    """the reference's points in the ABI's order: the live oracle where oracle/_ref/ has it, else the recording"""
    if oracle_lib() is not None:
        return by_channel(oracle(values, buf, offset))
    rec = recording().get(key(values, buf, offset))
    assert rec is not None, "no recorded adaptive signal for this input: rebuild oracle/_ref/ and run tests/golden/make_adaptive_golden.py"
    return rec


def trz_members(path):
    """{name: bytes} of the members of a .trz"""
    with tarfile.open(path, "r:gz") as tar:
        return {m.name: tar.extractfile(m).read() for m in tar.getmembers()}


# the .trz cases: (radio case, logic case, time range or None for a Write command without one)
TRZ_RADIO = ("fixture", "test_NFC-A_106kbps_001", BUFFER)
TRZ_LOGIC = ("t0_direct", LOGIC_F32, 4)
TRZ_RANGES = {"whole": (0.0, 1.0), "window": (0.002, 0.0095), "none": None}


def fits_reference(values, buf):
    """every buffer's points fit the reference's output buffer (elements + elements / 255 points, :170, :242) and every
    radio buffer holds the 25 samples its initial sum reads: the reference is defined on this input"""
    x = np.asarray(values)
    n = x.shape[0]
    if x.ndim == 1 and n % buf and n % buf < 25:
        return False
    pts = host(values, buf)
    for ch in np.unique(pts["channel"]):
        per = np.bincount(pts["sample"][pts["channel"] == ch].astype(np.int64) // buf, minlength=(n + buf - 1) // buf)
        size = np.minimum(buf, n - np.arange(len(per)) * buf)
        if np.any(per > size + size // 255):
            return False
    return True


def record(tmpdir, path=RECORDED):
    """write the live oracle's points of every case, keyed by input, and the .apcm members of the .trz cases"""
    arrays = {}
    for case in RADIO_CASES:
        _, _, mag, buf = radio_input(case)
        assert fits_reference(mag, buf), case
        arrays[key(mag, buf)] = by_channel(oracle(mag, buf))
    for case in LOGIC_CASES:
        _, _, x = logic_input(case)
        assert fits_reference(x, BUFFER), case
        arrays[key(x, BUFFER)] = by_channel(oracle(x, BUFFER))
    for name, rng in TRZ_RANGES.items():
        for kind, values in (("radio", radio_input(TRZ_RADIO)[2]), ("logic", logic_input(TRZ_LOGIC)[2])):
            p = os.path.join(tmpdir, "%s-%s.trz" % (kind, name))
            oracle(values, BUFFER, trz=p, time_range=rng)
            for member, data in trz_members(p).items():
                arrays["trz/%s/%s/%s" % (kind, name, member)] = np.frombuffer(data, dtype=np.uint8)
    buf = io.BytesIO()
    np.savez(buf, **arrays)
    with lzma.open(path, "wb", preset=9 | lzma.PRESET_EXTREME) as f:
        f.write(buf.getvalue())
    return len(arrays)


def recorded_members(kind, name):
    """{member: bytes} the reference's TraceStorageTask wrote for a .trz case"""
    prefix = "trz/%s/%s/" % (kind, name)
    return {k[len(prefix):]: v.tobytes() for k, v in recording().items() if k.startswith(prefix)}


@functools.lru_cache(maxsize=None)
def host_lib():
    """the host build of the device steps, compiled like tests/native/spectrum_host.cpp"""
    src = os.path.join(U.ROOT, "tests", "native", "adaptive_host.cpp")
    hdr = os.path.join(U.ROOT, "nfc_laboratory_b200", "csrc", "adaptive.cuh")
    so = os.path.join(U.ROOT, "build", "libadaptivehost.so")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        os.makedirs(os.path.dirname(so), exist_ok=True)
        tmp = so + ".tmp%d" % os.getpid()
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-msse2", "-mfpmath=sse", "-ffp-contract=off", "-shared", "-fPIC", src, "-o", tmp])
        os.replace(tmp, so)
    lib = C.CDLL(so)
    lib.adaptive_radio_host.restype = C.c_uint64
    lib.adaptive_radio_host.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64]
    lib.adaptive_logic_host.restype = C.c_uint64
    lib.adaptive_logic_host.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
    return lib


def host(values, buf, offset=0):
    """host build: points (channel, sample, value) of one stream in the ABI's order; values [n] magnitudes or [n, ch]"""
    x = np.ascontiguousarray(values, dtype=np.float32)
    cap = 2 * x.size + 4 * (x.shape[0] // buf + 1)
    val, sample, channel = np.zeros(cap, np.float32), np.zeros(cap, np.uint64), np.zeros(cap, np.uint32)
    if x.ndim == 1:
        n = host_lib().adaptive_radio_host(x.ctypes.data, x.shape[0], buf, offset, val.ctypes.data, sample.ctypes.data, cap)
    else:
        n = host_lib().adaptive_logic_host(x.ctypes.data, x.shape[1], x.shape[0], buf, offset, val.ctypes.data, sample.ctypes.data,
                                           channel.ctypes.data, cap)
    assert n <= cap
    return _points(val, sample, channel, n)


def same(a, b):
    """point lists equal field by field, values as bits"""
    return len(a) == len(b) and np.array_equal(a["channel"], b["channel"]) and np.array_equal(a["sample"], b["sample"]) and \
        np.array_equal(np.asarray(a["value"], np.float32).view(np.uint32), np.asarray(b["value"], np.float32).view(np.uint32))


def alternating(n=20000, seed=3):
    """a magnitude that deviates at every sample, the first included: every sample is kept and the first one twice, one
    point more per buffer than the reference's output buffer (elements + elements / 255 points) holds below 255 samples"""
    x = np.full(n, 0.5, dtype=np.float32)
    x[1::2] += np.float32(0.05)
    x[::7] -= np.float32(0.02) * np.random.default_rng(seed).random(len(x[::7])).astype(np.float32)
    return x


def reference_capacity(n, buf):
    """points the reference's output buffers hold for a stream of n samples (SignalResamplingTask.cpp:170)"""
    return sum(min(buf, n - b0) + min(buf, n - b0) // 255 for b0 in range(0, n, buf))
