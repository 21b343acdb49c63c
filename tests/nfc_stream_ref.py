"""Checkers of the streaming NFC decode (nfcb200_stream_push, lab::NfcDecoder::nextFrames fed buffer by buffer) and of the
decoder settings: one live reference decoder driven call by call (oracle/_ref/libnfcref.so: nfcref_create / _set_* /
_push / _flush / _destroy), its recorded output (tests/golden/ref_nfc_stream.json.xz) where that library was not built,
the device's frames read field by field from nfcb200_frame, and the buffer plans and settings the tests push.

A record is every field of a frame: (tech, type, flags, phase, rate, sample_start, sample_end, payload hex, sample_rate,
time_start, time_end, date_time), the three times as float.hex() so that equality is bit equality."""
import contextlib
import ctypes as C
import functools
import hashlib
import json
import lzma
import os
import zlib

import numpy as np

import nfcutil as U
from nfc_laboratory_b200.binding import CFrame

GOLDEN = os.path.join(U.GOLDEN, "ref_nfc_stream.json.xz")
RATE = 10_000_000
STREAM_TIME = 1_700_000_000
TINY_WINDOW = 150_000   # samples pushed 1-63 at a time around the first poll / listen exchange in the "tiny" plan


def record(tech, ftype, flags, phase, rate, start, end, data, sample_rate, t0, t1, dt):
    return (int(tech), int(ftype), int(flags), int(phase), int(rate), int(start), int(end), bytes(data).hex(), int(sample_rate),
            float(t0).hex(), float(t1).hex(), float(dt).hex())


def records(buf, n):
    """records of frames 0..n of an nfcb200_frame or nfcref_frame array"""
    return [record(f.tech_type, f.frame_type, f.frame_flags, f.frame_phase, f.frame_rate, f.sample_start, f.sample_end, f.data[:f.length],
                   f.sample_rate, f.time_start, f.time_end, f.date_time) for f in buf[:n]]


def keys(recs):
    """the 8-tuples of nfcutil.ref_decode / Frame.key() of a list of records"""
    return [tuple(r[:7]) + (bytes.fromhex(r[7]),) for r in recs]


# --- settings ------------------------------------------------------------------------------------------------------------
DEFAULT = dict(enabled=0xF, corr=(0.75, 0.5, 0.5, 0.5), mod_min=(0.9, 0.1, 0.1, 0.9), mod_max=(1.0, 0.9, 0.9, 1.0), power=0.01, stream_time=0)


def settings(**kw):
    """DEFAULT with some values changed; corr / mod_min / mod_max take {tech index: value}"""
    s = dict(DEFAULT)
    for k, v in kw.items():
        if isinstance(v, dict):
            t = list(s[k])
            for i, x in v.items():
                t[i] = x
            v = tuple(t)
        s[k] = v
    return s


def settings_id(s):
    parts = []
    for k in ("enabled", "corr", "mod_min", "mod_max", "power", "stream_time"):
        if s[k] != DEFAULT[k]:
            parts.append("%s=%s" % (k, ",".join("%g" % x for x in s[k]) if isinstance(s[k], tuple) else "%g" % s[k]))
    return ";".join(parts) or "default"


A106, B106, F212, V26 = "test_NFC-A_106kbps_001", "test_NFC-B_106kbps_001", "test_NFC-F_212kbps_001", "test_NFC-V_26kbps_001"
POLLS = ["test_POLL_ABF_001", "test_POLL_AB_001"]
MASK_CAPTURES = POLLS + [A106, B106, F212, V26]
MASKS = [0x0, 0x1, 0x2, 0x4, 0x8, 0x3, 0xF]
# (settings, captures) of the settings matrix; every one set before the first buffer
MATRIX = ([(settings(enabled=m), MASK_CAPTURES) for m in MASKS] + [
    (settings(corr={0: 0.2}), ["test_NFC-A_424kbps_001", "test_NFC-A_424kbps_002", "test_NFC-A_106kbps_212kbps_001", A106, "test_POLL_ABF_001"]),
    (settings(corr={0: 0.95}), ["test_NFC-A_424kbps_001", "test_NFC-A_106kbps_212kbps_001", A106, "test_POLL_ABF_001"]),
    (settings(corr={2: 0.2}), ["test_NFC-F_212kbps_002", "test_NFC-F_212kbps_004", "test_POLL_ABF_001"]),
    (settings(corr={3: 0.2}), ["test_NFC-V_26kbps_001", "test_NFC-V_26kbps_002"]),
    (settings(mod_min={1: 0.05}, mod_max={1: 0.95}), ["test_NFC-B_106kbps_001", "test_NFC-B_106kbps_002"] + POLLS),
    (settings(mod_min={1: 0.3}, mod_max={1: 0.6}), ["test_NFC-B_106kbps_001", "test_NFC-B_106kbps_002"] + POLLS),
    (settings(power=0.003), [A106, B106, "test_POLL_AB_001", V26]),
    (settings(power=0.05), [A106, B106, "test_POLL_AB_001", V26]),
    (settings(stream_time=STREAM_TIME), [A106, "test_NFC-F_212kbps_003"]),
])


def matrix_cases():
    return [(s, name) for s, names in MATRIX for name in names]


# --- the live reference ----------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def ref_lib():
    """libnfcref.so with the live-decoder entry points declared, or None where oracle/_ref/ was not built"""
    lib = U.ref_lib()
    if lib is None:
        return None
    lib.nfcref_create.restype = C.c_void_p
    lib.nfcref_destroy.argtypes = [C.c_void_p]
    lib.nfcref_set_enabled.argtypes = [C.c_void_p, C.c_uint]
    lib.nfcref_set_thresholds.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_float, C.c_float]
    lib.nfcref_set_power_threshold.argtypes = [C.c_void_p, C.c_float]
    lib.nfcref_set_stream_time.argtypes = [C.c_void_p, C.c_long]
    lib.nfcref_push.restype = C.c_long
    lib.nfcref_push.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.POINTER(U.RefFrame), C.c_long]
    lib.nfcref_flush.restype = C.c_long
    lib.nfcref_flush.argtypes = [C.c_void_p, C.POINTER(U.RefFrame), C.c_long]
    return lib


def ref_run(steps, s=DEFAULT):
    """the reference's records of one lab::NfcDecoder with settings `s` set before the first buffer, run through `steps`:
    ("push", magnitude, rate, chunk) -- nextFrames per chunk-sample buffer --, or ("flush",) -- nextFrames({})"""
    lib = ref_lib()
    cap = 1 << 14
    d = lib.nfcref_create()
    try:
        lib.nfcref_set_enabled(d, s["enabled"])
        for t in range(4):
            lib.nfcref_set_thresholds(d, t, s["corr"][t], s["mod_min"][t], s["mod_max"][t])
        lib.nfcref_set_power_threshold(d, s["power"])
        lib.nfcref_set_stream_time(d, s["stream_time"])
        out = []
        for st in steps:
            buf = (U.RefFrame * cap)()
            if st[0] == "push":
                x = np.ascontiguousarray(st[1], dtype=np.float32)
                n = lib.nfcref_push(d, x.ctypes.data, x.size, st[2], st[3], buf, cap)
            else:
                n = lib.nfcref_flush(d, buf, cap)
            assert 0 <= n <= cap
            out += records(buf, n)
        return out
    finally:
        lib.nfcref_destroy(d)


def steps_key(steps, s):
    h = hashlib.sha256(json.dumps(s, sort_keys=True).encode())
    for st in steps:
        h.update(st[0].encode())
        if st[0] == "push":
            h.update(np.ascontiguousarray(st[1], dtype=np.float32).tobytes())
            h.update(b"%d/%d" % (st[2], st[3]))
    return h.hexdigest()[:24]


@functools.lru_cache(maxsize=1)
def golden():
    if not os.path.exists(GOLDEN):
        return {}
    with lzma.open(GOLDEN, "rt") as f:
        return json.load(f)


def expected(name, steps, s=DEFAULT):
    """the reference's records of `steps` under settings `s`: live where oracle/_ref/libnfcref.so exists, else the recorded
    entry `name`, which must have been recorded from the same input"""
    if ref_lib() is not None:
        return ref_run(steps, s)
    g = golden().get(name)
    assert g is not None, "no recorded reference output %r: regenerate tests/golden/ref_nfc_stream.json.xz with the reference" % name
    assert g["key"] == steps_key(steps, s), "the input of %r differs from the recorded one" % name
    return [tuple(r) for r in g["frames"]]


# --- inputs --------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=4)
def capture(name):
    return U.fixture_wav(name)[0]


def whole_steps(x, rate=RATE):
    """the reference's own harness: 65 536-sample buffers, then nextFrames({})"""
    return [("push", x, rate, 65536), ("flush",)]


def capture_expected(name, s=DEFAULT):
    """records of a fixture capture pushed whole and flushed: the answer for every buffer plan (the reference's frames do
    not depend on where its buffers end)"""
    return expected("%s/%s" % (name, settings_id(s)), whole_steps(capture(name)), s)


def iq_of(mag, seed=7):
    """float2 IQ of a magnitude with a slowly drifting phase, as test_iq_input_equals_reference builds it"""
    rng = np.random.default_rng(seed)
    phi = rng.uniform(0, 2 * np.pi) + np.cumsum(rng.normal(0, 1e-4, mag.size))
    return np.stack([mag * np.cos(phi), mag * np.sin(phi)], axis=-1).astype(np.float32)


def iq16_of(mag, seed=11):
    """int16 IQ as test_int16_iq_ingest_equals_reference builds it"""
    rng = np.random.default_rng(seed)
    phi = rng.uniform(0, 2 * np.pi) + np.cumsum(rng.normal(0, 1e-4, mag.size))
    return np.stack([np.round(mag * np.cos(phi) * 32767.0), np.round(mag * np.sin(phi) * 32767.0)], axis=-1).astype(np.int16)


def ref_iq_magnitude(iq):
    """the reference's magnitude of float2 IQ, or of int16 IQ read as s / 32768.f"""
    if iq.dtype == np.int16:
        iq = iq.astype(np.float32) / np.float32(32768.0)
    return U.ref_iq_magnitude(iq)


IQ_CAPTURES = ["test_NFC-A_106kbps_002", "test_NFC-A_424kbps_001", "test_NFC-B_106kbps_001", "test_POLL_AB_001"]
IQ16_CAPTURES = ["test_NFC-A_106kbps_001", "test_NFC-B_106kbps_001", "test_NFC-F_212kbps_002"]
SYNTH = ["nfca106", "nfcb106", "nfca424", "mixed"]
SYNTH_STREAMS, SYNTH_SAMPLES, SYNTH_SEED = 2, 1_500_000, 77


@functools.lru_cache(maxsize=1)
def synth_iq(config):
    from nfc_laboratory_b200 import synth as Y
    return Y.synth_batch(config, SYNTH_STREAMS, SYNTH_SAMPLES, seed=SYNTH_SEED).numpy()


# a capture at another supported rate (16-bit representable magnitude, as tools/cpu_fuzz_rates.py builds them)
OTHER_RATE, OTHER_SAMPLES, OTHER_SEED = 5_000_000, 1_200_000, 1300003


@functools.lru_cache(maxsize=1)
def other_rate_capture():
    from nfc_laboratory_b200 import synth as Y
    iq = Y.synth_batch("nfca106", 1, OTHER_SAMPLES, seed=OTHER_SEED, fs=OTHER_RATE)[0].numpy()
    mag = np.sqrt(iq[:, 0] ** 2 + iq[:, 1] ** 2).astype(np.float32)
    return np.round(np.clip(mag, 0, 0.9999) * 32768.0).astype(np.int16).astype(np.float32) / np.float32(32768.0)


def rate_change_steps(order):
    """one 10 MS/s fixture and the OTHER_RATE capture pushed in one stream ("up": the fixture first), then the flush"""
    a = ("push", capture(A106), RATE, 65536)
    b = ("push", other_rate_capture(), OTHER_RATE, 65536)
    return ([a, b] if order == "up" else [b, a]) + [("flush",)]


def _rng(*parts):
    return np.random.default_rng(zlib.crc32("/".join(map(str, parts)).encode()))


def _random_chunks(rng, n, lo, hi):
    out, at = [], 0
    while at < n:
        out.append(int(min(rng.integers(lo, hi + 1), n - at)))
        at += out[-1]
    return out


def _fixed(n, size):
    return [size] * (n // size) + ([n % size] if n % size else [])


def _cuts(n, cuts):
    b = sorted({c for c in cuts if 0 < c < n})
    return [e - a for a, e in zip([0] + b, b + [n])]


def plans(name, n, frames):
    """plan name -> buffer lengths of one capture of n samples; `frames`: the reference's records of it"""
    out = {"whole": [n]}
    for size in (65536, 4096, 256, 255, 257):
        out["p%d" % size] = _fixed(n, size)
    out["random"] = _random_chunks(_rng(name, "random"), n, 1_000, 300_000)
    exch = [f[5] for f in frames if f[1] in (0x102, 0x103)]
    a = max(0, min(exch[0] if exch else 0, n - TINY_WINDOW) - 2_000)
    e = min(n, a + TINY_WINDOW)
    out["tiny"] = _fixed(a, 65536) + _random_chunks(_rng(name, "tiny"), e - a, 1, 63) + _fixed(n - e, 65536)
    edges = [f[k] + d for f in frames[:-1] for k in (5, 6) for d in (-1, 0, 1)]
    out["edges"] = _cuts(n, edges)
    assert all(sum(p) == n and min(p) > 0 for p in out.values())
    return out


# --- the host model with settings ------------------------------------------------------------------------------------------
@contextlib.contextmanager
def host_settings(s):
    """tests/native/host_sim.cpp decodes with the thresholds and power level of `s` inside the block"""
    lib = U.sim_lib()
    lib.hostsim_set_settings.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_float]
    arr = [np.ascontiguousarray(s[k], dtype=np.float32) for k in ("corr", "mod_min", "mod_max")]
    lib.hostsim_set_settings(*(a.ctypes.data for a in arr), s["power"])
    try:
        yield
    finally:
        lib.hostsim_set_settings(None, None, None, 0.0)


# --- the device ----------------------------------------------------------------------------------------------------------
def configure(dec, s):
    """nfcb200_configure of a binding.NfcDecoder with settings `s`"""
    cfg = dec._cfg
    cfg.enabled = s["enabled"]
    cfg.power_level_threshold = s["power"]
    for t in range(4):
        cfg.correlation_threshold[t] = s["corr"][t]
        cfg.modulation_min[t] = s["mod_min"][t]
        cfg.modulation_max[t] = s["mod_max"][t]
    cfg.stream_time = s["stream_time"]
    dec._apply()


class Stream:
    """nfcb200_stream_push / _pending / _reset of one handle, called directly; every call returns records"""

    def __init__(self, dec, cap=4096):
        self.lib, self.h, self.cap = dec._lib, dec._h, cap
        self.buf = (CFrame * cap)()

    def raw_push(self, x, sigtype, rate, cap):
        """(rc, records delivered, *n_out) of one push of x (numpy, the sigtype's dtype) or of the flush (x None)"""
        n = C.c_uint64(0)
        if x is None:
            rc = self.lib.nfcb200_stream_push(self.h, None, sigtype, 0, rate, self.buf, cap, C.byref(n))
        else:
            a = np.ascontiguousarray(x)
            count = a.shape[0]
            rc = self.lib.nfcb200_stream_push(self.h, a.ctypes.data, sigtype, count, rate, self.buf, cap, C.byref(n))
        return rc, records(self.buf, min(n.value, cap)), n.value

    def pending(self, cap):
        """(rc, records, n_out, n_left) of nfcb200_stream_pending"""
        n, left = C.c_uint64(0), C.c_uint64(0)
        rc = self.lib.nfcb200_stream_pending(self.h, self.buf if cap else None, cap, C.byref(n), C.byref(left))
        return rc, records(self.buf, n.value), n.value, left.value

    def push(self, x, sigtype, rate):
        """records of one push (x None: the flush), pending ones drained"""
        rc, out, _ = self.raw_push(x, sigtype, rate, self.cap)
        if rc == -4:
            while True:
                rc2, more, _, left = self.pending(self.cap)
                assert rc2 == 0
                out += more
                if not left:
                    break
        else:
            assert rc == 0, (rc, self.lib.nfcb200_last_error())
        return out

    def plan(self, x, chunks, sigtype, rate, flush=True):
        out, at = [], 0
        for c in chunks:
            out += self.push(x[at:at + c], sigtype, rate)
            at += c
        assert at == len(x)
        if flush:
            out += self.push(None, sigtype, rate)
        return out

    def reset(self):
        assert self.lib.nfcb200_stream_reset(self.h) == 0


def batch_records(dec, x, sigtype, rate):
    """records of decode_batch of one stream (raw frames, every field)"""
    a = np.ascontiguousarray(x)
    buf, n = dec.decode_batch_ptr(a.ctypes.data, False, sigtype, 1, a.shape[0], rate, raw=True)
    return records(buf, n)


# --- what the golden records -----------------------------------------------------------------------------------------------
def flush_sequences():
    """name -> steps of the flush cases: a fresh decoder flushed, two flushes in a row, push / flush / push / flush"""
    x = capture(A106)
    h = len(x) // 2
    return {"flush/fresh": [("flush",)], "flush/twice": whole_steps(x) + [("flush",)],
            "flush/again": [("push", x[:h], RATE, 65536), ("flush",), ("push", x[h:], RATE, 65536), ("flush",)]}


def golden_entries():
    """(name, steps, settings) of every reference run the GPU tests compare with"""
    out = [("%s/default" % name, whole_steps(capture(name)), DEFAULT) for name in U.fixture_names()]
    out += [("%s/%s" % (name, settings_id(s)), whole_steps(capture(name)), s) for s, name in matrix_cases() if s != DEFAULT]
    out += [("%s/iq" % name, whole_steps(ref_iq_magnitude(iq_of(capture(name)))), DEFAULT) for name in IQ_CAPTURES]
    out += [("%s/iq16" % name, whole_steps(ref_iq_magnitude(iq16_of(capture(name)))), DEFAULT) for name in IQ16_CAPTURES]
    out += [("synth/%s/%d" % (c, k), whole_steps(ref_iq_magnitude(synth_iq(c)[k])), DEFAULT) for c in SYNTH for k in range(SYNTH_STREAMS)]
    out += [(name, steps, DEFAULT) for name, steps in flush_sequences().items()]
    out += [("rate/%s" % o, rate_change_steps(o), DEFAULT) for o in ("up", "down")]
    out += [("rate/%s/%s" % (o, part), steps, DEFAULT) for o in ("up", "down") for part, steps in restart_steps(o).items()]
    return out


def restart_steps(order):
    """the two halves of rate_change_steps(order) on decoders of their own: what the device's restart at a sample-rate
    change gives (DESIGN.md section 2)"""
    steps = rate_change_steps(order)
    return {"first": steps[:1], "second": steps[1:]}
