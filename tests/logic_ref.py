"""Checkers of the reference's 8-bit logic WAVs: the ISO 7816 captures of iso_ref at 4, 5 and 8 channels (the channels
past VCC carry seeded noise and pulses), written by the reference's hw::RecordDevice and replayed into its
lab::IsoDecoder as SignalStorageTask::readLogic streams them (oracle/_ref/libnfcref_logic_replay.so, where it was built),
the same driver over the drop-in shim (libnfcref_logic_b200.so), and the recorded output
(tests/golden/ref_iso7816_u8.json.xz)."""
import ctypes as C
import functools
import hashlib
import json
import lzma
import os
import zlib

import numpy as np

import iso_ref as R
import iso_stream_ref as T
from nfc_laboratory_b200 import logic_wav as W
from nfc_laboratory_b200.binding import CFrame

GOLDEN = os.path.join(R.ROOT, "tests", "golden", "ref_iso7816_u8.json.xz")
CHANNELS = (4, 5, 8)
CASES = [(case, ch) for case in T.CASES for ch in CHANNELS]
EPOCH = 1_700_000_000
KEYS = (101, 102, 103, 104, 105, 106, 107, 108)
PUSH = 65_536  # samples per buffer of SignalStorageTask::readLogic


def case_id(case):
    return "%s-ch%d" % (T.case_id(case[0]), case[1])


@functools.lru_cache(maxsize=4)
def samples(case):
    """float32 [n, channels] in [0, 1]: the capture clipped to [0, 1] (RecordDevice converts values outside it with an
    undefined cast), then channels of uniform noise with runs at 1 and 0"""
    iso, ch = case
    x = np.clip(T.case_capture(iso), 0.0, 1.0).astype(np.float32)
    n = len(x)
    rng = np.random.default_rng(zlib.crc32(case_id(case).encode()))
    extra = rng.random((n, ch - 4), dtype=np.float32)
    for c in range(ch - 4):
        for start in rng.integers(0, n, 64):
            extra[start:start + int(rng.integers(1, 2000)), c] = float(rng.integers(0, 2))
    return np.concatenate([x, extra], axis=1)


def u8(case):
    """the 8-bit samples RecordDevice stores for samples(case)"""
    return W.logic_bytes(samples(case))


def as_float(b):
    """8-bit samples as RecordDevice reads them: b / 255.f"""
    return np.asarray(b, dtype=np.float32) / np.float32(255)


def write(path, case):
    iso, ch = case
    W.write_logic_wav(path, samples(case), iso[1], EPOCH, KEYS[:ch])


def sha256(path):
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def _lib(name):
    so = os.path.join(R.ROOT, "oracle", "_ref", name)
    if not os.path.exists(so):
        return None
    lib = C.CDLL(so)
    lib.ref_logic_write.restype = C.c_int
    lib.ref_logic_write.argtypes = [C.c_char_p, C.c_void_p, C.c_ulong, C.c_uint, C.c_uint, C.c_uint, C.c_void_p, C.c_uint]
    lib.ref_logic_read.restype = C.c_long
    lib.ref_logic_read.argtypes = [C.c_char_p, C.POINTER(C.c_uint), C.POINTER(C.c_uint), C.POINTER(C.c_uint), C.c_void_p, C.c_void_p, C.c_ulong]
    lib.ref_logic_replay.restype = C.c_long
    lib.ref_logic_replay.argtypes = [C.c_char_p, C.c_uint, C.c_void_p, C.c_long]
    return lib


@functools.lru_cache(maxsize=None)
def ref_lib():
    """the reference's RecordDevice and lab::IsoDecoder"""
    return _lib("libnfcref_logic_replay.so")


@functools.lru_cache(maxsize=None)
def shim_lib():
    """the same driver over the drop-in lab::IsoDecoder (needs a GPU)"""
    return _lib("libnfcref_logic_b200.so")


def ref_write(lib, path, case):
    iso, ch = case
    x = np.ascontiguousarray(samples(case))
    keys = np.asarray(KEYS[:ch], dtype=np.int32)
    assert lib.ref_logic_write(path.encode(), x.ctypes.data, len(x), ch, iso[1], EPOCH, keys.ctypes.data, ch) == 0


def ref_read(lib, path, cap):
    """(rate, channels, epoch, keys, float samples [n, channels]) as RecordDevice reads the file"""
    rate, ch, epoch = C.c_uint(), C.c_uint(), C.c_uint()
    keys = np.zeros(8, dtype=np.int32)
    out = np.zeros(cap * 8, dtype=np.float32)
    n = lib.ref_logic_read(path.encode(), C.byref(rate), C.byref(ch), C.byref(epoch), keys.ctypes.data, out.ctypes.data, cap)
    assert n >= 0
    return rate.value, ch.value, epoch.value, tuple(int(k) for k in keys), out[:min(n, cap) * ch.value].reshape(-1, ch.value)


def replay(lib, path, stream_time=EPOCH):
    cap = 4096
    while True:
        buf = (CFrame * cap)()
        n = lib.ref_logic_replay(path.encode(), stream_time, buf, cap)
        assert n >= 0
        if n <= cap:
            return R.rows(buf, n)
        cap = n


def chunks(n):
    return [PUSH] * (n // PUSH) + ([n % PUSH] if n % PUSH else [])


@functools.lru_cache(maxsize=None)
def golden():
    with lzma.open(GOLDEN, "rt") as f:
        return json.load(f)


def expected(case):
    return golden()[case_id(case)]["frames"]
