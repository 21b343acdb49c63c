"""Checkers of the streaming ISO 7816 decode: seeded chunk plans over the captures of iso_ref, the host build of the
stream push (tests/native/iso_stream_host.cpp), the live chunked oracle and the drop-in shim behind the same driver
(oracle/_ref/libnfcref_iso_stream.so and libnfcref_iso_b200.so, where they were built), and the recorded oracle output
(tests/golden/ref_iso7816_stream.json.xz)."""
import ctypes as C
import functools
import hashlib
import json
import lzma
import os
import subprocess
import zlib

import numpy as np

import iso_ref as R
from nfc_laboratory_b200.binding import CFrame

GOLDEN = os.path.join(R.ROOT, "tests", "golden", "ref_iso7816_stream.json.xz")

# (scenario, rate, multi-level clock kind or None): the 15 captures of iso_ref.CASES and the 4 of CLOCK_CASES
CASES = [(sc, rate, None) for sc, rate in R.CASES] + list(R.CLOCK_CASES)
TINY_WINDOW = 65_536  # samples pushed 1-63 at a time in the "tiny" plan


def case_id(case):
    sc, rate, kind = case
    return "%s-%dM" % (sc, rate // 1_000_000) + ("-" + kind if kind else "")


def case_capture(case):
    sc, rate, kind = case
    return R.clock_capture(sc, rate, kind) if kind else R.capture(sc, rate)


def _rng(case, plan):
    return np.random.default_rng(zlib.crc32(("%s/%s" % (case_id(case), plan)).encode()))


def _random_chunks(rng, n, lo, hi):
    out = []
    while sum(out) < n:
        out.append(int(min(rng.integers(lo, hi + 1), n - sum(out))))
    return out


def rst_low_windows(x):
    """[begin, end) of every run of samples with RST at or below 0"""
    low = np.asarray(x)[:, 2] <= 0
    edges = np.flatnonzero(np.diff(np.concatenate(([0], low.view(np.int8), [0]))))
    return list(zip(edges[::2].tolist(), edges[1::2].tolist()))


@functools.lru_cache(maxsize=2)
def plans(case):
    """name -> (samples [n, 4] float32, chunk lengths, chunk rates): one stream fed buffer by buffer"""
    x = case_capture(case)
    n, rate = len(x), case[1]
    out = {"whole": (x, [n], [rate])}
    rng = _rng(case, "tiny")
    a = n // 2 - TINY_WINDOW // 2
    tiny = _random_chunks(rng, TINY_WINDOW, 1, 63)
    out["tiny"] = (x, [a] + tiny + [n - a - TINY_WINDOW], [rate] * (len(tiny) + 2))
    out["p65536"] = (x, [65_536] * (n // 65_536) + ([n % 65_536] if n % 65_536 else []), None)
    out["random"] = (x, _random_chunks(_rng(case, "random"), n, 1_000, 300_000), None)
    # a capture at one rate followed by the same scenario at another, in one stream, and the other way round
    other = R.RATES[(R.RATES.index(rate) + 1) % len(R.RATES)]
    y = R.capture(case[0], other)
    for name, parts in (("rate_up", ((x, rate), (y, other))), ("rate_down", ((y, other), (x, rate)))):
        rng = _rng(case, name)
        chunks, rates = [], []
        for z, r in parts:
            c = _random_chunks(rng, len(z), 1_000, 300_000)
            chunks += c
            rates += [r] * len(c)
        out[name] = (np.concatenate([p[0] for p in parts]), chunks, rates)
    if case[0] == "warm_reset" and case[2] is None:
        for k, (b, e) in enumerate(rst_low_windows(x)):
            m = (b + e) // 2
            out["split_rst%d" % k] = (x, [m, n - m], None)
    return {k: (z, c, r if r is not None else [rate] * len(c)) for k, (z, c, r) in out.items()}


def plan_key(x, chunks, rates):
    h = hashlib.sha256(np.ascontiguousarray(x, dtype=np.float32).tobytes())
    h.update(np.asarray(chunks, dtype=np.uint64).tobytes())
    h.update(np.asarray(rates, dtype=np.uint32).tobytes())
    h.update(b"%d" % R.STREAM_TIME)
    return h.hexdigest()[:24]


@functools.lru_cache(maxsize=None)
def host_lib():
    """the host build of the stream push, compiled like tests/native/iso_host.cpp"""
    src = os.path.join(R.ROOT, "tests", "native", "iso_stream_host.cpp")
    hdr = os.path.join(R.ROOT, "nfc_laboratory_b200", "csrc", "iso_core.h")
    so = os.path.join(R.ROOT, "build", "libisostreamhost.so")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        os.makedirs(os.path.dirname(so), exist_ok=True)
        tmp = so + ".tmp%d" % os.getpid()
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-msse2", "-mfpmath=sse", "-ffp-contract=off", "-shared", "-fPIC", src, "-o", tmp])
        os.replace(tmp, so)
    lib = C.CDLL(so)
    lib.iso_host_stream.restype = C.c_long
    lib.iso_host_stream.argtypes = [C.c_void_p, C.c_int, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_long]
    return lib


def _collect(call):
    cap = 4096
    while True:
        buf = (CFrame * cap)()
        n = call(buf, cap)
        if n <= cap:
            return R.rows(buf, n)
        cap = n


def host(x, chunks, rates, sigtype=5, stream_time=R.STREAM_TIME):
    """host build: x [n, 4] (float32 for sigtype 5, int16 for 6) pushed as `chunks` at `rates`"""
    a = np.ascontiguousarray(x, dtype=np.float32 if sigtype == 5 else np.int16)
    c = np.asarray(chunks, dtype=np.uint64)
    r = np.asarray(rates, dtype=np.uint32)
    return _collect(lambda buf, cap: host_lib().iso_host_stream(a.ctypes.data, sigtype, len(a), c.ctypes.data, r.ctypes.data, len(c), stream_time,
                                                                buf, cap))


def _chunk_lib(name):
    so = os.path.join(R.ROOT, "oracle", "_ref", name)
    if not os.path.exists(so):
        return None
    lib = C.CDLL(so)
    lib.ref_iso_decode_chunks.restype = C.c_long
    lib.ref_iso_decode_chunks.argtypes = [C.c_void_p, C.c_ulong, C.c_void_p, C.c_uint, C.c_void_p, C.c_ulong, C.c_void_p, C.c_long]
    return lib


@functools.lru_cache(maxsize=None)
def ref_lib():
    """one reference lab::IsoDecoder fed chunk by chunk"""
    return _chunk_lib("libnfcref_iso_stream.so")


@functools.lru_cache(maxsize=None)
def shim_lib():
    """the same driver over the drop-in lab::IsoDecoder (nfc_laboratory_b200/shim/IsoDecoderB200.cpp, needs a GPU)"""
    return _chunk_lib("libnfcref_iso_b200.so")


def chunked(lib, x, chunks, rates, stream_time=R.STREAM_TIME):
    a = np.ascontiguousarray(x, dtype=np.float32)
    c = np.asarray(chunks, dtype=np.uint64)
    r = np.asarray(rates, dtype=np.uint32)
    return _collect(lambda buf, cap: lib.ref_iso_decode_chunks(a.ctypes.data, len(a), r.ctypes.data, stream_time, c.ctypes.data, len(c), buf, cap))


@functools.lru_cache(maxsize=None)
def golden():
    with lzma.open(GOLDEN, "rt") as f:
        return json.load(f)


def expected(case, plan):
    """the recorded oracle frames of one case pushed by one plan (the plan must be the one recorded)"""
    x, chunks, rates = plans(case)[plan]
    g = golden()["%s/%s" % (case_id(case), plan)]
    assert g["key"] == plan_key(x, chunks, rates), "the chunk plan differs from the recorded one"
    return g["frames"]


def push(dec, x, chunks, rates, sigtype):
    """the device: one iso7816_push per chunk on `dec`, then the flush, as rows"""
    frames = []
    at = 0
    for c, r in zip(chunks, rates):
        frames += dec.iso7816_push(x[at:at + c], sigtype, r, raw=True)
        at += c
    frames += dec.iso7816_flush(raw=True)
    return R.rows(frames, len(frames))
