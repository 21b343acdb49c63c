"""Long-frame captures: NFC-A I-blocks from 1 to 513 bytes at 106 / 212 / 424 kbps, frames around the frame-size limit a
RATS, ATQB or ATTRIB negotiates (NFC_FDS_TABLE: 16 ... 512 bytes, and 0), NFC-F frames up to 257 bytes, a dense batch
of such streams and two captures whose single push overflows the stream's initial frame pool.  Test infrastructure built
from the waveform helpers of nfc_laboratory_b200/synth.py and tests/extra_signals.py; every capture is seeded float32
magnitude.

A case is (samples, built): `built` lists the (frame type, payload) of every poll / listen frame the capture was built
with, in order, or is None where the reference truncates a frame at its limit."""
import functools
import hashlib
import json
import lzma
import os
import zlib

import numpy as np

import extra_signals as X
import nfc_stream_ref as T
import nfcutil as U
from nfc_laboratory_b200 import synth as Y

FS = 10_000_000
POLL, LISTEN = 0x102, 0x103
FDS = [16, 24, 32, 40, 48, 64, 96, 128, 256, 512, 1024, 2048, 4096, 0, 0, 0]   # NFC_FDS_TABLE
A_LENGTHS = [1, 79, 80, 81, 128, 207, 208, 209, 255, 256, 257]
A_LENGTHS_512 = [335, 336, 337, 463, 464, 465, 511, 512, 513]
RATS_FSDI = [0, 1, 2, 5, 8, 9]
F_LENGTHS = [78, 80, 81, 206, 209, 254]
GAP = 20_000        # idle samples that put the next exchange into a lane of its own
PCM = 32768.0


def _rng(*parts):
    return np.random.default_rng(zlib.crc32("/".join(map(str, parts)).encode()))


def noisy(m, seed, amplitude=0.3, sigma=8e-4, lead=60_000, tail=80_000):
    """carrier of `amplitude` modulated by m, with idle carrier before and after, |x + noise|, quantised to int16 steps
    (so that the int16 input of the same capture is exact)"""
    x = np.concatenate([np.ones(lead, np.float32), m, np.ones(tail, np.float32)]) * np.float32(amplitude)
    x = np.abs(x + _rng("noise", seed).normal(0, sigma, x.size))
    return (np.round(np.clip(x, 0, 0.9999) * PCM) / PCM).astype(np.float32)


def s16(x):
    pcm = np.round(x * PCM).astype(np.int16)
    assert np.array_equal(pcm.astype(np.float32) / np.float32(PCM), x)
    return pcm


def iblock(n, pcb, *seed):
    """an ISO-DEP block of n bytes: PCB, seeded payload, CRC_A; n == 1: the short REQA"""
    if n == 1:
        return b"\x26"
    b = bytes([pcb]) + _rng("iblock", n, pcb, *seed).integers(0, 256, n - 3, dtype=np.uint8).tobytes()
    return b + Y.crc_a(b)


def with_crc_a(b):
    return bytes(b) + Y.crc_a(bytes(b))


def rats(fsdi):
    return with_crc_a([0xE0, (fsdi << 4) | 0])


ATS = with_crc_a([0x05, 0x78, 0x80, 0x70, 0x02])
SPACE = np.ones(GAP, np.float32)


def render(w, t_end):
    """synth.Wave.render, the same samples, with each interval found by bisection instead of a mask over the whole
    capture (a 512-byte frame has thousands of intervals)"""
    n = int(np.ceil(t_end * w.fs / Y.FC))
    t = np.arange(n, dtype=np.float64) * Y.FC / w.fs
    m = np.ones(n, dtype=np.float64)
    for (t0, t1, lv) in w.iv:
        m[np.searchsorted(t, t0):np.searchsorted(t, t1)] = lv
    for (t0, t1, depth, inv) in w.sub:
        a, b = np.searchsorted(t, t0), np.searchsorted(t, t1)
        ph = np.floor((t[a:b] - t0) / 8.0).astype(np.int64) & 1
        m[a:b] -= depth * (ph == (1 if inv else 0)).astype(np.float64)
    return m.astype(np.float32)


def a_exchange(poll, listen, rate=0, lead=4000.0):
    """synth.nfca_exchange rendered by render()"""
    w = Y.Wave(FS)
    last_rise, last_bit, t = Y.nfca_poll(w, lead, poll, rate, short=poll == b"\x26")
    ts = last_rise + (1236 if last_bit else 1172)
    t = Y.nfca_listen_106(w, ts, listen) if rate == 0 else Y.nfca_listen_bpsk(w, ts, listen, rate)
    return render(w, t + lead)


def b_exchange(poll, listen, lead=4000.0):
    """synth.nfcb_exchange rendered by render()"""
    w = Y.Wave(FS)
    t = Y.nfcb_poll(w, lead, poll)
    t = Y.nfcb_listen(w, t + 1024 + 200 * Y.FC / FS, listen)
    return render(w, t + lead)


def _fits(frames, limit):
    return all(len(p) <= limit for _, p in frames)


def nfca_case(n, rate, fsdi=None, later=False):
    """an NFC-A poll / listen I-block pair of n bytes each at 106 kbps << rate, behind a RATS with `fsdi` (at 106 kbps, in
    the same segment or GAP idle samples later) or alone; the listen of n == 1 is an ATQA"""
    parts, frames = [], []
    if fsdi is not None:
        parts.append(a_exchange(rats(fsdi), ATS))
        frames += [(POLL, rats(fsdi)), (LISTEN, ATS)]
        if later:
            parts.append(SPACE)
    poll, listen = iblock(n, 0x02, rate, fsdi), (b"\x04\x00" if n == 1 else iblock(n, 0x03, rate, fsdi))
    parts.append(a_exchange(poll, listen, rate))
    frames += [(POLL, poll), (LISTEN, listen)]
    limit = 256 if fsdi is None else FDS[fsdi]
    x = noisy(np.concatenate(parts), ("a", n, rate, fsdi, later))
    return x, frames if _fits(frames, limit) else None


def fsdi0_case():
    """RATS with FSDI 13 (frame-size limit 0) and, each in a lane of its own, a REQA / ATQA, an I-block pair and a second
    RATS at FSDI 8 with an I-block pair behind it"""
    parts = [a_exchange(rats(13), ATS), SPACE, a_exchange(b"\x26", b"\x04\x00"), SPACE]
    parts += [a_exchange(iblock(20, 0x02, 13), iblock(20, 0x03, 13)), SPACE, a_exchange(rats(8), ATS), SPACE]
    parts += [a_exchange(iblock(40, 0x02, 8), iblock(40, 0x03, 8))]
    return noisy(np.concatenate(parts), "fsdi13"), None


REQB = bytes([0x05, 0x00, 0x00])


def atqb(fsci):
    return bytes([0x50, 0x11, 0x22, 0x33, 0x44, 0x00, 0x00, 0x00, 0x00, 0x00, (fsci << 4) | 0x01, 0x71])


def attrib(fsdi):
    return bytes([0x1D, 0x11, 0x22, 0x33, 0x44, 0x00, fsdi & 0xF, 0x01, 0x00])


def b_block(n, pcb, *seed):
    """an NFC-B block of n bytes with its CRC_B (nfcb_exchange appends the CRC)"""
    return bytes([pcb]) + _rng("bblock", n, pcb, *seed).integers(0, 256, n - 3, dtype=np.uint8).tobytes()


def with_crc_b(b):
    return bytes(b) + Y.crc_b(bytes(b))


def nfcb_case(kind, code, n):
    """REQB / ATQB with FSCI `code` ("atqb") or REQB / ATQB / ATTRIB with FSDI `code` ("attrib"), then a block pair of n
    bytes (CRC included) GAP idle samples later"""
    parts = [b_exchange(REQB, atqb(code if kind == "atqb" else 8))]
    frames = [(POLL, with_crc_b(REQB)), (LISTEN, with_crc_b(atqb(code if kind == "atqb" else 8)))]
    if kind == "attrib":
        parts += [SPACE, b_exchange(attrib(code), b"\x00")]
        frames += [(POLL, with_crc_b(attrib(code))), (LISTEN, with_crc_b(b"\x00"))]
    poll, listen = b_block(n, 0x02, kind, code), b_block(n, 0x03, kind, code)
    parts += [SPACE, b_exchange(poll, listen)]
    frames += [(POLL, with_crc_b(poll)), (LISTEN, with_crc_b(listen))]
    x = noisy(np.concatenate(parts), ("b", kind, code, n))
    return x, frames if _fits(frames, FDS[code]) else None


def nfcf_case(n, rate):
    """one NFC-F poll frame with an n-byte payload at 212 kbps (rate 1) or 424 kbps (rate 2): LEN, payload, CRC"""
    payload = _rng("f", n, rate).integers(0, 256, n, dtype=np.uint8).tobytes()
    w = Y.Wave(FS)
    t = X.nfcf_frame(w, 4000.0, payload, rate, 0.40)
    body = bytes([n + 1]) + payload
    frames = [(POLL, body + Y.crc_f(body))]
    return noisy(render(w, t + 4000.0), ("f", n, rate)), frames if _fits(frames, 256) else None


def case_builders():
    """name -> zero-argument builder of every long-frame case"""
    out = {}
    for rate in (0, 1, 2):
        for n in A_LENGTHS:
            out["a%d/n%d" % (rate, n)] = functools.partial(nfca_case, n, rate)
        for n in A_LENGTHS_512:
            out["a%d/fsdi9/n%d" % (rate, n)] = functools.partial(nfca_case, n, rate, 9)
    for fsdi in RATS_FSDI:
        limit = FDS[fsdi]
        for n in sorted({limit - 1, limit, limit + 1, 300}):
            for later in (False, True):
                out["a0/fsdi%d/%s/n%d" % (fsdi, "later" if later else "same", n)] = functools.partial(nfca_case, n, 0, fsdi, later)
    out["a0/fsdi13"] = fsdi0_case
    for kind, codes in (("atqb", (0, 2)), ("attrib", (0, 8))):
        for code in codes:
            limit = FDS[code]
            for n in sorted({limit - 1, limit, limit + 1, 100}):
                out["b/%s%d/n%d" % (kind, code, n)] = functools.partial(nfcb_case, kind, code, n)
    for rate in (1, 2):
        for n in F_LENGTHS:
            out["f%d/n%d" % (rate, n)] = functools.partial(nfcf_case, n, rate)
    return out


NAMES = list(case_builders())
def comparable(recs):
    """the part of a frame list (records or 8-tuples) that the reference answers deterministically: up to and including
    the first 1-byte RATS (0xE0) poll frame, which noise after a truncated frame can produce.  There the reference reads
    the FSDI from the byte after the frame, recycled frame-pool memory whose content depends on what the process decoded
    before, where the port reads 0 (DESIGN.md section 2)"""
    for i, r in enumerate(recs):
        if r[1] == POLL and (r[7] == "e0" or r[7] == b"\xe0"):
            return list(recs[:i + 1])
    return list(recs)


@functools.lru_cache(maxsize=None)
def case(name):
    return case_builders()[name]()


def input_hash(x):
    return hashlib.sha256(np.ascontiguousarray(x, dtype=np.float32).tobytes()).hexdigest()[:24]


# --- the dense batch -----------------------------------------------------------------------------------------------------
DENSE_STREAMS, DENSE_SAMPLES = 12, 3_000_000


@functools.lru_cache(maxsize=1)
def dense_batch():
    """[DENSE_STREAMS, DENSE_SAMPLES]: each stream a seeded shuffle of the long-frame cases and short REQA / ATQA
    exchanges behind a different length of idle carrier, cut at DENSE_SAMPLES"""
    short = a_exchange(b"\x26", b"\x04\x00")
    room = DENSE_SAMPLES - 140_000   # what noisy() adds around the modulation
    rows = []
    for s in range(DENSE_STREAMS):
        rng = _rng("dense", s)
        parts = [np.ones(10_000 + 37_000 * s, np.float32)]
        at = parts[0].size
        for k in rng.permutation(len(NAMES)):
            m = np.clip(case(NAMES[k])[0] / np.float32(0.3), 0, 1.2)
            more = [m, short] if rng.random() < 0.5 else [m]
            size = sum(p.size for p in more)
            if at + size <= room:
                parts += more
                at += size
        parts.append(np.ones(room - at, np.float32))
        rows.append(noisy(np.concatenate(parts), ("dense", s)))
    return np.stack(rows)


# --- captures that overflow one push's initial frame pool (2^14 records, 2^12 extension chunks) -------------------------
REQA_PAIRS, REQA_SPACING = 8_400, 6_000
EXT_PAIRS = 2_100


@functools.lru_cache(maxsize=2)
def overflow_capture(kind):
    """int16 magnitude: "records" -- REQA_PAIRS REQA / ATQA exchanges every REQA_SPACING samples, more than 2^14 frames;
    "chunks" -- EXT_PAIRS pairs of 81-byte I-blocks at 424 kbps, one extension chunk each, more than 2^12 chunks"""
    if kind == "records":
        m = a_exchange(b"\x26", b"\x04\x00", lead=1000.0)
        unit = np.concatenate([m, np.ones(REQA_SPACING - m.size, np.float32)])
        body = np.tile(unit, REQA_PAIRS)
    else:
        m = a_exchange(iblock(81, 0x02, "ext"), iblock(81, 0x03, "ext"), 2, lead=1000.0)
        body = np.tile(m, EXT_PAIRS)
    return s16(noisy(body, ("overflow", kind)))


# --- the reference's answers -------------------------------------------------------------------------------------------
GOLDEN = os.path.join(U.GOLDEN, "ref_long_frames.json.xz")
DIGESTED = ("overflow/",)   # entries recorded as a count and a digest of their records (thousands of frames)


def digest(recs):
    return hashlib.sha256(json.dumps(recs, separators=(",", ":")).encode()).hexdigest()[:32]


def golden_inputs():
    """name -> float32 magnitude of every reference run the tests compare with, built lazily"""
    out = {"case/" + name: functools.partial(lambda n: case(n)[0], name) for name in NAMES}
    out.update({"dense/%d" % s: functools.partial(lambda k: dense_batch()[k], s) for s in range(DENSE_STREAMS)})
    out.update({"overflow/" + k: functools.partial(lambda k: overflow_capture(k).astype(np.float32) / np.float32(PCM), k)
                for k in ("records", "chunks")})
    return out


def steps(x):
    """the reference's run of input x: 65 536-sample buffers, then the flush, fed 2^20 samples per call to the oracle (its
    output buffer holds 2^14 frames)"""
    return [("push", x[a:a + (1 << 20)], T.RATE, 65536) for a in range(0, len(x), 1 << 20)] + [("flush",)]


def golden_entry(name, x):
    """what the golden file records for input x: its hash and the reference's records, or their count and digest"""
    recs = T.ref_run(steps(x))
    if name.startswith(DIGESTED):
        return {"key": T.steps_key(steps(x), T.DEFAULT), "count": len(recs), "digest": digest(recs)}
    return {"key": T.steps_key(steps(x), T.DEFAULT), "frames": recs}


@functools.lru_cache(maxsize=1)
def golden():
    if not os.path.exists(GOLDEN):
        return {}
    with lzma.open(GOLDEN, "rt") as f:
        return json.load(f)


def expected(name, x):
    """the reference's records of input x (entry `name`): live where oracle/_ref/libnfcref.so exists, else recorded; a
    digested entry gives (count, digest)"""
    if T.ref_lib() is not None:
        g = golden_entry(name, x)
    else:
        g = golden().get(name)
        assert g is not None, "no recorded reference output %r: regenerate tests/golden/ref_long_frames.json.xz" % name
        assert g["key"] == T.steps_key(steps(x), T.DEFAULT), "the input of %r differs from the recorded one" % name
    return (g["count"], g["digest"]) if name.startswith(DIGESTED) else [tuple(r) for r in g["frames"]]


# --- the packed device records (include/nfcb200.h nfcb200_device_frames) --------------------------------------------------
RECORD = np.dtype([("stream", "<u4"), ("gen", "<u4"), ("seq", "<u4"), ("tech", "<u4"), ("type", "<u4"), ("flags", "<u4"),
                   ("phase", "<u4"), ("rate", "<u4"), ("start", "<u4"), ("end", "<u4"), ("len", "<u4"), ("ext", "<u4"),
                   ("data", "u1", 80)])
CHUNK = 128
NO_EXT = 0xFFFFFFFF
assert RECORD.itemsize == 128


def pack_records(frames):
    """(records, chunks) of frames [(stream, tech, type, flags, phase, rate, start, end, payload)]: the first 80 payload
    bytes inline, the rest in consecutive 128-byte chunks numbered from 0"""
    rec = np.zeros(len(frames), RECORD)
    chunks = []
    for i, (stream, tech, ftype, flags, phase, rate, start, end, p) in enumerate(frames):
        for k, v in zip(("stream", "seq", "tech", "type", "flags", "phase", "rate", "start", "end", "len"),
                        (stream, i, tech, ftype, flags, phase, rate, start, end, len(p))):
            rec[i][k] = v
        rec[i]["data"][:min(80, len(p))] = np.frombuffer(p[:80], np.uint8)
        rec[i]["ext"] = NO_EXT
        if len(p) > 80:
            rec[i]["ext"] = len(chunks)
            rest = p[80:]
            chunks += [rest[k:k + CHUNK].ljust(CHUNK, b"\0") for k in range(0, len(rest), CHUNK)]
    return rec, np.frombuffer(b"".join(chunks), np.uint8).copy()


def parse_records(rec, ext, stream_offset=0):
    """[(stream + stream_offset, tech, type, flags, phase, rate, start, end, payload)] of packed records and their chunks"""
    rec = np.frombuffer(np.ascontiguousarray(rec).tobytes(), RECORD)
    ext = np.ascontiguousarray(ext, dtype=np.uint8).tobytes()
    out = []
    for r in rec:
        n = int(r["len"])
        p = r["data"][:min(n, 80)].tobytes()
        if n > 80:
            e = int(r["ext"]) * CHUNK
            assert r["ext"] != NO_EXT and e + n - 80 <= len(ext), "payload of %d bytes without its chunks" % n
            p += ext[e:e + n - 80]
        out.append((int(r["stream"]) + stream_offset,) + tuple(int(r[k]) for k in ("tech", "type", "flags", "phase", "rate", "start", "end")) + (p,))
    return out
