"""Protocol-layer captures: responses swept across the guard and waiting edges of the listen window each command or
negotiated value sets (NFC-A FWT_ATQA / activation / FWI 0-15, NFC-B ATQB / FWI, NFC-F time slots, NFC-V), the same edges
at every position of a 32-sample chunk, responses that arrive after an idle stretch inside a negotiated window, Mifare
encrypted sessions, frames with a flipped parity or CRC bit and partial-byte anticollision frames, and long captures of
sessions for the carry exchange.  Test infrastructure built from the waveform helpers of nfc_laboratory_b200/synth.py,
tests/extra_signals.py and tests/long_frames.py; every capture is seeded float32 magnitude at 10 MS/s, quantised so that
its int16 input is exact.

A capture is built from parts: modulation arrays and `Gap(n)` (n samples of unmodulated carrier).  A response at delay d
starts d samples after the last sample of its poll frame's rendering.  The edge delays are measured on the reference
(tests/golden/make_protocol_golden.py) and read from the golden file, so that the captures exist without the reference.

A case is (samples, built): `built` lists the (frame type, payload) of every poll / listen frame the capture was built
with, in order, or is None where the reference's answer is not a plain function of the payloads (errors, partial bytes)."""
import functools
import json
import lzma
import os

import numpy as np

import extra_signals as X
import long_frames as L
import nfc_stream_ref as T
import nfcutil as U
from nfc_laboratory_b200 import synth as Y

FS = L.FS
POLL, LISTEN = L.POLL, L.LISTEN
GAP = L.GAP
FL_SHORT, FL_ENCRYPTED, FL_PARITY, FL_CRC = 0x01, 0x02, 0x10, 0x20
STU = FS / Y.FC
_rng = L._rng


def _odd(b):
    return Y._odd_parity(b)


def byte_bits(data, flip_parity=None, parity=None, last_partial=None):
    """LSB-first data bits, each byte followed by its odd parity bit: `flip_parity` inverts the parity of that byte index,
    `parity` gives every parity bit explicitly; `last_partial` sends only that many bits of the last byte, no parity"""
    bits = []
    for i, b in enumerate(data):
        if last_partial is not None and i == len(data) - 1:
            bits += [(b >> k) & 1 for k in range(last_partial)]
            break
        p = _odd(b) if parity is None else parity[i]
        bits += [(b >> k) & 1 for k in range(8)] + [p ^ (1 if i == flip_parity else 0)]
    return bits


# --- NFC-A ----------------------------------------------------------------------------------------------------------------
def a_poll_bits(bits, rate=0, lead=4000.0, depth=0.98):
    """modified Miller poll frame of explicit bits (synth.nfca_poll), rendered up to the rise of its last pause"""
    T_ = 128 >> rate
    pw = 32 if rate == 0 else (20 if rate == 1 else 10)
    w = Y.Wave(FS)
    lv = 1.0 - depth
    t = lead
    w.low(t, t + pw, lv)
    last_rise = t + pw
    t += T_
    prev = 0
    for b in bits:
        if b:
            w.low(t + T_ / 2, t + T_ / 2 + pw, lv)
            last_rise = t + T_ / 2 + pw
        elif prev == 0:
            w.low(t, t + pw, lv)
            last_rise = t + pw
        prev = b
        t += T_
    if prev == 0:
        w.low(t, t + pw, lv)
        last_rise = t + pw
    return L.render(w, last_rise)


def a_poll(data, rate=0, **kw):
    """poll frame of bytes (one byte of 7 bits when `short`)"""
    short = kw.pop("short", False)
    bits = [(data[0] >> k) & 1 for k in range(7)] if short else byte_bits(data, **kw)
    return a_poll_bits(bits, rate)


def a_listen_bits(bits, rate=0, depth=None):
    """listen frame of explicit bits starting at sample 0: Manchester at 106 kbps (SOF bit first), BPSK at 212 / 424
    kbps (reference phase, start bit 0), rendered to its end"""
    w = Y.Wave(FS)
    t = 0.0
    if rate == 0:
        for b in [1] + bits:
            if b:
                w.burst(t, t + 64, 0.08 if depth is None else depth)
            else:
                w.burst(t + 64, t + 128, 0.08 if depth is None else depth)
            t += 128
    else:
        T_ = 128 >> rate
        d = 0.10 if depth is None else depth
        w.burst(t, t + 32 * 16, d)
        t += 32 * 16
        for b in [0] + bits:
            w.burst(t, t + T_, d, inverted=(b == 0))
            t += T_
    return L.render(w, t + 64)


def a_listen(data, rate=0, flip_parity=None, parity=None, last_partial=None, first_bits=None):
    """listen frame of bytes; BPSK frames invert the last parity bit (NfcA.cpp, ISO 14443-3 at 212 / 424 kbps);
    `first_bits` sends only the high bits from that bit index of the first byte (the anticollision answer to a partial
    byte), then its parity"""
    if parity is None:
        parity = [_odd(b) for b in data]
        if rate:
            parity[-1] ^= 1
    bits = byte_bits(data, flip_parity=flip_parity, parity=parity, last_partial=last_partial)
    if first_bits is not None:
        bits = bits[first_bits:]
    return a_listen_bits(bits, rate)


A_NOMINAL = int(round(1172 * STU))       # FDT of a poll frame ending in logic 0, in samples


class Gap:
    def __init__(self, n):
        self.n = int(n)


def concat(parts):
    return np.concatenate([np.ones(p.n, np.float32) if isinstance(p, Gap) else p for p in parts])


def with_crc_a(b):
    return L.with_crc_a(b)


def bad_crc(b):
    """frame b with the lowest bit of its CRC flipped"""
    return bytes(b[:-2]) + bytes([b[-2] ^ 1, b[-1]])


UID = bytes([0x08, 0x12, 0x34, 0x56])
BCC = bytes([UID[0] ^ UID[1] ^ UID[2] ^ UID[3]])
REQA, WUPA, ATQA = b"\x26", b"\x52", b"\x04\x00"
SEL = with_crc_a(bytes([0x93, 0x70]) + UID + BCC)
SAK = with_crc_a(b"\x08")
HLTA = with_crc_a(b"\x50\x00")


def ats(fwi=None, sfgi=0):
    """ATS with FSCI 8 and TA / TC; TB = FWI, SFGI when fwi is given, else no TB"""
    if fwi is None:
        return with_crc_a([0x04, 0x58, 0x80, 0x02])
    return with_crc_a([0x05, 0x78, 0x80, (fwi << 4) | sfgi, 0x02])


RATS = L.rats(8)
PPS_REQ = {1: with_crc_a([0xD0, 0x11, 0x05]), 2: with_crc_a([0xD0, 0x11, 0x0A])}
PPS_RSP = with_crc_a([0xD0])


def iblock(n, pcb, *seed):
    return L.iblock(n, pcb, "proto", *seed)


def a_pair(poll, listen, rate=0, delay=A_NOMINAL, short=False):
    """parts of one NFC-A exchange, the response `delay` samples after the poll's rendering"""
    p = a_poll(poll, rate, short=short)
    return [p] if listen is None else [p, Gap(delay), a_listen(listen, rate)]


# --- NFC-B ----------------------------------------------------------------------------------------------------------------
B_NOMINAL = int(round(1024 * STU)) + 200
REQB = L.REQB


def atqb(fwi):
    return bytes([0x50, 0x11, 0x22, 0x33, 0x44, 0x00, 0x00, 0x00, 0x00, 0x00, 0x81, (fwi << 4) | 0x01])


ATTRIB = L.attrib(8)


def b_poll(data, crc=True):
    """NFC-B poll frame of data (+ CRC_B unless crc is False: data carries its own), rendered to its EOF's end"""
    w = Y.Wave(FS)
    T_, lv, t = 128, 1.0 - 0.12, 4000.0
    w.low(t, t + 10.5 * T_, lv)
    t += 13 * T_
    for b in Y._nfcb_chars(data + (Y.crc_b(data) if crc else b"")):
        if not b:
            w.low(t, t + T_, lv)
        t += T_
    w.low(t, t + 10.5 * T_, lv)
    return L.render(w, t + 10.5 * T_)


def b_listen(data, crc=True):
    """NFC-B listen frame from sample 0 (synth.nfcb_listen)"""
    w = Y.Wave(FS)
    payload = data + (Y.crc_b(data) if crc else b"")
    t = 0.0
    depth = 0.08
    w.burst(t, t + 80 * 16, depth)
    t += 80 * 16
    w.burst(t, t + 10.5 * 128, depth, inverted=True)
    t += 10.5 * 128
    w.burst(t, t + 2.5 * 128, depth)
    t += 2.5 * 128
    for b in Y._nfcb_chars(payload):
        w.burst(t, t + 128, depth, inverted=(b == 0))
        t += 128
    w.burst(t, t + 10.5 * 128, depth, inverted=True)
    t += 10.5 * 128
    w.burst(t, t + 128, depth)
    t += 128
    return L.render(w, t + 64)


def b_pair(poll, listen, delay=B_NOMINAL):
    return [b_poll(poll)] + ([] if listen is None else [Gap(delay), b_listen(listen)])


# --- NFC-F ----------------------------------------------------------------------------------------------------------------
F_NOMINAL = 4425


def f_frame(payload, rate, depth, body=None):
    """FeliCa frame from sample 0 (extra_signals.nfcf_frame), rendered to its end; `body` replaces LEN + payload + CRC"""
    w = Y.Wave(FS)
    if body is None:
        X.nfcf_frame(w, 0.0, payload, rate, depth)
        n = len(payload) + 1
    else:
        H, lv, t = 64 >> rate, 1.0 - depth, 0.0
        for b in bytes(6) + b"\xB2\x4D" + body:
            for k in range(7, -1, -1):
                if (b >> k) & 1:
                    w.low(t + H, t + 2 * H, lv)
                else:
                    w.low(t, t + H, lv)
                t += 2 * H
        n = len(body) - 2
    return L.render(w, (8 + n + 2) * 16 * (64 >> rate))


def reqc(tsn):
    return bytes([0x00, 0xFF, 0xFF, 0x00, tsn])


RESC = X.RESC


def f_body(payload):
    b = bytes([len(payload) + 1]) + payload
    return b + Y.crc_f(b)


def f_pair(poll, listen, rate, delay=F_NOMINAL):
    p = [np.ones(4000, np.float32), f_frame(poll, rate, 0.40)]
    return p + ([] if listen is None else [Gap(delay), f_frame(listen, rate, 0.25)])


# --- NFC-V ----------------------------------------------------------------------------------------------------------------
V_NOMINAL = int(round(4320 * STU))       # t1 of ISO 15693 (4320 / fc)
INVENTORY = X.INVENTORY
V_RESPONSE = bytes([0x00, 0x00]) + bytes([0xE0, 0x04, 0x01, 0x50, 0x12, 0x34, 0x56, 0x78])[::-1]


def v_crc(data):
    c = Y._crc16_refl(data, 0xFFFF) ^ 0xFFFF
    return bytes([c & 0xFF, c >> 8])


def v_poll(data, crc=True):
    """ISO 15693 1-of-4 poll frame (synth.nfcv_poll), rendered to the end of its EOF"""
    w = Y.Wave(FS)
    U_, lv, t = 128, 1.0 - 0.98, 4000.0
    frame = data + (v_crc(data) if crc else b"")
    w.low(t, t + U_, lv)
    w.low(t + 5 * U_, t + 6 * U_, lv)
    t += 8 * U_
    for b in frame:
        for k in range(4):
            v = (b >> (2 * k)) & 3
            w.low(t + (2 * v + 1) * U_, t + (2 * v + 2) * U_, lv)
            t += 8 * U_
    w.low(t + 2 * U_, t + 3 * U_, lv)
    return L.render(w, t + 4 * U_)


def v_listen(data, crc=True, depth=0.08):
    """ISO 15693 VICC response, one sub-carrier (fc / 32) at the high data rate, from sample 0: SOF (768 / fc unmodulated,
    24 pulses, logic 1), Manchester bits LSB first (logic 0: 8 pulses then 256 / fc unmodulated), EOF"""
    w = Y.Wave(FS)
    lv = 1.0 - depth

    def pulses(t, k):
        for i in range(k):
            w.low(t + 32 * i, t + 32 * i + 16, lv)
        return t + 32 * k

    payload = data + (v_crc(data) if crc else b"")
    t = 768.0
    t = pulses(t, 24)
    t = pulses(t + 256, 8)
    for b in payload:
        for k in range(8):
            if (b >> k) & 1:
                t = pulses(t + 256, 8)
            else:
                t = pulses(t, 8) + 256
    t = pulses(t, 8) + 256
    t = pulses(t, 24) + 768
    return L.render(w, t + 64)


# the response opens with 768 / fc (566 samples) of unmodulated carrier: a negative delay drops up to that many of them,
# which moves its sub-carrier pulses earlier than any gap can, to 6 samples after the poll's rendering
V_MIN_DELAY = -560


def v_pair(poll, listen, delay=V_NOMINAL):
    if listen is None:
        return [v_poll(poll)]
    assert delay >= V_MIN_DELAY
    r = v_listen(listen)
    return [v_poll(poll), Gap(max(delay, 0)), r[max(-delay, 0):]]


# --- the window-edge contexts ---------------------------------------------------------------------------------------------
def xgt(i):
    return int(STU * (4096 << i))


A_FWT, A_FWT_ATQA, A_FWT_ACTIVATION = int(STU * 65536), int(STU * 2304), int(STU * 71680)


class Ctx:
    """one window-edge context: the exchanges before it (parts, frames), the poll under test and its response, and the
    window the reference sets for that response (for the coarse delays)"""

    def __init__(self, name, pre, pre_frames, pair, poll, listen, nominal, fwt, min_delay=0):
        self.name, self.pre, self.pre_frames, self.pair = name, pre, pre_frames, pair
        self.poll, self.listen, self.nominal, self.fwt = poll, listen, nominal, fwt
        self.min_delay = min_delay

    def parts(self, delay):
        return self.pre + self.pair(delay)

    def frames(self):
        return self.pre_frames + [(POLL, self.poll), (LISTEN, self.listen)]


def _a_ctx(name, pre_pairs, poll, listen, rate, fwt, short=False):
    pre, frames = [], []
    for (p, l, r) in pre_pairs:
        pre += a_pair(p, l, r, short=p in (REQA, WUPA)) + [Gap(8000)]
        frames += [(POLL, p), (LISTEN, l)]
    return Ctx(name, pre, frames, lambda d: a_pair(poll, listen, rate, d, short=short), poll, listen, A_NOMINAL, fwt)


def _b_ctx(name, pre_pairs, poll, listen, fwt):
    pre, frames = [], []
    for (p, l) in pre_pairs:
        pre += b_pair(p, l) + [Gap(8000)]
        frames += [(POLL, p + Y.crc_b(p)), (LISTEN, l + Y.crc_b(l))]
    return Ctx(name, pre, frames, lambda d: b_pair(poll, listen, d), poll + Y.crc_b(poll), listen + Y.crc_b(listen), B_NOMINAL, fwt)


A_FWIS = [0, 1, 4, 7, 9, 15]
B_FWIS = [0, 4, 8]
F_TSNS = [0, 3, 15]


@functools.lru_cache(maxsize=1)
def contexts():
    out = {}
    ib = lambda r, *s: (iblock(12, 0x02, r, *s), iblock(8, 0x02, "rsp", r, *s))
    out["a0/reqa"] = _a_ctx("a0/reqa", [], REQA, ATQA, 0, A_FWT_ATQA, short=True)
    out["a0/sel"] = _a_ctx("a0/sel", [(REQA, ATQA, 0)], SEL, SAK, 0, A_FWT_ATQA)
    out["a0/rats"] = _a_ctx("a0/rats", [], RATS, ats(7), 0, A_FWT_ACTIVATION)
    out["a0/i"] = _a_ctx("a0/i", [], *ib(0), 0, A_FWT)
    for fwi in A_FWIS:
        out["a0/i/fwi%d" % fwi] = _a_ctx("a0/i/fwi%d" % fwi, [(RATS, ats(fwi), 0)], *ib(0, fwi), 0, xgt(4 if fwi == 15 else fwi))
    out["a0/i/notb"] = _a_ctx("a0/i/notb", [(RATS, ats(None), 0)], *ib(0, "notb"), 0, A_FWT)
    for rate in (1, 2):
        out["a%d/i" % rate] = _a_ctx("a%d/i" % rate, [], *ib(rate), rate, A_FWT)
        out["a%d/i/pps" % rate] = _a_ctx("a%d/i/pps" % rate, [(RATS, ats(None), 0), (PPS_REQ[rate], PPS_RSP, 0)], *ib(rate, "pps"), rate, A_FWT)
        out["a%d/i/fwi0" % rate] = _a_ctx("a%d/i/fwi0" % rate, [(RATS, ats(0), 0), (PPS_REQ[rate], PPS_RSP, 0)], *ib(rate, 0), rate, xgt(0))
    out["b/reqb"] = _b_ctx("b/reqb", [], REQB, atqb(4), int(STU * 7680))
    out["b/attrib"] = _b_ctx("b/attrib", [(REQB, atqb(4))], ATTRIB, b"\x00", xgt(4))
    for fwi in B_FWIS:
        out["b/i/fwi%d" % fwi] = _b_ctx("b/i/fwi%d" % fwi, [(REQB, atqb(fwi)), (ATTRIB, b"\x00")], L.b_block(12, 0x02, fwi),
                                        L.b_block(8, 0x02, "rsp", fwi), xgt(fwi))
    for rate in (1, 2):
        for tsn in F_TSNS:
            name = "f%d/tsn%d" % (rate, tsn)
            out[name] = Ctx(name, [], [], functools.partial(lambda r, t, d: f_pair(reqc(t), RESC, r, d), rate, tsn),
                            f_body(reqc(tsn)), f_body(RESC), F_NOMINAL, int(STU * (512 * 64 + (tsn + 1) * 256 * 64)))
    out["v/inventory"] = Ctx("v/inventory", [], [], lambda d: v_pair(INVENTORY, V_RESPONSE, d), INVENTORY + v_crc(INVENTORY),
                             V_RESPONSE + v_crc(V_RESPONSE), V_NOMINAL, A_FWT, V_MIN_DELAY)
    return out


CONTEXTS = list(contexts())
# the contexts whose edges are swept across every position of a 32-sample chunk (short windows: small captures)
CHUNK_CONTEXTS = ["a0/reqa", "a0/i/fwi0", "a0/i", "a1/i/fwi0", "b/reqb", "f1/tsn0"]


def edge_capture(ctx, delay, shift=0, amplitude=0.3, sigma=8e-4, lead=60_000, tail=80_000):
    """context ctx with its response at `delay`, behind `shift` leading samples, as long_frames.noisy builds a capture but
    with noise that moves with the signal: one sequence over everything before the response and one that starts with
    the response, each drawn per context, and `shift` prepended samples with noise of their own.  So every capture of a
    context has the same poll frame, ending at the same sample plus the shift, and the same response with the same noise;
    only the gap between them changes"""
    parts = contexts()[ctx].parts(delay)
    m = concat(parts)
    split = shift + lead + m.size - parts[-1].size
    x = np.concatenate([np.ones(shift + lead, np.float32), m, np.ones(tail, np.float32)]) * np.float32(amplitude)
    trim = max(-delay, 0)   # the leading carrier samples a negative NFC-V delay drops (v_pair)
    z = np.concatenate([_rng("edge/shift", ctx).normal(0, sigma, shift), _rng("edge", ctx).normal(0, sigma, split - shift),
                        _rng("edge/response", ctx).normal(0, sigma, x.size - split + trim)[trim:]])
    x = np.abs(x + z)
    return (np.round(np.clip(x, 0, 0.9999) * L.PCM) / L.PCM).astype(np.float32)


def responds(recs, ctx):
    """the response of context ctx is among the records (or 8-tuples)"""
    want = contexts()[ctx].listen
    for r in recs:
        p = r[7] if isinstance(r[7], bytes) else bytes.fromhex(r[7])
        if r[1] == LISTEN and p == want:
            return True
    return False


# --- late responses across lanes ------------------------------------------------------------------------------------------
def late_cases():
    """name -> (parts, built, padded?): a poll, then more than GAP samples of silence inside its negotiated window, then the
    response, a new poll or the end of the capture"""
    out = {}
    for fwi, silence in ((7, 30_000), (7, 100_000), (7, 300_000), (9, 1_000_000)):
        poll, listen = iblock(20, 0x02, "late", fwi, silence), iblock(10, 0x03, "late", fwi, silence)
        parts = a_pair(RATS, ats(fwi)) + [Gap(10_000)] + a_pair(poll, listen, delay=silence)
        out["late/a/fwi%d/%d" % (fwi, silence)] = (parts, [(POLL, RATS), (LISTEN, ats(fwi)), (POLL, poll), (LISTEN, listen)], True)
    poll, listen = L.b_block(14, 0x02, "late"), L.b_block(9, 0x02, "late/rsp")
    parts = b_pair(REQB, atqb(8)) + [Gap(10_000)] + b_pair(ATTRIB, b"\x00") + [Gap(10_000)] + b_pair(poll, listen, 400_000)
    out["late/b/fwi8"] = (parts, [(POLL, L.with_crc_b(REQB)), (LISTEN, L.with_crc_b(atqb(8))), (POLL, L.with_crc_b(ATTRIB)),
                                  (LISTEN, L.with_crc_b(b"\x00")), (POLL, L.with_crc_b(poll)), (LISTEN, L.with_crc_b(listen))], True)
    poll = iblock(20, 0x02, "late", "poll")
    parts = a_pair(RATS, ats(7)) + [Gap(10_000)] + a_pair(poll, None) + [Gap(60_000)] + a_pair(REQA, None, short=True)
    parts += [Gap(60_000)] + a_pair(REQA, ATQA, short=True)
    out["late/a/fwi7/poll"] = (parts, [(POLL, RATS), (LISTEN, ats(7)), (POLL, poll), (POLL, REQA), (POLL, REQA), (LISTEN, ATQA)], True)
    parts = b_pair(REQB, atqb(8)) + [Gap(10_000)] + b_pair(poll[:-2], None) + [Gap(50_000)] + b_pair(REQB, atqb(0))
    out["late/b/fwi8/poll"] = (parts, None, True)
    # the capture ends inside the window: padding would lengthen the wait, these are decoded as they are
    out["late/a/fwi7/end"] = (a_pair(RATS, ats(7)) + [Gap(10_000)] + a_pair(poll, None), [(POLL, RATS), (LISTEN, ats(7)), (POLL, poll)], False)
    out["late/a/fwi9/end"] = (a_pair(RATS, ats(9)) + [Gap(10_000)] + a_pair(poll, None) + [Gap(200_000)],
                              [(POLL, RATS), (LISTEN, ats(9)), (POLL, poll)], False)
    out["late/b/fwi8/end"] = (b_pair(REQB, atqb(8)) + [Gap(10_000)] + b_pair(poll[:-2], None), None, False)
    return out


# --- encrypted sessions ---------------------------------------------------------------------------------------------------
def _enc_frame(rng, n):
    """n random bytes with random parity bits (the wire form of Crypto1 traffic), as (bytes, parity bits)"""
    return rng.integers(0, 256, n, dtype=np.uint8).tobytes(), [int(v) for v in rng.integers(0, 2, n)]


def enc_pair(rng, n_poll, n_listen, first=None):
    p, pp = _enc_frame(rng, n_poll)
    if first is not None:
        p = first + p[len(first):]
    l, lp = _enc_frame(rng, n_listen)
    return [a_poll_bits(byte_bits(p, parity=pp)), Gap(A_NOMINAL), a_listen(l, parity=lp)], [(POLL, p), (LISTEN, l)]


def encrypted_session(variant, seed):
    """REQA / ATQA, SEL / SAK, AUTH (0x60 / 0x61 by seed) / 4-byte nonce, encrypted exchanges in the AUTH's lane and after
    1, 2 and 5 GAP idle samples, an encrypted 6-byte frame starting 50 00 (not an HLTA: that is 4 bytes), then WUPA / ATQA and a plain I-block exchange.
    variant: "plain", "auth_bad_crc" (the AUTH's CRC flipped), "auth_no_answer", "hlta_bad_crc" (an HLTA with a flipped
    CRC before the AUTH)"""
    rng = _rng("enc", variant, seed)
    parts, frames = [], []

    def add(pp, ff, gap=5000):
        parts.extend(pp + [Gap(gap)])
        frames.extend(ff)

    add(a_pair(REQA, ATQA, short=True), [(POLL, REQA), (LISTEN, ATQA)])
    add(a_pair(SEL, SAK), [(POLL, SEL), (LISTEN, SAK)])
    if variant == "hlta_bad_crc":
        add(a_pair(bad_crc(HLTA), None), [(POLL, bad_crc(HLTA))])
    auth = with_crc_a([0x60 + (seed & 1), 0x04])
    if variant == "auth_bad_crc":
        auth = bad_crc(auth)
    nonce = rng.integers(0, 256, 4, dtype=np.uint8).tobytes()
    if variant == "auth_no_answer":
        add(a_pair(auth, None), [(POLL, auth)], gap=8000)
    else:
        add(a_pair(auth, nonce), [(POLL, auth), (LISTEN, nonce)])
    for idle in (5000, GAP, 2 * GAP, 5 * GAP):
        for k in range(2):
            pp, ff = enc_pair(rng, int(rng.integers(4, 19)), int(rng.integers(4, 19)))
            add(pp, ff, gap=idle if k else 5000)
    pp, ff = enc_pair(rng, 6, 4, first=b"\x50\x00")
    add(pp, ff)
    pp, ff = enc_pair(rng, 8, 5)
    add(pp, ff, gap=GAP)
    wake = WUPA if seed & 1 else REQA
    add(a_pair(wake, ATQA, short=True), [(POLL, wake), (LISTEN, ATQA)])
    poll, listen = iblock(16, 0x02, "after", variant, seed), iblock(6, 0x03, "after", variant, seed)
    add(a_pair(poll, listen), [(POLL, poll), (LISTEN, listen)])
    return parts, frames


ENC_VARIANTS = [("plain", 0), ("plain", 1), ("auth_bad_crc", 0), ("auth_no_answer", 1), ("hlta_bad_crc", 0)]


# --- error flags ----------------------------------------------------------------------------------------------------------
def error_cases():
    """name -> (parts, frame index, flag): one capture per error, the flag the frame at that index (poll / listen frames
    only) must carry, or None where only the reference's answer is pinned"""
    out = {}
    i12 = iblock(12, 0x02, "err")
    r12 = iblock(9, 0x03, "err")
    # one flipped parity bit: poll and listen at 106, BPSK listens (the last parity bit is inverted on the wire)
    out["parity/a0/poll"] = ([a_poll(i12, flip_parity=5), Gap(A_NOMINAL), a_listen(r12)], 0, FL_PARITY)
    out["parity/a0/listen"] = ([a_poll(i12), Gap(A_NOMINAL), a_listen(r12, flip_parity=3)], 1, FL_PARITY)
    for rate in (1, 2):
        for where, k in (("mid", 4), ("last", len(r12) - 1)):
            out["parity/a%d/listen/%s" % (rate, where)] = ([a_poll(i12, rate), Gap(A_NOMINAL), a_listen(r12, rate, flip_parity=k)], 1, FL_PARITY)
        out["parity/a%d/poll" % rate] = ([a_poll(i12, rate, flip_parity=2), Gap(A_NOMINAL), a_listen(r12, rate)], 0, FL_PARITY)
    # one flipped CRC bit per NFC-A command class
    classes = {
        "rats": ([], RATS, ats(4), 0), "ats": ([], RATS, ats(4), 1),
        "pps": ([(RATS, ats(4))], PPS_REQ[1], PPS_RSP, 0), "pps_rsp": ([(RATS, ats(4))], PPS_REQ[1], PPS_RSP, 1),
        "auth": ([(REQA, ATQA), (SEL, SAK)], with_crc_a([0x60, 0x08]), None, 0),
        "i": ([], i12, r12, 0), "i_rsp": ([], i12, r12, 1),
        "r": ([], with_crc_a([0xA2]), with_crc_a([0xA3]), 0), "r_rsp": ([], with_crc_a([0xA2]), with_crc_a([0xA3]), 1),
        "s": ([], with_crc_a([0xC2, 0x01]), with_crc_a([0xC2, 0x01]), 0), "s_rsp": ([], with_crc_a([0xC2, 0x01]), with_crc_a([0xC2, 0x01]), 1),
        "hlta": ([(REQA, ATQA)], HLTA, None, 0),
        "other": ([], with_crc_a([0x30, 0x04]), iblock(18, 0x55, "other"), 0),
        "other_rsp": ([], with_crc_a([0x30, 0x04]), iblock(18, 0x55, "other"), 1),
    }
    for name, (pre, poll, listen, which) in classes.items():
        parts, k = [], 0
        for p, l in pre:
            parts += a_pair(p, l, short=p == REQA) + [Gap(5000)]
            k += 2
        if which == 0:
            poll = bad_crc(poll)
        else:
            listen = bad_crc(listen)
        parts += a_pair(poll, listen)
        if name == "hlta":
            # after a CRC-failed 50 00: does the lane still decode?  An I-block exchange shows it
            parts += [Gap(5000)] + a_pair(i12, r12)
        out["crc/a0/" + name] = (parts, k + which, FL_CRC)
    # a bad CRC in NFC-B, NFC-F and NFC-V frames
    out["crc/b/poll"] = ([b_poll(REQB + bad_crc(b"\0\0" + Y.crc_b(REQB))[-2:], crc=False), Gap(B_NOMINAL), b_listen(atqb(4))], 0, FL_CRC)
    out["crc/b/listen"] = ([b_poll(REQB), Gap(B_NOMINAL), b_listen(atqb(4) + bad_crc(b"\0\0" + Y.crc_b(atqb(4)))[-2:], crc=False)], 1, FL_CRC)
    for rate in (1, 2):
        out["crc/f%d/poll" % rate] = ([np.ones(4000, np.float32), f_frame(None, rate, 0.40, body=bad_crc(f_body(reqc(0)))), Gap(F_NOMINAL),
                                       f_frame(RESC, rate, 0.25)], 0, FL_CRC)
        out["crc/f%d/listen" % rate] = ([np.ones(4000, np.float32), f_frame(reqc(0), rate, 0.40), Gap(F_NOMINAL),
                                         f_frame(None, rate, 0.25, body=bad_crc(f_body(RESC)))], 1, FL_CRC)
    out["crc/v/poll"] = ([v_poll(bad_crc(INVENTORY + v_crc(INVENTORY)), crc=False), Gap(V_NOMINAL), v_listen(V_RESPONSE)], 0, FL_CRC)
    out["crc/v/listen"] = ([v_poll(INVENTORY), Gap(V_NOMINAL), v_listen(bad_crc(V_RESPONSE + v_crc(V_RESPONSE)), crc=False)], 1, FL_CRC)
    # anticollision with NVB 0x21 ... 0x67: a partial last byte of 1 ... 7 bits, answered by the rest of the UID
    uid = UID + BCC
    for nbytes in range(2, 7):
        for nbits in range(1, 8):
            nvb = (nbytes << 4) | nbits
            known = nbytes - 2
            sent = bytes([0x93, nvb]) + uid[:known + 1]
            poll = a_poll_bits(byte_bits(sent, last_partial=nbits))
            rest = uid[known:]
            parts = a_pair(REQA, ATQA, short=True) + [Gap(5000), poll, Gap(A_NOMINAL + 64 * nbits), a_listen(rest, first_bits=nbits)]
            out["sdd/nvb%02x" % nvb] = (parts, None, None)
    # 7-bit short frames other than REQA / WUPA
    for b in (0x35, 0x40, 0x43, 0x7F, 0x00):
        out["short/%02x" % b] = (a_pair(bytes([b]), ATQA, short=True), None, None)
    return out


# --- long captures for the carry exchange ---------------------------------------------------------------------------------
LONG_CAPTURES = 3
LONG_SAMPLES = 4_000_000


@functools.lru_cache(maxsize=LONG_CAPTURES)
def long_capture(k):
    """about 4e6 samples: late-response cases and encrypted sessions in a seeded order, with long idle points inside the
    encrypted sessions and after FWI changes"""
    rng = _rng("long", k)
    late = late_cases()
    pieces = [concat(encrypted_session(v, s + 10 * k)[0]) for v, s in ENC_VARIANTS]
    pieces += [concat(late[n][0]) for n in sorted(late) if late[n][2] and "fwi9" not in n]
    parts, at = [], 0
    for i in rng.permutation(len(pieces)):
        if at + pieces[i].size > LONG_SAMPLES - 300_000:
            continue
        parts.append(pieces[i])
        gap = int(rng.integers(5_000, 120_000))
        parts.append(np.ones(gap, np.float32))
        at += pieces[i].size + gap
    parts.append(np.ones(max(0, LONG_SAMPLES - 140_000 - at), np.float32))
    return L.noisy(np.concatenate(parts), ("long", k))


# --- the golden -----------------------------------------------------------------------------------------------------------
GOLDEN = os.path.join(U.GOLDEN, "ref_protocol.json.xz")
SWEEP = range(-3, 4)


@functools.lru_cache(maxsize=1)
def golden():
    if not os.path.exists(GOLDEN):
        return {}
    with lzma.open(GOLDEN, "rt") as f:
        return json.load(f)


def edges():
    """ctx -> {"guard": d*, "wait": d*}: the first delay at which the response decodes and the last one, measured on the
    reference by make_protocol_golden.py"""
    g = golden().get("edges")
    assert g is not None, "no recorded edge delays: regenerate tests/golden/ref_protocol.json.xz with the reference"
    return g


def coarse_delays(ctx):
    """6 delays from the nominal response time to 1.2 x the window"""
    c = contexts()[ctx]
    return [int(v) for v in np.linspace(c.nominal, 1.2 * c.fwt, 6)]


def sweep_delays(ctx):
    e = edges()[ctx]
    lo = contexts()[ctx].min_delay
    out = {e[k] + s for k in ("guard", "wait") if e[k] is not None for s in SWEEP} | set(coarse_delays(ctx))
    if lo < 0:
        out |= {lo, lo // 2, 0}
    return sorted(d for d in out if d >= lo)


def case_builders():
    """name -> zero-argument builder of (samples, built) for every case; built: [(type, payload)] or None"""
    out = {}
    for ctx in CONTEXTS:
        for d in sweep_delays(ctx):
            out["edge/%s/d%d" % (ctx, d)] = functools.partial(lambda c, d: (edge_capture(c, d), None), ctx, d)
    for ctx in CHUNK_CONTEXTS:
        w = edges()[ctx]["wait"]
        for d in (w, w + 1):
            for shift in range(32):
                out["chunk/%s/d%d/s%d" % (ctx, d, shift)] = functools.partial(lambda c, d, s: (edge_capture(c, d, s), None), ctx, d, shift)
    for name, (parts, built, padded) in late_cases().items():
        tail = 80_000 if padded else 20_000
        out[name] = functools.partial(lambda p, b, t, n: (L.noisy(concat(p), n, tail=t), b), parts, built, tail, name)
    for v, s in ENC_VARIANTS:
        name = "enc/%s/%d" % (v, s)
        out[name] = functools.partial(lambda v, s, n: (L.noisy(concat(encrypted_session(v, s)[0]), n), encrypted_session(v, s)[1]), v, s, name)
    for name, (parts, _, _) in error_cases().items():
        out["err/" + name] = functools.partial(lambda p, n: (L.noisy(concat(p), n), None), parts, name)
    return out


@functools.lru_cache(maxsize=1)
def _builders():
    return case_builders()


def names():
    return list(_builders())


def unpadded(name):
    return name.startswith("late/") and name.endswith("/end")


@functools.lru_cache(maxsize=None)
def case(name):
    return _builders()[name]()


def steps(x):
    return L.steps(x)


@functools.lru_cache(maxsize=1)
def families():
    """family -> case names decoded in one batch call: the edge sweeps per context, the chunk shifts per context and
    delay, the late responses, the encrypted sessions and the error cases; every capture that ends inside a pending
    window alone"""
    out = {}
    for n in names():
        kind = n.split("/")[0]
        if kind == "edge":
            out.setdefault("edge/" + n.split("/d")[0].split("/", 1)[1], []).append(n)
        elif kind == "chunk":
            out.setdefault(n.rsplit("/", 1)[0], []).append(n)
        elif unpadded(n):
            out[n] = [n]
        else:
            out.setdefault(kind, []).append(n)
    return out


@functools.lru_cache(maxsize=None)
def family_length(family):
    return max(len(case(n)[0]) for n in families()[family])


def family_of(name):
    return next(f for f, ns in families().items() if name in ns)


def padded(name):
    """the capture of `name` as its family's batch holds it: padded to the family's longest capture with its last
    sample.  That adds no frame unless the capture ends inside a frame: then the decode of that frame goes on into the
    padding (a response read from its middle can run that long), and the padded capture has the frame the capture
    alone does not"""
    x = case(name)[0]
    return np.concatenate([x, np.full(family_length(family_of(name)) - len(x), x[-1], np.float32)])


def golden_inputs():
    """"case/<name>": every case as built; "padded/<name>": every case whose family pads it; "long/<k>": the long
    captures"""
    out = {"case/" + n: functools.partial(lambda n: case(n)[0], n) for n in names()}
    out.update({"padded/" + n: functools.partial(padded, n) for n in names() if len(case(n)[0]) < family_length(family_of(n))})
    out.update({"long/%d" % k: functools.partial(long_capture, k) for k in range(LONG_CAPTURES)})
    return out


def golden_entry(name, x):
    return {"key": T.steps_key(steps(x), T.DEFAULT), "frames": T.ref_run(steps(x))}


def expected(name, x):
    """the reference's records of input x (entry `name`): live where oracle/_ref/libnfcref.so exists, else recorded"""
    if T.ref_lib() is not None:
        g = golden_entry(name, x)
    else:
        g = golden().get("runs", {}).get(name)
        assert g is not None, "no recorded reference output %r: regenerate tests/golden/ref_protocol.json.xz" % name
        assert g["key"] == T.steps_key(steps(x), T.DEFAULT), "the input of %r differs from the recorded one" % name
    return [tuple(r) for r in g["frames"]]
