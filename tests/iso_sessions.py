"""Seeded ISO 7816 sessions built character by character, for the protocol tests (tests/test_iso7816_protocol.py).

A capture is 4 logic channels (IO, CLK, RST, VCC) as 0 / 1, in samples at the capture's rate.  Unlike
synth.iso7816_capture, every character's start sample is under the caller's control, and so is the CLK waveform: a
frequency per stretch, ramps, period jitter, explicit integer periods and stops with CLK held low or high.  Characters
follow synth._IsoLine's conventions: a start bit, 8 data bits, even parity, LSB first (MSB first and inverted in the
inverse convention), one ETU per bit, the receiver's error signal after the parity bit when asked.

The case families:
  edge/<ctx>/r<M>/d<delay>     a character swept across the guard edge and, in T=1, the waiting edge of its context
  shift/<ctx>/<edge>/s<k>      the edge delay d* and d* +- 1 with 0 ... 31 leading samples
  bit/<conv>/r<M>/k<skew>      one bit boundary moved -2 ... +2 samples around the decoder's sampling point
  atr/..., pps/..., err/...    ATR parameters, PPS variants, error signals and parity errors
  clk/...                      clock drift thresholds, ramps, jitter, stops, the device walk's 32-wide clock batch
The expected frames come from the reference (tests/golden/ref_iso_protocol.json.xz, make_iso_protocol_golden.py)."""
import functools
import hashlib
import json
import lzma
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_iso_protocol.json.xz")
RATES = (10_000_000, 25_000_000, 50_000_000)
STREAM_TIME = 1000
FI = [0, 372, 558, 744, 1116, 1488, 1860, 0, 0, 512, 768, 1024, 1536, 2048, 0, 0]
DI = [0, 1, 2, 4, 8, 16, 32, 64, 12, 20, 0, 0, 0, 0, 0, 0]
ATR = 0x210
FLAG_PARITY, FLAG_CRC = 0x10, 0x20


def lrc(data):
    x = 0
    for b in data:
        x ^= b
    return x


def pps(pps0, pps1=None, pps2=None, pps3=None):
    b = [0xFF, pps0] + [v for v in (pps1, pps2, pps3) if v is not None]
    return b + [lrc(b)]


def block(nad, pcb, inf):
    b = [nad, pcb, len(inf)] + list(inf)
    return b + [lrc(b)]


class Session:
    """a capture under construction.  Times are in samples (float); a character starts on the sample its start is
    rounded to, so that its start bit's falling edge lies there exactly"""

    def __init__(self, rate, fclk=4e6, inverse=False, seed=0, lead=0):
        self.rate = rate
        self.inverse = inverse
        self.rng = np.random.default_rng(seed)
        self.spc = rate / fclk               # samples per clock, for the characters' timing
        self.etu = 372 * self.spc
        self.etu_ts = self.etu                # the ETU of the ATR (Fi 1 / Di 1 at the first clock)
        self.low = []                         # IO low intervals [a, b)
        self.starts = []                      # start sample of every character
        self.t_vcc = lead + int(20e-6 * rate)
        self.t_clk = self.t_vcc + int(5e-6 * rate)
        self.t_rst = self.t_clk + int(round(500 * self.spc))
        self.t = float(self.t_rst + int(round(600 * self.spc)))
        self.rst_low = []
        self.clk_plan = [(self.t_clk, ("run", fclk, 0.0))]   # (from sample, segment)

    # --- IO --------------------------------------------------------------------------------------------------------
    def char(self, byte, at=None, parity_error=False, error_etu=None, skew=None):
        """one character at sample `at` (default: the cursor).  error_etu: the receiver pulls IO low for that many ETU
        from 10.2 ETU on.  skew (k, s): the boundary before bit k sits at sample `s` instead of its nominal place"""
        start = int(round(self.t if at is None else at))
        bits = [(byte >> i) & 1 for i in (range(7, -1, -1) if self.inverse else range(8))]
        par = (bin(byte).count("1") & 1) ^ (1 if parity_error else 0)
        levels = [0] + [(1 - b) if self.inverse else b for b in bits] + [(1 - par) if self.inverse else par]
        bounds = [start + k * self.etu for k in range(11)]
        if skew is not None:
            bounds[skew[0]] = skew[1]
        for k, lv in enumerate(levels):
            if lv == 0:
                self.low.append((bounds[k], bounds[k + 1]))
        self.starts.append(start)
        if error_etu:
            self.low.append((start + 10.2 * self.etu, start + (10.2 + error_etu) * self.etu))
            self.t = start + (12.2 + error_etu) * self.etu
        else:
            self.t = start + 12 * self.etu
        return start

    def frame(self, data, gap=20.0, delays=None, step=12.0, errors=None, skew=None):
        """bytes `step` ETU apart (delays: index -> samples from the previous character's start instead); errors: index
        -> (error signal ETU, repeats): the character goes out with a parity error and the error signal, `repeats`
        times, then right"""
        delays, errors = delays or {}, errors or {}
        for i, b in enumerate(data):
            for _ in range(errors.get(i, (0, 0))[1]):
                self.char(b, parity_error=True, error_etu=errors[i][0])
            at = self.starts[-1] + delays[i] if i in delays else None
            if i and i not in delays and at is None:
                at = self.starts[-1] + step * self.etu if self.t <= self.starts[-1] + step * self.etu else None
            self.char(b, at=at, skew=skew if skew and skew[0] == i else None)
            if skew and skew[0] == i:
                skew = None
        self.t += (gap - 12) * self.etu
        return self

    def use(self, fi, di, fclk=None):
        """characters from here at Fi / Di (and at clock `fclk` when given)"""
        if fclk is not None:
            self.spc = self.rate / fclk
        self.etu = FI[fi] / DI[di] * self.spc
        return self

    def wait(self, etu):
        self.t += etu * self.etu
        return self

    # --- CLK -------------------------------------------------------------------------------------------------------
    def clock(self, at, kind, *args):
        """from sample `at`: ("run", hz, jitter), ("ramp", hz0, hz1), ("periods", [integer periods], high samples),
        ("pattern", [integer periods], high samples) repeated, ("stop", level)"""
        self.clk_plan.append((int(round(at)), (kind,) + args))
        self.clk_plan.sort(key=lambda p: p[0])
        return self

    def _clock(self, end):
        hs, he = [], []
        c = float(self.t_clk)
        plan = self.clk_plan + [(end, None)]
        for (a, seg), (b, _) in zip(plan[:-1], plan[1:]):
            c = max(c, float(a))
            kind = seg[0]
            if kind == "stop":
                if seg[1]:
                    hs.append(c)
                    he.append(float(b))
                c = float(b)
                continue
            if kind in ("periods", "pattern"):
                per, high = seg[1], seg[2]
                i = 0
                while c < b and (kind == "pattern" or i < len(per)):
                    hs.append(c)
                    he.append(c + high)
                    c += per[i % len(per)]
                    i += 1
                continue
            if kind == "run":
                nom = self.rate / seg[1]
                k = int((b - c) / (nom * (1 - seg[2]))) + 2
                p = nom * (1 + seg[2] * self.rng.uniform(-1, 1, k))
                st = c + np.concatenate(([0.0], np.cumsum(p)[:-1]))
                m = int(np.searchsorted(st, b))
                hs += st[:m].tolist()
                he += (st[:m] + p[:m] / 2).tolist()
                c = float(st[m - 1] + p[m - 1]) if m else c
                continue
            while c < b:
                p = self.rate / (seg[1] + (seg[2] - seg[1]) * (c - a) / max(b - a, 1))
                hs.append(c)
                he.append(c + p / 2)
                c += p
        return np.asarray(hs), np.asarray(he)

    # --- render ----------------------------------------------------------------------------------------------------
    def render(self, tail=100e-6):
        t_off = int(self.t + tail * self.rate)
        n = t_off + int(30e-6 * self.rate)
        i = np.arange(n, dtype=np.float64)
        vcc = ((i >= self.t_vcc) & (i < t_off)).astype(np.float32)
        rst = ((i >= self.t_rst) & (i < t_off)).astype(np.float32)
        for a, b in self.rst_low:
            rst[(i >= a) & (i < b)] = 0
        hs, he = self._clock(t_off - int(10e-6 * self.rate))
        k = np.searchsorted(hs, i, side="right") - 1
        clk = ((k >= 0) & (i < he[np.maximum(k, 0)])).astype(np.float32)
        io = ((i >= self.t_vcc + int(2e-6 * self.rate)) & (i < t_off)).astype(np.float32)
        for a, b in self.low:
            io[int(np.ceil(a)):int(np.ceil(b))] = 0
        return np.stack([io, clk, rst, vcc], axis=1)


def measurement_edges(x):
    """samples of the CLK falling edges that bring the decoder's clock counter to 10, for a capture with no reset and no
    empty frame before them (the counter then counts from the first sample)"""
    clk = np.asarray(x)[:, 1]
    falls = np.flatnonzero(np.diff(clk, prepend=np.float32(0)) < 0)
    return falls[9::10]


# --- sessions ------------------------------------------------------------------------------------------------------------
ATR_T0 = [0x3B, 0x12, 0x11, 0x41, 0x42]                           # TA1, 2 historical bytes
SELECT = [0x00, 0xA4, 0x04, 0x00, 0x02, 0xA4, 0x3F, 0x00, 0x90, 0x00]


def atr_t1(ifsc=0xFE, bwi_cwi=0x45, tc1=None, hist=(0x4A,)):
    t0 = 0x80 | len(hist) | (0x40 if tc1 is not None else 0)
    b = [0x3B, t0] + ([tc1] if tc1 is not None else []) + [0x81, 0x31, ifsc, bwi_cwi] + list(hist)
    return b + [lrc(b[1:])]


def atr_t0(tc1=None, tc2=None, hist=(0x41, 0x42)):
    """TA1 = 0x11; TC1 when given; TC2 (WI) through TD1 = 0x40 when given"""
    y1 = 0x10 | (0x40 if tc1 is not None else 0) | (0x80 if tc2 is not None else 0)
    b = [0x3B, y1 | len(hist), 0x11] + ([tc1] if tc1 is not None else [])
    if tc2 is not None:
        b += [0x40, tc2]
    return b + list(hist)


def start(rate, atr, pps_bytes=None, resp=None, fi_di=None, **kw):
    """power-up, clock, reset, the ATR and, when given, a PPS request and its response (default: the request echoed);
    characters after it at the response's Fi / Di"""
    s = Session(rate, **kw)
    s.frame(atr, gap=200)
    if pps_bytes is not None:
        s.frame(pps_bytes, gap=30)
        if resp is not False:
            s.frame(resp or pps_bytes, gap=100)
        if fi_di is not None:
            s.use(*fi_di)
    return s


class Context:
    """one edge context: a session whose character `index` of its last frame `frame` starts `d` samples after the
    character before it; `t1`: the frame ends by timeout, so its waiting edge is swept too"""

    def __init__(self, build, frame, index, t1, rates=RATES, atr=False):
        self.build, self.frame, self.index, self.t1, self.rates, self.atr = build, frame, index, t1, rates, atr

    def capture(self, rate, d, lead=0):
        s = self.build(rate, lead)
        if self.atr:
            s.frame(self.frame, gap=200, delays={self.index: d})
        else:
            s.frame(self.frame, gap=80, delays={self.index: d})
        s.frame([0x90, 0x00] if not self.t1 else block(0x00, 0x40, [0x90, 0x00]), gap=40)
        return s.render()

    def etu(self, rate):
        s = self.build(rate, 0)
        return s.etu


def _atr_ctx(rate, lead):
    return Session(rate, lead=lead)


def _tc1_t0(tc1):
    return lambda rate, lead: start(rate, atr_t0(tc1=tc1), lead=lead)


def _tc1_t1(tc1):
    return lambda rate, lead: start(rate, atr_t1(tc1=tc1), pps(0x11, 0x13), fi_di=(1, 3), lead=lead)


@functools.lru_cache(maxsize=None)
def contexts():
    c = {
        "atr": Context(_atr_ctx, ATR_T0, 3, False, atr=True),
        "t0_pps": Context(lambda r, l: start(r, ATR_T0, pps(0x10, 0x13), fi_di=(1, 3), lead=l), SELECT, 5, False),
    }
    for cwi in (0, 1, 5, 9):
        c["t1_cwi%d" % cwi] = Context(lambda r, l, cwi=cwi: start(r, atr_t1(bwi_cwi=0x40 | cwi), pps(0x11, 0x13), fi_di=(1, 3), lead=l),
                                      block(0x00, 0x00, [0x00, 0xA4, 0x04, 0x00]), 3, True)
    for tc1 in (0, 1, 254, 255):
        c["t0_tc1_%d" % tc1] = Context(_tc1_t0(tc1), SELECT, 5, False)
        c["t1_tc1_%d" % tc1] = Context(_tc1_t1(tc1), block(0x00, 0x00, [0x00, 0xA4, 0x04, 0x00]), 3, True)
    return c


CONTEXTS = list(contexts())
SHIFT_CONTEXTS = ("t0_pps", "t1_cwi1", "t1_tc1_255")
SHIFT_RATE = 25_000_000


def responds(rows, ctx):
    """the frame under test decodes to the bytes it was built with"""
    want = bytes(contexts()[ctx].frame).hex()
    return any(r[1] == 0x201 and r[13] == want for r in rows)


def sweep(edges, ctx, rate):
    """the delays of one context's sweep: d* - 3 ... d* + 3 of each edge plus coarse delays"""
    e = edges["%s/r%d" % (ctx, rate // 1_000_000)]
    etu = contexts()[ctx].etu(rate)
    out = {int(round(12 * etu)), int(round(20 * etu))}
    for k in ("guard", "wait"):
        if e[k] is not None:
            out |= {e[k] + j for j in range(-3, 4)}
    if e["wait"] is not None:
        out.add(int(e["wait"] * 1.5))
    return sorted(out)


# --- single cases ----------------------------------------------------------------------------------------------------------
def _atr_cases():
    out = {}
    r = 25_000_000
    for wi in (1, 10, 255):
        for after in (False, True):
            # TC2 sets CWT = WI x 960 x Di with the Di in force when the ATR is parsed; a PPS to Di 3 afterwards keeps it
            def b(wi=wi, after=after):
                s = start(r, atr_t0(tc2=wi), pps(0x10, 0x13) if after else None, fi_di=(1, 3) if after else None)
                s.frame(SELECT, gap=40)
                return s.render()
            out["atr/tc2_%d/%s" % (wi, "pps" if after else "nopps")] = b
    for wi in (1, 2):
        for late in (500, 2000):
            # TC2 in a T=1 session: CWT = WI x 960 ETU with the Di of the ATR (1), then a PPS to Di 3; a character of the
            # next block `late` ETU after the one before it
            def b(wi=wi, late=late):
                a = [0x3B, 0x80, 0x41, wi]
                s = start(r, a + [lrc(a[1:])], pps(0x11, 0x13), fi_di=(1, 3))
                s.frame(block(0x00, 0x00, [0x00, 0xA4, 0x04, 0x00]), gap=80, delays={3: int(round(late * s.etu))})
                s.frame(block(0x00, 0x40, [0x90, 0x00]), gap=40)
                return s.render()
            out["atr/tc2_t1_%d/%d" % (wi, late)] = b
    for ifsc in (4, 16, 254):
        for extra in (-1, 0, 1, 2):
            # T=1 blocks of IFSC + 3 + extra bytes (IFSC + 4 is where decodeFrameT1 cuts); the payload is truncated at 250
            def b(ifsc=ifsc, extra=extra):
                s = start(r, atr_t1(ifsc=ifsc), pps(0x11, 0x13), fi_di=(1, 3))
                n = ifsc + 3 + extra
                data = [0x00, 0x00, min(ifsc, 255)] + [(7 * i) & 0xFF for i in range(max(n - 3, 0))]
                s.frame(data[:n], gap=80)
                s.frame(block(0x00, 0x40, [0x90, 0x00]), gap=40)
                return s.render()
            out["atr/ifsc_%d/%+d" % (ifsc, extra)] = b
    for ifsc in (4, 16):
        for extra in (0, 1, 2):
            # a block whose LEN (255) never matches its size: decodeFrameT1 ends it at IFSC + 4 bytes
            def b(ifsc=ifsc, extra=extra):
                s = start(r, atr_t1(ifsc=ifsc), pps(0x11, 0x13), fi_di=(1, 3))
                s.frame([0x00, 0x00, 0xFF] + [(5 * i + 1) & 0xFF for i in range(ifsc + extra)], gap=80)
                s.frame(block(0x00, 0x40, [0x90, 0x00]), gap=40)
                return s.render()
            out["atr/ifsc_cut_%d/%+d" % (ifsc, extra)] = b
    # TD chains: T=1 -> T=15 global bytes (TA TB TC of T=15), with TCK right and wrong
    chains = {
        "t15": [0x3B, 0x80, 0x81, 0x1F, 0x03],
        "t15_full": [0x3B, 0x81, 0x80, 0x8F, 0x7F, 0x01, 0x02, 0x03, 0x0F, 0x55],
        "t1_t15": [0x3B, 0x80, 0x81, 0xB1, 0xFE, 0x45, 0x1F, 0xC3],
    }
    for name, atr in chains.items():
        for tck in ("right", "wrong"):
            def b(atr=atr, tck=tck):
                a = list(atr) + [lrc(atr[1:]) ^ (0 if tck == "right" else 0x5A)]
                s = Session(r)
                s.frame(a, gap=200)
                return s.render()
            out["atr/%s/tck_%s" % (name, tck)] = b
    # an ATR with fewer historical bytes than T0 announces and no TCK: it never completes
    def b():
        s = Session(r)
        s.frame([0x3B, 0x04, 0x41, 0x42], gap=300)
        s.frame(SELECT[:5], gap=40)
        return s.render()
    out["atr/short_history"] = b
    return out


def _pps_cases():
    out = {}
    r = 25_000_000
    for name, req, resp, fd in (("pps1_absent_0", pps(0x00), None, None), ("pps1_absent_1", pps(0x01), None, None),
                                ("pps2_pps3", pps(0x70, 0x13, 0x02, 0x00), None, (1, 3)),
                                ("no_response", pps(0x10, 0x13), False, None),
                                ("counter", pps(0x10, 0x96), pps(0x10, 0x13), (1, 3))):
        def b(req=req, resp=resp, fd=fd):
            s = start(r, ATR_T0, req, resp, fi_di=fd)
            s.frame(SELECT, gap=40)
            return s.render()
        out["pps/" + name] = b
    # every valid Fi x Di whose ETU is at least about 8 samples at 10 MS/s with a 4 MHz clock, and one below that
    r10 = 10_000_000
    for fi in (1, 2, 3, 4, 5, 6, 9, 10, 11, 12, 13):
        for di in (1, 2, 3, 4, 5, 6, 7, 8, 9):
            etu = FI[fi] / DI[di] * r10 / 4e6
            if etu < 8 and (fi, di) != (1, 6):
                continue
            if (fi + di) % 3 and (fi, di) != (1, 6):   # a third of them, to keep the golden small
                continue
            def b(fi=fi, di=di):
                p = pps(0x10, (fi << 4) | di)
                s = start(r10, ATR_T0, p, fi_di=(fi, di))
                s.frame(SELECT, gap=40)
                return s.render()
            out["pps/fidi/%x%x" % (fi, di)] = b
    # RFU Fi / Di: the reference's ETU becomes 0 or infinite; what it does next comes from its golden
    for fi, di in [(0, 3), (7, 3), (8, 3), (14, 3), (15, 3), (1, 0), (1, 10), (1, 12), (1, 15), (0, 0)]:
        def b(fi=fi, di=di):
            s = start(r10, ATR_T0, pps(0x10, (fi << 4) | di))
            s.frame(SELECT, gap=40)
            s.frame([0x90, 0x00], gap=40)
            return s.render()
        out["pps/rfu/%x%x" % (fi, di)] = b
    return out


def _err_cases():
    out = {}
    r = 25_000_000
    for etu in (1.0, 1.5, 2.0):
        for rep in (1, 2):
            def b(etu=etu, rep=rep):
                s = start(r, ATR_T0, pps(0x10, 0x13), fi_di=(1, 3))
                s.frame(SELECT, gap=40, errors={6: (etu, rep)})
                return s.render()
            out["err/signal_%g/x%d" % (etu, rep)] = b
    for k in (0, 2, 4):
        def b(k=k):
            s = start(r, atr_t1(), pps(0x11, 0x13), fi_di=(1, 3))
            blk = block(0x00, 0x00, [0x00, 0xA4, 0x04, 0x00])
            for i, v in enumerate(blk):
                s.char(v, parity_error=(i == k), at=s.starts[-1] + 12 * s.etu if i else None)
            s.wait(80)
            s.frame(block(0x00, 0x40, [0x90, 0x00]), gap=40)
            return s.render()
        out["err/t1_parity_%d" % k] = b
    return out


def _bit_cases():
    """one bit boundary moved to the decoder's sampling point of that bit + skew, in both conventions: the IO edge and
    searchSyncTime on one sample at skew 0"""
    out = {}
    for conv in ("direct", "inverse"):
        for rate in RATES:
            for k in range(-2, 3):
                def b(conv=conv, rate=rate, k=k):
                    s = Session(rate, inverse=conv == "inverse")
                    atr = [0x3F if conv == "inverse" else 0x3B, 0x12, 0x11, 0x41, 0x42]
                    s.frame(atr[:2], gap=12)
                    # TA1 = 0x11: the boundary into data bit 5 (bit 4 and bit 5 differ in both conventions)
                    st = int(round(s.starts[-1] + 12 * s.etu))
                    s.char(atr[2], at=st, skew=(5, sync_point(s, st, 5) + k))
                    s.frame(atr[3:], gap=200)
                    s.frame(SELECT[:5], gap=40)
                    return s.render()
                out["bit/%s/r%d/k%+d" % (conv, rate // 1_000_000, k)] = b
    return out


def ts_clock(s):
    """the clock frequency the decoder derives from TS (detectSync): its start bit and the falling edge 3 ETU later"""
    a = s.starts[0]
    b = int(np.ceil(a + 3 * s.etu_ts))
    return (s.rate / ((b - a) / 3.0)) * (372 / 1)


def sync_point(s, start, k):
    """the decoder's sampling sample of bit k of a character whose start bit falls at `start` (decodeSymbol /
    decodeCharacter arithmetic at the TS-derived clock, Fi 1 / Di 1)"""
    et = s.rate * 372.0 / (1 * ts_clock(s))
    half = et / 2
    sst = int(start + half)
    chr_start = int(sst - half)
    return int(chr_start + et * k + half)


def _clock_cases():
    out = {}
    r = 25_000_000
    # CLK 4.9 % and 5.1 % away from the TS clock, from the start and as a mid-session step; with and without jitter
    for off in (-0.051, -0.049, 0.049, 0.051):
        for jit in (0.0, 0.03, 0.06):
            for where in ("start", "step"):
                def b(off=off, jit=jit, where=where):
                    s = Session(r, seed=int(1000 * abs(off)) + int(100 * jit))
                    f0 = 4e6
                    if where == "start":
                        s.clk_plan = [(s.t_clk, ("run", f0 * (1 + off), jit))]
                    s.frame(ATR_T0, gap=200)
                    s.frame(pps(0x10, 0x13), gap=30).frame(pps(0x10, 0x13), gap=100).use(1, 3)
                    if where == "step":
                        s.clock(s.t, "run", f0 * (1 + off), jit)
                        s.wait(400)
                    s.use(1, 3, fclk=f0 * (1 + off))
                    s.frame(SELECT, gap=40)
                    return s.render()
                out["clk/drift/%s/%+.3f/j%g" % (where, off, jit)] = b
    # slow ramps that update the protocol several times, a frame after each stretch
    for f1 in (3.2e6, 4.8e6):
        def b(f1=f1):
            s = Session(r)
            s.frame(ATR_T0, gap=200)
            s.frame(pps(0x10, 0x13), gap=30).frame(pps(0x10, 0x13), gap=100).use(1, 3)
            a = s.t
            s.clock(a, "ramp", 4e6, f1)
            for j in range(6):
                s.wait(300)
                s.frame([0x00, 0xB0, 0x00, 0x00, 0x00], gap=40)
            s.clock(s.t, "run", f1, 0.0)
            s.wait(300).use(1, 3, fclk=f1)
            s.frame(SELECT, gap=40)
            return s.render()
        out["clk/ramp/%g" % f1] = b
    # clock stops with CLK held low or high, then a restart at another frequency
    for n in (1_000, 10_000, 100_000, 1_000_000):
        for level in (0, 1):
            def b(n=n, level=level):
                s = Session(10_000_000)
                s.frame(ATR_T0, gap=200)
                s.frame(pps(0x10, 0x13), gap=30).frame(pps(0x10, 0x13), gap=100).use(1, 3)
                s.clock(s.t, "stop", level)
                s.t += n
                s.clock(s.t, "run", 4.6e6, 0.0)
                s.wait(200).use(1, 3, fclk=4.6e6)
                s.frame(SELECT, gap=40)
                return s.render()
            out["clk/stop/%d/%s" % (n, "high" if level else "low")] = b
    return out


# the device walk's clock batch: integer CLK periods of 6 / 7 samples at 25 MS/s (63 samples per 10 clocks), the ATR's
# ETU matching it, then a step to periods whose measurements read 61, 59, 58 ... samples per 10 clocks: the 59 is the
# first that updates the protocol (63 / 59 > 1.05, 61 / 59 < 1.05), and a measurement lost or taken at the wrong place
# leaves the protocol at another clock, which shows in the next frame's frame_rate
BATCH_RATE = 25_000_000
BATCH_PATTERN = [6, 6, 7, 6, 6, 7, 6, 6, 7, 6]
BATCH_STEP = [6, 6, 6, 6, 6, 6, 6, 6, 6, 7] + [6, 6, 6, 6, 6, 6, 6, 6, 6, 5] + [6, 6, 6, 6, 6, 6, 6, 6, 5, 5]
BATCH_AFTER = [6, 6, 6, 6, 6, 6, 6, 6, 5, 5]
BATCH_K = 41


def _batch_session(k, coincide=None):
    r = BATCH_RATE
    s = Session(r, fclk=r / 6.3)
    s.clk_plan = [(s.t_clk, ("pattern", BATCH_PATTERN, 3))]
    s.frame(ATR_T0, gap=12)
    last = s.starts[-1]
    x = s.render()
    m = measurement_edges(x)
    # the walk's last step after the ATR: the decoder samples the last character's guard bit ~10.5 ETU after its start
    first = int(np.searchsorted(m, last + 10.5 * s.etu + 2))
    at = m[first + k]
    s.clock(at, "periods", BATCH_STEP, 3)
    s.clock(at + sum(BATCH_STEP), "pattern", BATCH_AFTER, 3)
    s.t = float(at + sum(BATCH_STEP) + 400 * 58 / 10)
    s.use(1, 1, fclk=r * 10 / 58)
    if coincide == "io":
        # a frame whose start bit falls on the sample of the acting measurement
        s.t = float(at + sum(BATCH_STEP[:20]) + 3 + sum(BATCH_STEP[20:]) - 10)
    s.step_at = int(at)
    s.frame(pps(0x10, 0x13), gap=30)
    return s


def _batch_cases():
    out = {}
    for k in range(BATCH_K):
        out["clk/batch/k%02d" % k] = lambda k=k: _batch_session(k).render()
    return out


def _coincide_cases():
    """a 10th CLK falling edge on the same sample as an IO edge and as a pending timer"""
    out = {}
    r = BATCH_RATE
    for what in ("io", "timer"):
        for dk in range(-1, 2):
            def b(what=what, dk=dk):
                s = Session(r, fclk=r / 6.3)
                s.clk_plan = [(s.t_clk, ("pattern", BATCH_PATTERN, 3))]
                s.frame(ATR_T0[:2], gap=12)
                x = s.render(tail=5e-3)
                m = measurement_edges(x)
                if what == "io":
                    # the next character's start bit on a measurement edge
                    target = m[np.searchsorted(m, s.starts[-1] + 12 * s.etu)] + dk
                    s.frame(ATR_T0[2:], gap=200, delays={0: int(target - s.starts[-1])})
                else:
                    # a measurement edge on the sampling sample of bit 4 of the next character: shift the character
                    st = s.starts[-1] + 12 * s.etu
                    sp = sync_point(s, int(round(st)), 4)
                    j = np.searchsorted(m, sp)
                    s.frame(ATR_T0[2:], gap=200, delays={0: int(round(st)) + int(m[j] - sp) + dk - s.starts[-1]})
                s.frame(SELECT[:5], gap=40)
                return s.render()
            out["clk/coincide/%s/%+d" % (what, dk)] = b
    return out


@functools.lru_cache(maxsize=None)
def _singles():
    out = {}
    for f in (_atr_cases, _pps_cases, _err_cases, _bit_cases, _clock_cases, _batch_cases, _coincide_cases):
        out.update(f())
    return out


# --- case list -------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def golden():
    with lzma.open(GOLDEN, "rt") as f:
        return json.load(f)


def edges():
    return golden()["edges"]


def edge_name(ctx, rate, d):
    return "edge/%s/r%d/d%d" % (ctx, rate // 1_000_000, d)


def builders(edge_table=None):
    """name -> () -> capture, for every case (the edge sweeps need the recorded edge delays)"""
    e = edge_table if edge_table is not None else edges()
    out = {}
    for ctx, c in contexts().items():
        for rate in c.rates:
            for d in sweep(e, ctx, rate):
                out[edge_name(ctx, rate, d)] = lambda c=c, rate=rate, d=d: c.capture(rate, d)
    for ctx in SHIFT_CONTEXTS:
        g = e["%s/r%d" % (ctx, SHIFT_RATE // 1_000_000)]
        for kind in ("guard", "wait"):
            if g[kind] is None:
                continue
            for d in (g[kind] - 1, g[kind], g[kind] + 1):
                for sh in range(32):
                    out["shift/%s/%s/d%d/s%d" % (ctx, kind, d, sh)] = lambda ctx=ctx, d=d, sh=sh: contexts()[ctx].capture(SHIFT_RATE, d, lead=sh)
    out.update(_singles())
    return out


def rate_of(name):
    if name.startswith(("edge/", "bit/")):
        return int(name.split("/r")[1].split("/")[0]) * 1_000_000
    if name.startswith("shift/") or name.startswith("clk/batch") or name.startswith("clk/coincide"):
        return SHIFT_RATE
    if name.startswith("pps/fidi") or name.startswith("pps/rfu") or name.startswith("clk/stop"):
        return 10_000_000
    return 25_000_000


def family(name):
    """the batch a case goes in: its first two name parts and its rate"""
    p = name.split("/")
    return "%s/%s/r%d" % (p[0], p[1], rate_of(name) // 1_000_000)


@functools.lru_cache(maxsize=None)
def names():
    return sorted(builders())


@functools.lru_cache(maxsize=64)
def case(name):
    return builders()[name]()


def families():
    out = {}
    for n in names():
        out.setdefault(family(n), []).append(n)
    return out


def padded(x, n):
    """x padded to n samples with its last sample, as a batch holds it"""
    return np.concatenate([x, np.repeat(x[-1:], n - len(x), axis=0)]) if n > len(x) else x


def key(x, rate):
    h = hashlib.sha256(np.ascontiguousarray(x, dtype=np.float32).tobytes())
    h.update(b"%d/%d" % (rate, STREAM_TIME))
    return h.hexdigest()[:24]


def stream_cuts(name, x, rows):
    """buffer ends for the stream push: at d* - 1, d*, d* + 1 samples after the swept character's predecessor, i.e. at
    and around the start bit of an edge case's swept character, and on the sample of the first acting clock measurement
    of a batch case"""
    if name.startswith("edge/"):
        ctx = name.split("/")[1]
        e = edges()["%s/r%d" % (ctx, rate_of(name) // 1_000_000)]
        io = np.asarray(x)[:, 0]
        falls = np.flatnonzero(np.diff(io, prepend=np.float32(0)) < 0)
        d = int(name.rsplit("/d", 1)[1])
        base = [f for f in falls if f + d < len(x) and io[f + d] == 0 and (f + d) in set(falls)]
        out = []
        for k in ("guard", "wait"):
            if e[k] is not None and base:
                out += [base[-1] + e[k] + j for j in (-1, 0, 1)]
        return sorted(c for c in set(out) if 0 < c < len(x))
    if name.startswith("clk/batch"):
        # the step's measurements: the acting one is among them
        m = measurement_edges(x)
        at = _batch_session(int(name.rsplit("k", 1)[1])).step_at
        return [int(c) for c in m[np.searchsorted(m, at):][:5]]
    return []


def chunk_plans(name, x):
    """name -> chunk lengths: the whole capture, 65 536-sample buffers and, where the case has them, cuts at its edges"""
    n = len(x)
    out = {"whole": [n], "p65536": [65_536] * (n // 65_536) + ([n % 65_536] if n % 65_536 else [])}
    cuts = stream_cuts(name, x, None)
    if cuts:
        pts = [0] + cuts + [n]
        out["cuts"] = [b - a for a, b in zip(pts[:-1], pts[1:]) if b > a]
    return out
