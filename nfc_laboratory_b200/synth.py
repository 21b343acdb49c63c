"""Synthetic NFC capture streams for the benchmark configs of BASELINE.json (SURVEY.md Appendix B recipes).

Every recipe is validated against the compiled reference decoder in tests/test_synth.py: the frames the generator
intends are exactly the frames the reference decodes.  Signals are built in the magnitude domain as a modulation
factor m[n] on a carrier of amplitude A, then wrapped as IQ:  I = A m cos(phi), Q = A m sin(phi), plus Gaussian noise
per component (noise is mandatory: the noise-free signal has exact plateaus and ties, SURVEY.md section 7).

numpy builds the (small) exchange templates; torch assembles the batch on any device.
"""
import numpy as np

FC = 13.56e6


# ---------------------------------------------------------------------------------------------------------------------
# checksums
# ---------------------------------------------------------------------------------------------------------------------
def _crc16_refl(data, init):
    crc = init
    for b in data:
        crc ^= b
        for _ in range(8):
            crc = (crc >> 1) ^ 0x8408 if crc & 1 else crc >> 1
    return crc & 0xFFFF


def crc_a(data):
    c = _crc16_refl(data, 0x6363)
    return bytes([c & 0xFF, c >> 8])


def crc_b(data):
    c = _crc16_refl(data, 0xFFFF) ^ 0xFFFF
    return bytes([c & 0xFF, c >> 8])


def crc_f(data):
    crc = 0
    for b in data:
        crc ^= b << 8
        for _ in range(8):
            crc = ((crc << 1) ^ 0x1021) & 0xFFFF if crc & 0x8000 else (crc << 1) & 0xFFFF
    return bytes([crc >> 8, crc & 0xFF])


def _odd_parity(b):
    return 1 ^ (bin(b).count("1") & 1)


# ---------------------------------------------------------------------------------------------------------------------
# waveform rendering: a list of (t_start, t_end, level) intervals in units of 1/fc, sampled at fs
# ---------------------------------------------------------------------------------------------------------------------
class Wave:
    def __init__(self, fs):
        self.fs = fs
        self.iv = []  # (t0, t1, level) in 1/fc units; level multiplies the carrier; default 1.0
        self.sub = []  # (t0, t1, depth, phase) sub-carrier bursts: level -= depth * sq(t), sq in {0,1}, period 16/fc
        self.t = 0.0

    def low(self, t0, t1, level):
        self.iv.append((t0, t1, level))

    def burst(self, t0, t1, depth, inverted=False):
        self.sub.append((t0, t1, depth, inverted))

    def render(self, t_end, pad_before=0.0):
        n = int(np.ceil((t_end + pad_before) * self.fs / FC))
        t = (np.arange(n, dtype=np.float64) * FC / self.fs) - pad_before
        m = np.ones(n, dtype=np.float64)
        for (t0, t1, lv) in self.iv:
            m[(t >= t0) & (t < t1)] = lv
        for (t0, t1, depth, inv) in self.sub:
            sel = (t >= t0) & (t < t1)
            ph = np.floor((t[sel] - t0) / 8.0).astype(np.int64) & 1  # half period = 8/fc
            sq = (ph == (1 if inv else 0)).astype(np.float64)
            m[sel] -= depth * sq
        return m.astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------------
# NFC-A
# ---------------------------------------------------------------------------------------------------------------------
def nfca_poll(w, t0, data, rate=0, short=False, depth=0.98):
    """modified Miller poll frame starting at t0 (1/fc).  Returns (t_end_of_last_pause_rising_edge, last_bit)"""
    T = 128 >> rate
    pw = 32 if rate == 0 else (20 if rate == 1 else 10)
    bits = []
    if short:
        bits = [(data[0] >> i) & 1 for i in range(7)]
    else:
        for b in data:
            bits += [(b >> i) & 1 for i in range(8)] + [_odd_parity(b)]
    lv = 1.0 - depth
    t = t0
    w.low(t, t + pw, lv)  # SOF: pattern Z
    last_rise = t + pw
    t += T
    prev = 0  # SOF counts as a logic 0 for the next symbol
    for b in bits:
        if b:
            w.low(t + T / 2, t + T / 2 + pw, lv)  # X
            last_rise = t + T / 2 + pw
        elif prev == 0:
            w.low(t, t + pw, lv)  # Z
            last_rise = t + pw
        # else Y: no pause
        prev = b
        t += T
    # end of communication: logic 0 followed by Y
    if prev == 0:
        w.low(t, t + pw, lv)
        last_rise = t + pw
    t += 2 * T
    return last_rise, (bits[-1] if bits else 0), t


def nfca_listen_106(w, t0, data, short4=False, depth=0.08):
    """Manchester sub-carrier listen frame at 106k starting at t0"""
    T = 128
    bits = [1]  # SOF
    if short4:
        bits += [(data[0] >> i) & 1 for i in range(4)]
    else:
        for b in data:
            bits += [(b >> i) & 1 for i in range(8)] + [_odd_parity(b)]
    t = t0
    for b in bits:
        if b:
            w.burst(t, t + T / 2, depth)
        else:
            w.burst(t + T / 2, t + T, depth)
        t += T
    return t


def nfca_listen_bpsk(w, t0, data, rate, depth=0.10):
    """BPSK sub-carrier listen frame at 212 / 424k: 32 cycles reference phase, start bit inverted, NRZ-L data"""
    T = 128 >> rate
    t = t0
    w.burst(t, t + 32 * 16, depth)
    t += 32 * 16
    bits = [0]
    for i, b in enumerate(data):
        par = _odd_parity(b)
        if i == len(data) - 1:
            par ^= 1  # last parity bit inverted (ISO 14443-3 high rate PICC->PCD; NfcA.cpp:728-735)
        bits += [(b >> k) & 1 for k in range(8)] + [par]
    for b in bits:
        w.burst(t, t + T, depth, inverted=(b == 0))
        t += T
    return t


def nfca_exchange(fs, poll, listen, rate=0, short=False, short4=False, lead=4000.0):
    """one poll / listen exchange; returns (modulation array, description)"""
    w = Wave(fs)
    last_rise, last_bit, t = nfca_poll(w, lead, poll, rate, short)
    if listen is not None:
        fdt = 1236 if last_bit else 1172
        ts = last_rise + fdt
        if rate == 0:
            t = nfca_listen_106(w, ts, listen, short4)
        else:
            t = nfca_listen_bpsk(w, ts, listen, rate)
    return w.render(t + lead)


# ---------------------------------------------------------------------------------------------------------------------
# NFC-B
# ---------------------------------------------------------------------------------------------------------------------
def _nfcb_chars(data):
    bits = []
    for b in data:
        bits += [0] + [(b >> k) & 1 for k in range(8)] + [1]
    return bits


def nfcb_poll(w, t0, data, depth=0.12):
    T = 128
    lv = 1.0 - depth
    t = t0
    w.low(t, t + 10.5 * T, lv)  # SOF: 10.5 ETU low, 2.5 ETU high
    t += 13 * T
    for b in _nfcb_chars(data + crc_b(data)):
        if not b:
            w.low(t, t + T, lv)
        t += T
    w.low(t, t + 10.5 * T, lv)  # EOF
    t += 10.5 * T
    return t


def nfcb_listen(w, t0, data, depth=0.08):
    T = 128
    t = t0
    w.burst(t, t + 80 * 16, depth)  # TR1: unmodulated sub-carrier, reference phase
    t += 80 * 16
    w.burst(t, t + 10.5 * T, depth, inverted=True)  # SOF low
    t += 10.5 * T
    w.burst(t, t + 2.5 * T, depth)
    t += 2.5 * T
    for b in _nfcb_chars(data + crc_b(data)):
        w.burst(t, t + T, depth, inverted=(b == 0))
        t += T
    w.burst(t, t + 10.5 * T, depth, inverted=True)  # EOF
    t += 10.5 * T
    w.burst(t, t + T, depth)
    t += T
    return t


def nfcb_exchange(fs, poll, listen, lead=4000.0):
    w = Wave(fs)
    t = nfcb_poll(w, lead, poll)
    if listen is not None:
        ts = t + 1024 + 200 * FC / fs
        t = nfcb_listen(w, ts, listen)
    return w.render(t + lead)


# ---------------------------------------------------------------------------------------------------------------------
# NFC-F
# ---------------------------------------------------------------------------------------------------------------------
def nfcf_poll(w, t0, payload, rate=1, depth=0.40):
    """FeliCa poll: 48 zero bits, sync B24D, LEN, payload, CRC; Manchester, bit 1 = high-then-low; MSB first"""
    H = (64 >> rate)  # half bit in 1/fc
    lv = 1.0 - depth
    body = bytes([len(payload) + 1]) + payload
    data = bytes(6) + b"\xB2\x4D" + body + crc_f(body)
    t = t0
    for b in data:
        for k in range(7, -1, -1):
            bit = (b >> k) & 1
            if bit:
                w.low(t + H, t + 2 * H, lv)
            else:
                w.low(t, t + H, lv)
            t += 2 * H
    return t


def nfcf_exchange(fs, payload, rate=1, lead=4000.0):
    w = Wave(fs)
    t = nfcf_poll(w, lead, payload, rate)
    return w.render(t + lead)


# ---------------------------------------------------------------------------------------------------------------------
# NFC-V
# ---------------------------------------------------------------------------------------------------------------------
def nfcv_poll(w, t0, data, depth=0.98):
    """ISO 15693 1-of-4 poll: slot = 128/fc; SOF pauses at slots 0 and 5 of 8; byte = 4 symbols of 8 slots"""
    U = 128
    lv = 1.0 - depth
    c = _crc16_refl(data, 0xFFFF) ^ 0xFFFF
    frame = data + bytes([c & 0xFF, c >> 8])
    t = t0
    w.low(t, t + U, lv)
    w.low(t + 5 * U, t + 6 * U, lv)
    t += 8 * U
    for b in frame:
        for k in range(4):
            v = (b >> (2 * k)) & 3
            w.low(t + (2 * v + 1) * U, t + (2 * v + 2) * U, lv)
            t += 8 * U
    w.low(t + 2 * U, t + 3 * U, lv)  # EOF
    t += 4 * U
    return t


def nfcv_exchange(fs, data, lead=4000.0):
    w = Wave(fs)
    t = nfcv_poll(w, lead, data)
    return w.render(t + lead)


# ---------------------------------------------------------------------------------------------------------------------
# sessions for the benchmark configs
# ---------------------------------------------------------------------------------------------------------------------
def session_templates(config, fs=10_000_000):
    """list of (modulation array, expected frames) for one config; expected = [(type, bytes)] with type 0x102 / 0x103"""
    uid = bytes([0x08, 0x12, 0x34, 0x56])
    bcc = bytes([uid[0] ^ uid[1] ^ uid[2] ^ uid[3]])
    T = []
    if config == "nfca106":
        sel = bytes([0x93, 0x70]) + uid + bcc
        T.append((nfca_exchange(fs, b"\x26", b"\x04\x00", short=True), [(0x102, b"\x26"), (0x103, b"\x04\x00")]))
        T.append((nfca_exchange(fs, b"\x93\x20", uid + bcc), [(0x102, b"\x93\x20"), (0x103, uid + bcc)]))
        T.append((nfca_exchange(fs, sel + crc_a(sel), b"\x20" + crc_a(b"\x20")), [(0x102, sel + crc_a(sel)), (0x103, b"\x20" + crc_a(b"\x20"))]))
        for blk in (bytes([0x02, 0x00, 0xA4, 0x04, 0x00, 0x07, 0xD2, 0x76, 0x00, 0x00, 0x85, 0x01, 0x01, 0x00]), bytes([0x03, 0x00, 0xB0, 0x00, 0x00, 0x0F])):
            rsp = bytes([blk[0], 0x90, 0x00])
            T.append((nfca_exchange(fs, blk + crc_a(blk), rsp + crc_a(rsp)), [(0x102, blk + crc_a(blk)), (0x103, rsp + crc_a(rsp))]))
        T.append((nfca_exchange(fs, b"\x50\x00" + crc_a(b"\x50\x00"), None), [(0x102, b"\x50\x00" + crc_a(b"\x50\x00"))]))
    elif config == "nfcb106":
        reqb = bytes([0x05, 0x00, 0x00])
        atqb = bytes([0x50, 0x11, 0x22, 0x33, 0x44, 0x00, 0x00, 0x00, 0x00, 0x00, 0x81, 0x81])
        attrib = bytes([0x1D, 0x11, 0x22, 0x33, 0x44, 0x00, 0x08, 0x01, 0x00])
        T.append((nfcb_exchange(fs, reqb, atqb), [(0x102, reqb + crc_b(reqb)), (0x103, atqb + crc_b(atqb))]))
        T.append((nfcb_exchange(fs, attrib, b"\x00"), [(0x102, attrib + crc_b(attrib)), (0x103, b"\x00" + crc_b(b"\x00"))]))
    elif config == "nfca424":
        blk = bytes([0x02, 0x00, 0xA4, 0x04, 0x00])
        rsp = bytes([0x02, 0x90, 0x00])
        T.append((nfca_exchange(fs, blk + crc_a(blk), rsp + crc_a(rsp), rate=2), [(0x102, blk + crc_a(blk)), (0x103, rsp + crc_a(rsp))]))
    elif config == "mixed":
        reqb = bytes([0x05, 0x00, 0x00])
        reqc = bytes([0x00, 0xFF, 0xFF, 0x00, 0x00])
        inv = bytes([0x26, 0x01, 0x00])
        T.append((nfca_exchange(fs, b"\x26", None, short=True), [(0x102, b"\x26")]))
        T.append((nfcb_exchange(fs, reqb, None), [(0x102, reqb + crc_b(reqb))]))
        T.append((nfcf_exchange(fs, reqc, rate=1), None))
        T.append((nfcf_exchange(fs, reqc, rate=2), None))
        T.append((nfcv_exchange(fs, inv), None))
    else:
        raise ValueError(config)
    return T


def schedule(config, n_streams, n_samples, seed, fs=10_000_000, gap_ms=(1.0, 5.0), first_gap=30000):
    """per-stream placement of exchange templates: arrays (stream, position, template id); deterministic in seed"""
    tmpl = session_templates(config, fs)
    lens = np.array([t[0].size for t in tmpl])
    rng = np.random.default_rng(seed)
    # the longest listen time-out after a poll without response must fit into the gap (FWT, 48330 samples at 10 MS/s)
    lo, hi = int(gap_ms[0] * fs / 1000), int(gap_ms[1] * fs / 1000)
    if config == "mixed":
        lo, hi = 60000, 120000
    places = []
    for s in range(n_streams):
        pos = first_gap + int(rng.integers(0, hi))
        k = int(rng.integers(0, len(tmpl)))
        while pos + lens[k] + 2048 < n_samples:
            places.append((s, pos, k))
            pos += int(lens[k]) + int(rng.integers(lo, hi + 1))
            k = (k + 1) % len(tmpl)
    return tmpl, np.array(places, dtype=np.int64).reshape(-1, 3)


# configs whose schedule alone fixes the frame count (checked against the reference in tests/test_synth.py, and on all
# 1024 x 1e7 streams of the benchmark batch).  Not among them: NFC-B (the reference misses exchanges that come within the
# first ~90 000 samples of a stream) and NFC-A 424 kbps (it loses an occasional BPSK listen frame to the noise).
SCHEDULE_FIXES_FRAME_COUNT = ("nfca106",)


def expected_frame_count(config, n_streams, n_samples, seed, fs=10_000_000):
    """number of poll + listen frames the batch of synth_batch(config, n_streams, n_samples, seed) is built to contain
    (every placed exchange is complete), or None when the config gives no such guarantee"""
    if config not in SCHEDULE_FIXES_FRAME_COUNT:
        return None
    tmpl, places = schedule(config, n_streams, n_samples, seed, fs)
    per = [None if t[1] is None else len(t[1]) for t in tmpl]
    if any(p is None for p in per):
        return None
    return int(sum(per[int(k)] for k in places[:, 2])) if places.size else 0


def expected_frames_per_stream(config, n_streams, n_samples, seed, fs=10_000_000):
    """per-stream version of expected_frame_count: int64 array [n_streams], or None"""
    if config not in SCHEDULE_FIXES_FRAME_COUNT:
        return None
    tmpl, places = schedule(config, n_streams, n_samples, seed, fs)
    per = [None if t[1] is None else len(t[1]) for t in tmpl]
    if any(p is None for p in per):
        return None
    out = np.zeros(n_streams, dtype=np.int64)
    if places.size:
        np.add.at(out, places[:, 0], np.array(per, dtype=np.int64)[places[:, 2]])
    return out


def synth_batch(config, n_streams, n_samples, seed=1, device="cpu", fs=10_000_000, iq=True, amplitude=(0.25, 0.40), sigma=(1e-3, 4e-3),
                chunk_streams=32, out=None):
    """[n_streams, n_samples, 2] float32 IQ (or [n_streams, n_samples] magnitude when iq=False) on `device`.

    Noise is drawn with torch's generator for `device`: CPU and CUDA draws differ, so cross-device comparisons copy the
    generated tensor instead of regenerating it."""
    import torch

    tmpl, places = schedule(config, n_streams, n_samples, seed, fs)
    rng = np.random.default_rng(seed + 7919)
    A = rng.uniform(amplitude[0], amplitude[1], n_streams).astype(np.float32)
    sg = np.exp(rng.uniform(np.log(sigma[0]), np.log(sigma[1]), n_streams)).astype(np.float32)
    phi0 = rng.uniform(0, 2 * np.pi, n_streams).astype(np.float32)
    drift = rng.normal(0, 2e-7, n_streams).astype(np.float32)  # rad / sample: slow phase drift

    dev = torch.device(device)
    tt = [torch.from_numpy(t[0]).to(dev) for t in tmpl]
    shape = (n_streams, n_samples, 2) if iq else (n_streams, n_samples)
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=dev)
    gen = torch.Generator(device=dev)
    n_idx = torch.arange(n_samples, device=dev, dtype=torch.float32)

    for s0 in range(0, n_streams, chunk_streams):
        s1 = min(n_streams, s0 + chunk_streams)
        m = torch.ones((s1 - s0, n_samples), dtype=torch.float32, device=dev)
        sel = places[(places[:, 0] >= s0) & (places[:, 0] < s1)]
        for k in range(len(tmpl)):
            pk = sel[sel[:, 2] == k]
            if pk.size == 0:
                continue
            L = tt[k].numel()
            rows = torch.from_numpy(pk[:, 0] - s0).to(dev)
            cols = torch.from_numpy(pk[:, 1]).to(dev)
            idx = cols[:, None] + torch.arange(L, device=dev)[None, :]
            m[rows[:, None].expand_as(idx), idx] = tt[k][None, :].expand(idx.shape[0], L)
        a = torch.from_numpy(A[s0:s1]).to(dev)[:, None]
        x = m * a
        gen.manual_seed(seed * 1000003 + s0)
        if iq:
            ph = torch.from_numpy(phi0[s0:s1]).to(dev)[:, None] + torch.from_numpy(drift[s0:s1]).to(dev)[:, None] * n_idx[None, :]
            sgm = torch.from_numpy(sg[s0:s1]).to(dev)[:, None]
            out[s0:s1, :, 0] = x * torch.cos(ph) + sgm * torch.randn(x.shape, generator=gen, device=dev)
            out[s0:s1, :, 1] = x * torch.sin(ph) + sgm * torch.randn(x.shape, generator=gen, device=dev)
        else:
            sgm = torch.from_numpy(sg[s0:s1]).to(dev)[:, None]
            out[s0:s1] = (x + sgm * torch.randn(x.shape, generator=gen, device=dev)).abs()
    return out


# ---------------------------------------------------------------------------------------------------------------------
# ISO 7816 contact smart-card captures: 4 logic channels IO, CLK, RST, VCC (the reference's logic capture layout)
# ---------------------------------------------------------------------------------------------------------------------
ISO_SCENARIOS = ("t0_direct", "t0_inverse", "t1_lrc", "t1_crc", "warm_reset")


def _iso_lrc(data):
    x = 0
    for b in data:
        x ^= b
    return x


class _IsoLine:
    """a capture under construction: times in seconds, IO as a list of low intervals, an ETU in seconds"""

    def __init__(self, rng, clock_hz, inverse):
        self.rng = rng
        self.clock = clock_hz
        self.inverse = inverse
        self.etu = 372.0 / clock_hz
        self.low = []           # IO low intervals (t0, t1)
        self.t = 0.0

    def char(self, byte, parity_error=False, error_signal=False):
        """one character from self.t: start bit, 8 data bits, even parity; the receiver's error signal when asked"""
        bits = [(byte >> i) & 1 for i in (range(7, -1, -1) if self.inverse else range(8))]
        par = (bin(byte).count("1") & 1) ^ (1 if parity_error else 0)
        levels = [0] + [(1 - b) if self.inverse else b for b in bits] + [(1 - par) if self.inverse else par]
        for k, lv in enumerate(levels):
            if lv == 0:
                self.low.append((self.t + k * self.etu, self.t + (k + 1) * self.etu))
        if error_signal:
            self.low.append((self.t + 10.2 * self.etu, self.t + 11.7 * self.etu))
            self.t += 14 * self.etu
        else:
            self.t += (12 + self.rng.uniform(0.0, 0.6)) * self.etu

    def frame(self, data, gap_etu=20.0, bad=None):
        """bytes back to back; index `bad` goes out once with a parity error, is refused and repeated"""
        for i, b in enumerate(data):
            if i == bad:
                self.char(b, parity_error=True, error_signal=True)
            self.char(b)
        self.t += gap_etu * self.etu


def iso7816_capture(scenario, rate, seed=1, glitches=True):
    """one seeded capture [n, 4] float32 (IO, CLK, RST, VCC as 0 / 1): power-up, clock, reset, ATR and an exchange.

    t0_direct   direct-convention ATR, PPS to Fi 1 / Di 3, T=0 TPDUs with NULL and ACK procedure bytes, one character
                with a parity error that the receiver signals and the sender repeats, a clock change of more than 5 %
    t0_inverse  the same in the inverse convention
    t1_lrc      ATR announcing T=1, PPS to T=1, I / R / S blocks with an LRC epilogue
    t1_crc      the same blocks with a CRC epilogue (the reference decodes with the LRC rule: its ATR parser never
                selects CRC)
    warm_reset  a T=0 session, RST low mid-capture, a second ATR
    Every capture ends with power-off.  `glitches` adds one-sample pulses on IO (before the reset) and on CLK."""
    rng = np.random.default_rng(seed)
    clock1 = float(rng.choice([3.5712e6, 4.0e6, 2.5e6]))
    clock2 = clock1 * float(rng.choice([0.85, 1.12]))
    line = _IsoLine(rng, clock1, scenario == "t0_inverse")
    t_vcc = 20e-6
    t_clk = t_vcc + 5e-6
    t_rst = t_clk + 500 / clock1
    line.t = t_rst + 600 / clock1
    t_chg = None
    rst_low = []

    if scenario.startswith("t1"):
        atr = [0x3B, 0x91, 0x13, 0x81, 0x31, 0xFE, 0x45, 0x4A]      # TA1 TD1(T=1) TD2 TA3(IFSC) TB3(BWI/CWI) + 1 hist
        atr.append(_iso_lrc(atr[1:]))
    elif scenario == "t0_inverse":
        atr = [0x3F, 0x12, 0x11, 0x41, 0x42]
    else:
        atr = [0x3B, 0x12, 0x11, 0x41, 0x42]
    line.frame(atr, gap_etu=200)

    t1 = scenario.startswith("t1")
    pps = [0xFF, 0x11 if t1 else 0x10, 0x13]
    pps.append(_iso_lrc(pps))
    line.frame(pps, gap_etu=30)
    line.frame(pps, gap_etu=100)
    line.etu = 372.0 / 4 / line.clock

    if t1:
        crc = scenario == "t1_crc"

        def block(nad, pcb, inf):
            b = [nad, pcb, len(inf)] + list(inf)
            if crc:
                c = _crc16_refl(b, 0xFFFF) ^ 0xFFFF
                return b + [c & 0xFF, c >> 8]
            return b + [_iso_lrc(b)]

        for blk in (block(0x00, 0x00, [0x00, 0xA4, 0x04, 0x00]), block(0x00, 0x00, [0x90, 0x00]),
                    block(0x00, 0x91, []), block(0x00, 0xC1, [0xFE]), block(0x00, 0xE1, [0xFE]),
                    block(0x00, 0x40, [0x00, 0xB0, 0x00, 0x00, 0x04]), block(0x00, 0x40, [0x01, 0x02, 0x03, 0x04, 0x90, 0x00])):
            line.frame(blk, gap_etu=80)
        t_chg = line.t
        line.clock = clock2
        line.etu = 372.0 / 4 / clock2
        line.t += 400 * line.etu
        line.frame(block(0x00, 0x00, [0x00, 0x84, 0x00, 0x00, 0x08]), gap_etu=80)
    else:
        # SELECT with an ACK procedure byte, one character repeated after a parity error
        line.frame([0x00, 0xA4, 0x04, 0x00, 0x02, 0xA4, 0x3F, 0x00, 0x90, 0x00], gap_etu=40, bad=6)
        # GET CHALLENGE with a NULL procedure byte, then per-byte ACKs (INS ^ 0xFF)
        line.frame([0x00, 0x84, 0x00, 0x00, 0x02, 0x60, 0x84, 0x11, 0x22, 0x90, 0x00], gap_etu=40)
        line.frame([0x80, 0xCA, 0x9F, 0x7F, 0x01, 0x35, 0x55, 0x61, 0x05], gap_etu=40)
        t_chg = line.t
        line.clock = clock2
        line.etu = 372.0 / 4 / clock2
        line.t += 400 * line.etu
        line.frame([0x00, 0xB0, 0x00, 0x00, 0x02, 0xB0, 0xAA, 0xBB, 0x90, 0x00], gap_etu=200)
        if scenario == "warm_reset":
            rst_low.append((line.t, line.t + 300 / line.clock))
            line.t += 300 / line.clock + 600 / line.clock
            line.etu = 372.0 / line.clock
            line.frame([0x3B, 0x00], gap_etu=100)
            line.frame([0x00, 0xA4, 0x04, 0x00, 0x02, 0xA4, 0x3F, 0x00, 0x90, 0x00], gap_etu=100)

    t_off = line.t + 100e-6
    n = int((t_off + 30e-6) * rate)
    t = np.arange(n, dtype=np.float64) / rate
    vcc = ((t >= t_vcc) & (t < t_off)).astype(np.float32)
    rst = ((t >= t_rst) & (t < t_off)).astype(np.float32)
    for a, b in rst_low:
        rst[(t >= a) & (t < b)] = 0
    phase = np.where(t < t_chg, (t - t_clk) * clock1, (t_chg - t_clk) * clock1 + (t - t_chg) * clock2)
    clk = (((phase % 1.0) < 0.5) & (t >= t_clk) & (t < t_off - 10e-6)).astype(np.float32)
    io = ((t >= t_vcc + 2e-6) & (t < t_off)).astype(np.float32)
    for a, b in line.low:
        io[(t >= a) & (t < b)] = 0
    if glitches:
        # IO glitches before the reset: a glitch inside a T=0 session starts a character that swallows the session
        # (a frame then ends only after CWT = 9600 ETU)
        idle = np.flatnonzero((io[1:-1] == 1) & (io[:-2] == 1) & (io[2:] == 1) & (t[1:-1] < t_rst)) + 1
        for i in rng.choice(idle, size=min(3, idle.size), replace=False):
            io[i] = 0
        for i in rng.integers(int(t_clk * rate) + 10, n - 10, size=3):
            clk[i] = 1 - clk[i]
    return np.stack([io, clk, rst, vcc], axis=1)
