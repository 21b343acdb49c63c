"""ISO 7816 contact smart-card decoding of 4-channel logic captures (nfcb200_iso7816_decode_batch, csrc/iso_core.h).

CPU: the host build of the event walk against the recorded reference output on every field and the payload, and
against the live reference where oracle/_ref/libnfcref_iso.so was built.
GPU: the device against the recorded output, int16 against float input, host against device input, a stream alone
against the same stream in a batch, every error path and the capacity path, and that the call leaves the NFC decode
state of the handle alone."""
import numpy as np
import pytest

import iso_ref as R
import nfcutil as U
import nfc_laboratory_b200 as N

CASE_IDS = ["%s-%dM" % (sc, rate // 1_000_000) for sc, rate in R.CASES]


@pytest.mark.parametrize("scenario,rate", R.CASES, ids=CASE_IDS)
def test_host_equals_golden(scenario, rate):
    x = R.capture(scenario, rate)
    assert R.host(x, rate) == R.expected(x, rate)


@pytest.mark.parametrize("scenario,rate", R.CASES, ids=CASE_IDS)
def test_host_equals_live_oracle(scenario, rate):
    if R.ref_lib() is None:
        pytest.skip("the reference oracle was not built (oracle/iso.mk needs the reference sources)")
    x = R.capture(scenario, rate)
    assert R.host(x, rate) == R.ref(x, rate)


CLOCK_IDS = ["%s-%dM-%s" % c for c in [(sc, rate // 1_000_000, kind) for sc, rate, kind in R.CLOCK_CASES]]


@pytest.mark.parametrize("scenario,rate,kind", R.CLOCK_CASES, ids=CLOCK_IDS)
def test_host_equals_golden_multilevel_clock(scenario, rate, kind):
    x = R.clock_capture(scenario, rate, kind)
    assert R.host(x, rate) == R.expected(x, rate)


@pytest.mark.parametrize("scenario,rate,kind", R.CLOCK_CASES, ids=CLOCK_IDS)
def test_host_equals_live_oracle_multilevel_clock(scenario, rate, kind):
    if R.ref_lib() is None:
        pytest.skip("the reference oracle was not built (oracle/iso.mk needs the reference sources)")
    x = R.clock_capture(scenario, rate, kind)
    assert R.host(x, rate) == R.ref(x, rate)


def test_library_exports_the_entry_point():
    """the library loads without a GPU and exports the ISO 7816 entry point the header declares"""
    header = open(R.os.path.join(R.ROOT, "include", "nfcb200.h")).read()
    assert "int nfcb200_iso7816_decode_batch(" in header
    assert hasattr(R.C.CDLL(N.library_path()), "nfcb200_iso7816_decode_batch")
    assert (N.SIG_LOGIC_F32, N.SIG_LOGIC_S16) == (5, 6)


def test_golden_covers_the_protocol():
    """the recorded captures exercise what the generator promises: both conventions, PPS, T=0, T=1, parity errors,
    CRC errors, power-off and the reset lines"""
    frames = [f for v in R.golden().values() for f in v]
    types = {f[2] for f in frames}
    assert {0x200, 0x201, 0x202, 0x203, 0x210, 0x211, 0x212, 0x213} <= types
    atrs = {f[13][:2] for f in frames if f[2] == 0x210}
    assert {"3b", "3f"} <= atrs
    flags = {f[3] for f in frames}
    assert any(fl & 0x20 for fl in flags)
    rates = {f[5] for f in frames if f[1] == 0x201}
    assert len(rates) >= 3  # default ETU, after PPS, after the clock change


def _s16(x):
    return (np.asarray(x) * 32767).astype(np.int16)


def _falls_per_tile(x):
    clk = np.asarray(x, dtype=np.float32)[:, 1]
    falls = np.diff(clk, prepend=np.float32(0)) < 0
    return np.add.reduceat(falls, np.arange(0, len(falls), 4096))


@pytest.fixture(scope="module")
def dec():
    d = N.NfcDecoder(device=0)
    d.setStreamTime(R.STREAM_TIME)
    yield d
    d.close()


def _decode(d, x, rate, sigtype=N.SIG_LOGIC_F32):
    buf, n = d.iso7816_decode(x, sigtype, rate, raw=True)
    return R.rows(buf, n)


@pytest.mark.gpu
@pytest.mark.parametrize("scenario,rate", R.CASES, ids=CASE_IDS)
def test_device_equals_golden(dec, scenario, rate):
    x = R.capture(scenario, rate)
    assert _decode(dec, x, rate) == R.expected(x, rate)


@pytest.mark.gpu
@pytest.mark.parametrize("scenario", R.S.ISO_SCENARIOS)
def test_s16_equals_f32(dec, scenario):
    x = R.capture(scenario, 25_000_000)
    assert _decode(dec, _s16(x), 25_000_000, N.SIG_LOGIC_S16) == _decode(dec, x, 25_000_000)


@pytest.mark.gpu
@pytest.mark.parametrize("scenario,rate,kind", R.CLOCK_CASES, ids=CLOCK_IDS)
def test_device_multilevel_clock(dec, scenario, rate, kind):
    """a CLK channel with more than two levels falls on consecutive samples: more than the first try's 2 048 falling
    edges per 4 096-sample tile for the staircase and the ramp"""
    x = R.clock_capture(scenario, rate, kind)
    if kind != "noise":
        assert _falls_per_tile(x).max() > 2048
    assert _decode(dec, x, rate) == R.expected(x, rate)
    q = R.s16(x)
    assert _decode(dec, q, rate, N.SIG_LOGIC_S16) == R.host(q, rate, sigtype=6)


@pytest.mark.gpu
def test_host_and_device_input_agree(dec):
    import torch
    x = R.capture("t1_lrc", 25_000_000)
    t = torch.from_numpy(x).cuda()
    assert _decode(dec, t, 25_000_000) == _decode(dec, x, 25_000_000) == R.expected(x, 25_000_000)
    ts = torch.from_numpy(_s16(x)).cuda()
    assert _decode(dec, ts, 25_000_000, N.SIG_LOGIC_S16) == R.expected(x, 25_000_000)


@pytest.mark.gpu
def test_stream_alone_equals_stream_in_batch(dec):
    rate = 25_000_000
    xs = [R.capture(sc, rate, seed=3) for sc in R.S.ISO_SCENARIOS]
    n = min(len(x) for x in xs)
    batch = np.stack([x[:n] for x in xs])
    together = _decode(dec, batch, rate)
    alone = []
    for i in range(len(xs)):
        for row in _decode(dec, batch[i], rate):
            row[0] = i
            alone.append(row)
    assert together == alone
    assert {r[0] for r in together} == set(range(len(xs)))


@pytest.mark.gpu
def test_many_streams_match_the_host_build():
    """a batch whose line events overflow the first try's slots (noise on IO) and whose 1 100 frames overflow the first
    frame pool of 1 024 (a fresh handle, so the pool has not grown in an earlier call)"""
    rate = 10_000_000
    x = R.capture("t0_direct", rate, seed=5)
    rng = np.random.default_rng(7)
    noisy = x.copy()
    noisy[:200_000, 0] = rng.integers(0, 2, 200_000)
    batch = np.stack([x] * 100 + [noisy])
    one, last = R.host(x, rate), R.host(noisy, rate)
    want = [[s] + r[1:] for s in range(100) for r in one] + [[100] + r[1:] for r in last]
    assert len(want) > 1024
    d = N.NfcDecoder(device=0)
    d.setStreamTime(R.STREAM_TIME)
    assert _decode(d, batch, rate) == want
    d.close()


@pytest.mark.gpu
def test_errors(dec):
    x = R.capture("t0_direct", 10_000_000)
    lib, h = dec._lib, dec._h
    buf = (R.CFrame * 4)()
    n = R.C.c_uint64(0)
    a = np.ascontiguousarray(x[None])
    call = lambda ptr, sig, ns, nsamp, rate, out=buf, cap=4: lib.nfcb200_iso7816_decode_batch(h, R.C.c_void_p(ptr), 0, sig, ns, nsamp, rate, out,
                                                                                              cap, R.C.byref(n))
    assert call(a.ctypes.data, N.SIG_MAG_F32, 1, len(x), 10_000_000) == -2
    assert call(a.ctypes.data, N.SIG_IQ_S16, 1, len(x), 10_000_000) == -2
    assert call(a.ctypes.data, 7, 1, len(x), 10_000_000) == -2
    assert call(a.ctypes.data, N.SIG_LOGIC_F32, 1, len(x), 0) == -2
    assert call(0, N.SIG_LOGIC_F32, 1, len(x), 10_000_000) == -2
    assert call(a.ctypes.data, N.SIG_LOGIC_F32, 0, len(x), 10_000_000) == -2
    assert call(a.ctypes.data, N.SIG_LOGIC_F32, 1, 0, 10_000_000) == -2
    assert call(a.ctypes.data, N.SIG_LOGIC_F32, 1, len(x), 10_000_000, out=None, cap=4) == -2
    assert call(a.ctypes.data, N.SIG_LOGIC_F32, 1, 0xFFFFFFFF, 10_000_000) == -5
    assert lib.nfcb200_iso7816_decode_batch(None, R.C.c_void_p(a.ctypes.data), 0, N.SIG_LOGIC_F32, 1, len(x), 10_000_000, buf, 4, R.C.byref(n)) == -2
    with pytest.raises(N.NfcB200Error):
        dec.iso7816_decode(x[:, :2], N.SIG_LOGIC_F32, 10_000_000)
    # a tensor whose dtype does not match the signal type is refused before anything reads it
    import torch
    with pytest.raises(N.NfcB200Error):
        dec.iso7816_decode(torch.from_numpy(_s16(x)).cuda(), N.SIG_LOGIC_F32, 10_000_000)
    with pytest.raises(N.NfcB200Error):
        dec.iso7816_decode(torch.from_numpy(x).cuda(), N.SIG_LOGIC_S16, 10_000_000)
    # capacity: the first cap frames, the total in n_out
    want = R.expected(x, 10_000_000)
    assert call(a.ctypes.data, N.SIG_LOGIC_F32, 1, len(x), 10_000_000) == -4
    assert n.value == len(want) > 4
    assert R.rows(buf, 4) == want[:4]
    assert call(a.ctypes.data, N.SIG_LOGIC_F32, 1, len(x), 10_000_000, out=None, cap=0) == -4
    assert n.value == len(want)


def _nfc_capture():
    mag, rate, _ = U.fixture_wav("test_NFC-A_106kbps_001")
    return mag, rate


@pytest.mark.gpu
def test_batch_decode_state_survives_an_iso_call():
    mag, rate = _nfc_capture()
    d = N.NfcDecoder(device=0)
    batch = np.stack([mag, mag[::-1].copy()])
    first = d.decode_batch(batch, N.SIG_MAG_F32, rate)
    flags, stats = d.block_flags(), d.stats()
    recs = d.device_frames()
    d.iso7816_decode(R.capture("t1_lrc", 10_000_000), N.SIG_LOGIC_F32, 10_000_000)
    assert d.device_frames() == recs
    assert np.array_equal(d.block_flags(), flags)
    assert d.stats() == stats
    assert d.decode_batch(batch, N.SIG_MAG_F32, rate) == first
    d.close()


@pytest.mark.gpu
def test_streaming_decode_split_by_an_iso_call():
    mag, rate = _nfc_capture()
    half = len(mag) // 2
    d = N.NfcDecoder(device=0)
    plain = d.nextFrames(mag[:half], rate) + d.nextFrames(mag[half:], rate) + d.nextFrames(None, rate)
    d.close()
    d = N.NfcDecoder(device=0)
    split = d.nextFrames(mag[:half], rate)
    d.iso7816_decode(R.capture("t0_inverse", 10_000_000), N.SIG_LOGIC_F32, 10_000_000)
    split += d.nextFrames(mag[half:], rate) + d.nextFrames(None, rate)
    d.close()
    assert split == plain and len(plain) > 0


def _cframe(tech, ftype, start, date_time, data=b""):
    f = R.CFrame()
    f.tech_type, f.frame_type, f.sample_start, f.sample_end, f.sample_rate = tech, ftype, start, start + 100, 10_000_000
    f.date_time, f.length = date_time, len(data)
    for i, b in enumerate(data):
        f.data[i] = b
    return f


def test_export_names_iso_frames_and_keeps_their_date_time():
    from nfc_laboratory_b200 import export as X
    atr = _cframe(0x0201, 0x0210, 3001, 1000.0, bytes([0x3B, 0x00]))
    e = X.trz_entry(atr, 10_000_000, stream_time=1000)
    assert e["dateTime"] == 1000.0 and e["frameData"] == "3B:00" and e["length"] == 2
    line = X.rx_json_line(atr, 10_000_000, stream_time=1000)
    assert '"tech":"ISO7816"' in line and '"type":"ATR"' in line and '"date_time":1000' in line
    vcc = _cframe(0x0200, 0x0201, 200, 1000.00002)
    assert X.trz_entry(vcc, 10_000_000, stream_time=1000)["dateTime"] == 1000.00002
    assert '"type":"VccHigh"' in X.rx_json_line(vcc, 10_000_000, stream_time=1000)
    # an NFC frame's date_time stays stream_time + time_start, whatever the record holds
    poll = _cframe(0x0101, 0x0102, 3001, 5.0, bytes([0x26]))
    assert X.trz_entry(poll, 10_000_000, stream_time=1000)["dateTime"] == 1000 + 3001 / 10_000_000
