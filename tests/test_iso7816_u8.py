"""ISO 7816 decode of logic captures of 4-8 channels and of the reference's 8-bit logic samples (SIG_LOGIC_U8) on the
H100: the _ch stream push of 8-bit WAV samples in SignalStorageTask::readLogic's 65 536-sample buffers against the
reference's replay of the same files, the _ch batch call against the 4-channel float call on b / 255.f, wider strides
against stride 4, host against device input, unaligned bases and pitches, the drop-in shim on stride-6 buffers, the error
paths, and isolation from the handle's other states."""
import ctypes as C

import numpy as np
import pytest

import iso_ref as R
import iso_stream_ref as T
import logic_ref as L
import nfcutil as U
import nfc_laboratory_b200 as N

IDS = [L.case_id(c) for c in L.CASES]
SMALL = [c for c in L.CASES if c[0][1] == 10_000_000 and c[0][2] is None]  # the 10 MS/s scenarios at 4, 5 and 8 channels


def test_library_exports_the_channel_entry_points():
    header = open(R.os.path.join(R.ROOT, "include", "nfcb200.h")).read()
    lib = C.CDLL(N.library_path())
    for name in ("nfcb200_iso7816_decode_batch_ch", "nfcb200_iso7816_stream_push_ch"):
        assert "int %s(" % name in header
        assert hasattr(lib, name)
    assert "NFCB200_SIG_LOGIC_U8 = 7" in header and N.SIG_LOGIC_U8 == 7


def test_recorded_frames_ignore_the_extra_channels():
    """the reference's frames for 5 and 8 channels are those for 4"""
    for case in L.CASES:
        assert L.expected(case) == L.expected((case[0], 4)), L.case_id(case)


@pytest.fixture(scope="module")
def dec():
    d = N.NfcDecoder(device=0)
    d.setStreamTime(L.EPOCH)
    yield d
    d.close()


def _push(d, x, sigtype, rate, chunks):
    d.iso7816_reset()
    return T.push(d, x, chunks, [rate] * len(chunks), sigtype)


def _rows(frames):
    buf, n = frames
    return R.rows(buf, n)


@pytest.mark.gpu
@pytest.mark.parametrize("case", L.CASES, ids=IDS)
def test_u8_push_equals_golden(dec, case):
    b = L.u8(case)
    assert _push(dec, b, N.SIG_LOGIC_U8, case[0][1], L.chunks(len(b))) == L.expected(case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", SMALL, ids=[L.case_id(c) for c in SMALL])
def test_u8_batch_equals_float_batch(dec, case):
    """bit for bit: the _ch batch of the bytes and the 4-channel float call on b / 255.f, one stream and three"""
    b = L.u8(case)
    rate = case[0][1]
    want = _rows(dec.iso7816_decode(L.as_float(b)[:, :4], N.SIG_LOGIC_F32, rate, raw=True))
    assert _rows(dec.iso7816_decode(b, N.SIG_LOGIC_U8, rate, raw=True)) == want
    three = np.stack([b, b, b])
    three[1, :, 4:] = 255 - three[1, :, 4:]
    got = _rows(dec.iso7816_decode(three, N.SIG_LOGIC_U8, rate, raw=True))
    assert [r[1:] for r in got] == [r[1:] for r in want] * 3
    assert [r[0] for r in got] == sorted([0, 1, 2] * len(want))


@pytest.mark.gpu
@pytest.mark.parametrize("sigtype", [N.SIG_LOGIC_F32, N.SIG_LOGIC_S16])
@pytest.mark.parametrize("channels", [5, 6, 7, 8])
def test_wider_strides_equal_stride_4(dec, sigtype, channels):
    for scenario, rate, kind in (("t1_crc", 10_000_000, None), ("t0_direct", 10_000_000, "staircase")):
        x = R.clock_capture(scenario, rate, kind) if kind else R.capture(scenario, rate)
        extra = np.random.default_rng(channels).uniform(-1, 1, (len(x), channels - 4)).astype(np.float32)
        w = np.concatenate([x, extra], axis=1)
        if sigtype == N.SIG_LOGIC_S16:
            x, w = R.s16(x), R.s16(w)
        want = _rows(dec.iso7816_decode(x, sigtype, rate, raw=True))
        assert len(want) > 0
        assert _rows(dec.iso7816_decode(w, sigtype, rate, raw=True)) == want
        chunks = T._random_chunks(np.random.default_rng(channels), len(x), 1_000, 300_000)
        assert _push(dec, w, sigtype, rate, chunks) == _push(dec, x, sigtype, rate, chunks)


@pytest.mark.gpu
@pytest.mark.parametrize("case", SMALL, ids=[L.case_id(c) for c in SMALL])
def test_host_and_device_input_agree(dec, case):
    import torch
    b = L.u8(case)
    rate = case[0][1]
    host = _rows(dec.iso7816_decode(b, N.SIG_LOGIC_U8, rate, raw=True))
    assert _rows(dec.iso7816_decode(torch.from_numpy(np.array(b)).cuda(), N.SIG_LOGIC_U8, rate, raw=True)) == host
    assert _rows(dec.iso7816_decode(torch.from_numpy(np.array(b)), N.SIG_LOGIC_U8, rate, raw=True)) == host


@pytest.mark.gpu
@pytest.mark.parametrize("channels", [4, 5, 7])
def test_unaligned_base_and_pitch(dec, channels):
    """streams of an odd length at 4, 5 and 7 channels, their batch one byte (8-bit) or one channel (float) past an aligned
    base: every stream decodes as it does alone"""
    import torch
    rate = 10_000_000
    xs = [np.clip(R.capture(sc, rate), 0, 1)[:600_001] for sc in ("t0_direct", "t1_lrc", "warm_reset")]
    rng = np.random.default_rng(channels)
    w = np.stack([np.concatenate([x, rng.random((len(x), channels - 4), dtype=np.float32)], axis=1) for x in xs]).astype(np.float32)
    b = (w * np.float32(255)).astype(np.uint8)
    alone_u8 = [_rows(dec.iso7816_decode(s[:, :4].copy(), N.SIG_LOGIC_U8, rate, raw=True)) for s in b]
    alone_f = [_rows(dec.iso7816_decode(s[:, :4].copy(), N.SIG_LOGIC_F32, rate, raw=True)) for s in w]
    assert all(len(a) > 0 for a in alone_u8)
    for data, sigtype, alone, shift in ((b, N.SIG_LOGIC_U8, alone_u8, 1), (w, N.SIG_LOGIC_F32, alone_f, 1)):
        raw = torch.zeros(data.size + shift, dtype=torch.from_numpy(data).dtype, device="cuda")
        t = raw[shift:].view(data.shape)
        t.copy_(torch.from_numpy(data))
        got = _rows(dec.iso7816_decode(t, sigtype, rate, raw=True))
        want = [[s] + r[1:] for s, a in enumerate(alone) for r in a]
        assert got == want, (sigtype, channels)


@pytest.mark.gpu
def test_u8_push_carries_across_formats_and_channels(dec):
    """one capture pushed in buffers that alternate 8-bit and float, 4 and 8 channels: the frames of one 8-bit stream"""
    case = (("t1_crc", 10_000_000, None), 8)
    b = L.u8(case)
    f = L.as_float(b)
    rate = case[0][1]
    dec.iso7816_reset()
    got, at = [], 0
    for k, c in enumerate(L.chunks(len(b))):
        part = b[at:at + c] if k % 2 else f[at:at + c]
        part = part if k % 3 else part[:, :4]
        got += dec.iso7816_push(part, N.SIG_LOGIC_U8 if k % 2 else N.SIG_LOGIC_F32, rate, raw=True)
        at += c
    got += dec.iso7816_flush(raw=True)
    assert R.rows(got, len(got)) == L.expected(case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", SMALL[::3], ids=[L.case_id(c) for c in SMALL[::3]])
def test_shim_on_stride_6_equals_reference(case, tmp_path):
    """the drop-in shim replays a 6-channel 8-bit WAV (float buffers of stride 6) as the reference does"""
    if L.shim_lib() is None:
        pytest.skip("the drop-in checker was not built (oracle/logic_replay.mk needs the reference sources)")
    six = (case[0], 6)
    path = str(tmp_path / "logic6.wav")
    L.write(path, six)
    want = L.replay(L.ref_lib(), path) if L.ref_lib() is not None else L.expected(case)
    assert L.replay(L.shim_lib(), path) == want
    assert want == L.expected(case)


@pytest.mark.gpu
def test_channel_and_format_errors(dec):
    b = L.u8(SMALL[0])[:10_000]
    lib, h = dec._lib, dec._h
    buf = (R.CFrame * 4)()
    n = C.c_uint64(0)
    for ch in (3, 9, 0):
        a = np.ascontiguousarray(np.zeros((len(b), max(ch, 1)), dtype=np.uint8))
        assert lib.nfcb200_iso7816_stream_push_ch(h, a.ctypes.data, N.SIG_LOGIC_U8, ch, len(b), 10_000_000, buf, 4, C.byref(n)) == -2
        assert lib.nfcb200_iso7816_decode_batch_ch(h, a.ctypes.data, 0, N.SIG_LOGIC_U8, ch, 1, len(b), 10_000_000, buf, 4, C.byref(n)) == -2
    a = np.ascontiguousarray(b[:, :4])
    # 8-bit samples only through the _ch calls; the _ch calls take logic formats only
    assert lib.nfcb200_iso7816_stream_push(h, a.ctypes.data, N.SIG_LOGIC_U8, len(a), 10_000_000, buf, 4, C.byref(n)) == -2
    assert lib.nfcb200_iso7816_decode_batch(h, a.ctypes.data, 0, N.SIG_LOGIC_U8, 1, len(a), 10_000_000, buf, 4, C.byref(n)) == -2
    assert lib.nfcb200_iso7816_stream_push_ch(h, a.ctypes.data, N.SIG_MAG_F32, 4, len(a), 10_000_000, buf, 4, C.byref(n)) == -2
    assert lib.nfcb200_iso7816_decode_batch_ch(h, a.ctypes.data, 0, N.SIG_IQ_S16, 4, 1, len(a), 10_000_000, buf, 4, C.byref(n)) == -2
    # the binding: 8-bit samples with a float / int16 type, anything else with SIG_LOGIC_U8, channel counts outside 4-8
    import torch
    for call in (dec.iso7816_decode, dec.iso7816_push):
        with pytest.raises(N.NfcB200Error):
            call(b, N.SIG_LOGIC_F32, 10_000_000)
        with pytest.raises(N.NfcB200Error):
            call(b, N.SIG_LOGIC_S16, 10_000_000)
        with pytest.raises(N.NfcB200Error):
            call(L.as_float(b), N.SIG_LOGIC_U8, 10_000_000)
        with pytest.raises(N.NfcB200Error):
            call(b[:, :3], N.SIG_LOGIC_U8, 10_000_000)
        with pytest.raises(N.NfcB200Error):
            call(np.zeros((100, 9), dtype=np.uint8), N.SIG_LOGIC_U8, 10_000_000)
    with pytest.raises(N.NfcB200Error):
        dec.iso7816_decode(torch.from_numpy(np.array(b)).cuda(), N.SIG_LOGIC_F32, 10_000_000)
    with pytest.raises(N.NfcB200Error):
        dec.iso7816_decode(torch.from_numpy(L.as_float(b)).cuda(), N.SIG_LOGIC_U8, 10_000_000)
    # the refused calls left no trace: the stream still decodes as fresh
    case = SMALL[0]
    assert _push(dec, L.u8(case), N.SIG_LOGIC_U8, case[0][1], L.chunks(len(L.u8(case)))) == L.expected(case)


@pytest.mark.gpu
def test_u8_calls_leave_the_other_states_alone():
    mag, rate, _ = U.fixture_wav("test_NFC-A_106kbps_001")
    half = len(mag) // 2
    case = SMALL[0]
    b = L.u8(case)
    d = N.NfcDecoder(device=0)
    plain = d.nextFrames(mag[:half], rate) + d.nextFrames(mag[half:], rate) + d.nextFrames(None, rate)
    d.close()
    d = N.NfcDecoder(device=0)
    d.setStreamTime(L.EPOCH)
    batch = mag[None]
    first = d.decode_batch(batch, N.SIG_MAG_F32, rate)
    flags, stats = d.block_flags(), d.stats()
    carry = d.carry_before(0)
    split = d.nextFrames(mag[:half], rate)
    got = d.iso7816_push(b[: len(b) // 2], N.SIG_LOGIC_U8, case[0][1], raw=True)
    iso_batch = _rows(d.iso7816_decode(np.stack([b, b]), N.SIG_LOGIC_U8, case[0][1], raw=True))
    split += d.nextFrames(mag[half:], rate)
    got += d.iso7816_push(b[len(b) // 2:], N.SIG_LOGIC_U8, case[0][1], raw=True)
    split += d.nextFrames(None, rate)
    got += d.iso7816_flush(raw=True)
    assert split == plain and len(plain) > 0
    assert np.array_equal(d.block_flags(), flags)
    assert d.stats() == stats
    assert d.carry_before(0) == carry
    assert d.decode_batch(batch, N.SIG_MAG_F32, rate) == first
    # and the ISO stream did not see the batch call in between
    whole = _rows(d.iso7816_decode(b, N.SIG_LOGIC_U8, case[0][1], raw=True))
    assert R.rows(got, len(got)) == whole
    assert [r[1:] for r in iso_batch] == [r[1:] for r in whole] * 2
    d.close()
