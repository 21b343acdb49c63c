"""nfcb200_adaptive_radio / nfcb200_adaptive_logic / NfcDecoder.adaptive_radio / adaptive_logic: the reference's adaptive
signal (lab::SignalResamplingTask), and its .apcm entries in a .trz (export.write_trz, read_trz_signals).

CPU: the host build of the device steps (tests/native/adaptive_host.cpp) against the reference's recorded points, as bits;
the complete list where the reference's output buffer is too small; the .apcm members against the ones the reference's
TraceStorageTask wrote; the ABI symbols.  GPU: the device against the reference and the host build for every format and
channel count, batches against single streams, device against host input, buffer-by-buffer calls against one batch call,
the capacity and argument errors, and that the calls leave the decode state of the handle alone.
"""
import ctypes as C

import numpy as np
import pytest

import adaptive_ref as R
import nfcutil as U


def N():
    import nfc_laboratory_b200 as mod
    return mod


def X():
    from nfc_laboratory_b200 import export
    return export


def pts(a):
    """a SIGNAL_POINT_DTYPE array (or the helpers' points) as (channel, sample, value)"""
    out = np.empty(len(a), dtype=R.POINTS)
    for f in ("channel", "sample", "value"):
        out[f] = a[f]
    return out


RADIO_IDS = [R.case_id(c) for c in R.RADIO_CASES]
LOGIC_IDS = [R.case_id(c) for c in R.LOGIC_CASES]


# --- CPU ---------------------------------------------------------------------------------------------------------------

def test_every_case_is_recorded():
    assert R.recording(), "tests/golden/ref_adaptive.npz.xz is missing"
    for case in R.RADIO_CASES:
        _, _, mag, buf = R.radio_input(case)
        assert R.key(mag, buf) in R.recording(), case
    for case in R.LOGIC_CASES:
        assert R.key(R.logic_input(case)[2], R.BUFFER) in R.recording(), case


@pytest.mark.parametrize("case", R.RADIO_CASES, ids=RADIO_IDS)
def test_host_build_equals_reference_radio(case):
    _, _, mag, buf = R.radio_input(case)
    assert R.same(R.host(mag, buf), R.reference(mag, buf))


@pytest.mark.parametrize("case", R.LOGIC_CASES, ids=LOGIC_IDS)
def test_host_build_equals_reference_logic(case):
    x = R.logic_input(case)[2]
    got = R.host(x, R.BUFFER)
    assert R.same(got, R.reference(x, R.BUFFER))
    assert 1 not in set(got["channel"].tolist())  # CLK has no points


SHORT = 100  # buffers under 255 samples: the reference's output buffer holds as many points as samples


def test_host_build_returns_points_past_the_reference_capacity():
    x = R.alternating()
    got = R.host(x, SHORT)
    assert len(got) == len(x) + len(x) // SHORT > R.reference_capacity(len(x), SHORT)
    assert not R.fits_reference(x, SHORT)
    # every sample is kept, each buffer's first sample twice
    assert np.all(np.diff(got["sample"].astype(np.int64)) >= 0)
    assert np.array_equal(np.unique(got["sample"]), np.arange(len(x)))


def test_host_build_offset_moves_samples():
    _, _, mag, buf = R.radio_input(R.RADIO_CASES[0])
    a, b = R.host(mag, buf), R.host(mag, buf, offset=12345)
    assert np.array_equal(a["sample"] + 12345, b["sample"]) and np.array_equal(a["value"], b["value"])


def _trz_points(kind):
    """the host build's points of a .trz case as the binding returns them"""
    values = R.radio_input(R.TRZ_RADIO)[2] if kind == "radio" else R.logic_input(R.TRZ_LOGIC)[2]
    h = R.host(values, R.BUFFER)
    out = np.zeros(len(h), dtype=N().SIGNAL_POINT_DTYPE)
    for f in ("channel", "sample", "value"):
        out[f] = h[f]
    return out


@pytest.mark.parametrize("kind", ["radio", "logic"])
@pytest.mark.parametrize("name", list(R.TRZ_RANGES))
def test_write_trz_members_equal_reference(tmp_path, kind, name):
    rng = R.TRZ_RANGES[name] or (0.0, 0.0)  # a Write command without a range writes [0, 0] (TraceStorageTask.cpp:228-229)
    p = tmp_path / "t.trz"
    points = _trz_points(kind)
    X().write_trz(p, [], R.RATE, **{kind: points}, range_start=rng[0], range_end=rng[1])
    got = R.trz_members(p)
    want = R.recorded_members(kind, name)
    assert want, "no recorded .trz members"
    assert list(got) == list(want)
    for member in want:
        if member.endswith(".apcm"):
            assert got[member] == want[member], member


@pytest.mark.parametrize("kind", ["radio", "logic"])
def test_read_trz_signals_round_trip(tmp_path, kind):
    p = tmp_path / "t.trz"
    points = _trz_points(kind)
    X().write_trz(p, [], R.RATE, **{kind: points})
    back = X().read_trz_signals(p)
    for ch in np.unique(points["channel"] if kind == "logic" else points["stream"]):
        name = "%s-%d.apcm" % (kind, ch)
        info, got = back[name]
        mine = points[(points["channel"] if kind == "logic" else points["stream"]) == ch]
        assert info[X().INFO_TOTAL_SAMPLES] == len(mine) and info[X().INFO_SAMPLE_RATE] == R.RATE
        assert np.array_equal(got["sample"], mine["sample"])
        if kind == "logic":
            assert np.array_equal(got["value"], (mine["value"] > 0.5).astype(np.float32))
        else:
            q = X()._short(mine["value"] * np.float32(32768.0))
            assert np.array_equal(got["value"], q.astype(np.float32) * np.float32(1.0 / 32768))


def test_write_trz_without_signals_keeps_one_member(tmp_path):
    p = tmp_path / "t.trz"
    X().write_trz(p, [], R.RATE)
    assert list(R.trz_members(p)) == ["frame.json"]


def test_abi_symbols_present():
    lib = C.CDLL(N().library_path()) if __import__("os").path.exists(N().library_path()) else None
    if lib is None:
        pytest.skip("libnfcb200.so not built")
    for name in ("nfcb200_adaptive_radio", "nfcb200_adaptive_logic"):
        assert hasattr(lib, name)
    assert N().SIGNAL_POINT_DTYPE.itemsize == 24


# --- GPU ---------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def dec():
    d = N().NfcDecoder(device=0)
    yield d
    d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", R.RADIO_CASES, ids=RADIO_IDS)
def test_device_equals_reference_radio(dec, case):
    data, sig, mag, buf = R.radio_input(case)
    got = dec.adaptive_radio(data, sig, R.RATE, buffer=buf)
    assert R.same(pts(got), R.reference(mag, buf))
    assert np.all(got["stream"] == 0) and np.all(got["channel"] == 0)


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in R.RADIO_CASES if c[0] == "iq_s16"], ids=lambda c: R.case_id(c))
def test_device_s16_equals_f32_of_the_same_grid(dec, case):
    data, _, _, buf = R.radio_input(case)
    f = data.astype(np.float32) / np.float32(32768.0)
    assert R.same(pts(dec.adaptive_radio(data, R.IQ_S16, R.RATE, buffer=buf)), pts(dec.adaptive_radio(f, R.IQ_F32, R.RATE, buffer=buf)))
    mag = R.magnitude(f)
    assert R.same(pts(dec.adaptive_radio(mag, R.MAG_F32, R.RATE, buffer=buf)), R.reference(mag, buf))


@pytest.mark.gpu
def test_device_mag_s16(dec):
    s = R.to_s16(R.radio_input(R.RADIO_CASES[0])[2] * np.float32(0.5))
    got = dec.adaptive_radio(s, R.MAG_S16, R.RATE)
    assert R.same(pts(got), R.host(s.astype(np.float32) / np.float32(32768.0), R.BUFFER))


@pytest.mark.gpu
@pytest.mark.parametrize("case", R.LOGIC_CASES, ids=LOGIC_IDS)
def test_device_equals_reference_logic(dec, case):
    data, sig, x = R.logic_input(case)
    got = dec.adaptive_logic(data, sig, R.RATE)
    assert R.same(pts(got), R.reference(x, R.BUFFER))


@pytest.mark.gpu
@pytest.mark.parametrize("ch", [5, 6, 7])
def test_device_logic_other_channel_counts(dec, ch):
    x = R.logic_input(("t1_crc", R.LOGIC_F32, 8))[2][:, :ch].copy()
    assert R.same(pts(dec.adaptive_logic(x, R.LOGIC_F32, R.RATE)), R.host(x, R.BUFFER))


@pytest.mark.gpu
def test_batch_equals_single_streams_and_device_input(dec):
    import torch
    cases = [c for c in R.RADIO_CASES if c[0] == "iq_f32" and c[2] == R.BUFFER]
    n = min(R.radio_input(c)[0].shape[0] for c in cases)
    batch = np.stack([R.radio_input(c)[0][:n] for c in cases] * 2)
    got = dec.adaptive_radio(batch, R.IQ_F32, R.RATE)
    for s in range(batch.shape[0]):
        one = dec.adaptive_radio(batch[s], R.IQ_F32, R.RATE)
        assert R.same(pts(got[got["stream"] == s]), pts(one))
    assert np.array_equal(got["stream"], np.sort(got["stream"], kind="stable"))
    dev = dec.adaptive_radio(torch.from_numpy(batch).cuda(), R.IQ_F32, R.RATE)
    assert dev.tobytes() == got.tobytes()
    lb = np.stack([R.logic_input(("t0_direct", R.LOGIC_U8, 8))[0], R.logic_input(("t0_direct", R.LOGIC_U8, 8))[0][::-1]])
    lgot = dec.adaptive_logic(lb, R.LOGIC_U8, R.RATE)
    for s in range(2):
        assert R.same(pts(lgot[lgot["stream"] == s]), pts(dec.adaptive_logic(lb[s], R.LOGIC_U8, R.RATE)))
    assert dec.adaptive_logic(torch.from_numpy(lb).cuda(), R.LOGIC_U8, R.RATE).tobytes() == lgot.tobytes()


@pytest.mark.gpu
def test_buffer_by_buffer_equals_batch(dec):
    data, sig, _, buf = R.radio_input(("iq_f32", "nfca106", R.BUFFER))
    whole = dec.adaptive_radio(data, sig, R.RATE, buffer=buf)
    parts = [dec.adaptive_radio(data[b0:b0 + buf], sig, R.RATE, buffer=len(data[b0:b0 + buf]), offset=b0) for b0 in range(0, len(data), buf)]
    assert np.concatenate(parts).tobytes() == whole.tobytes()
    x = R.logic_input(("t1_crc", R.LOGIC_S16, 4))[0]
    whole = pts(dec.adaptive_logic(x, R.LOGIC_S16, R.RATE))
    parts = pts(np.concatenate([dec.adaptive_logic(x[b0:b0 + R.BUFFER], R.LOGIC_S16, R.RATE, buffer=R.BUFFER, offset=b0)
                                for b0 in range(0, len(x), R.BUFFER)]))
    assert R.same(R.by_channel(parts), whole)


@pytest.mark.gpu
def test_device_equals_host_past_the_reference_capacity_and_on_random_input(dec):
    x = R.alternating()
    assert R.same(pts(dec.adaptive_radio(x, R.MAG_F32, R.RATE, buffer=SHORT)), R.host(x, SHORT))
    rng = np.random.default_rng(7)
    r = (0.5 + 0.004 * rng.standard_normal(10 ** 6)).astype(np.float32)
    r[rng.integers(0, len(r), 2000)] += np.float32(0.1)
    for buf in (R.BUFFER, 1000, 7, 26):
        assert R.same(pts(dec.adaptive_radio(r, R.MAG_F32, R.RATE, buffer=buf)), R.host(r, buf))
    lg = (rng.random((10 ** 6, 6)) < 0.01).astype(np.float32).cumsum(axis=0) % 2
    assert R.same(pts(dec.adaptive_logic(lg, R.LOGIC_F32, R.RATE, buffer=5000)), R.host(lg, 5000))


def _raw_radio(d, data, sig, cap, buf=R.BUFFER):
    out = np.zeros(max(cap, 1), dtype=N().SIGNAL_POINT_DTYPE)
    n = C.c_uint64(0)
    rc = d._lib.nfcb200_adaptive_radio(d._h, data.ctypes.data, 0, sig, 1, len(data), R.RATE, buf, 0, out.ctypes.data, cap, C.byref(n))
    return rc, int(n.value), out


@pytest.mark.gpu
def test_capacity_and_invalid_arguments(dec):
    data, sig, _, _ = R.radio_input(("iq_f32", "nfca106", R.BUFFER))
    full = dec.adaptive_radio(data, sig, R.RATE)
    rc, n, out = _raw_radio(dec, data, sig, 100)
    assert rc == -4 and n == len(full) and out[:100].tobytes() == full[:100].tobytes()
    rc, n, _ = _raw_radio(dec, data, sig, 0)
    assert rc == -4 and n == len(full)
    for bad_sig in (0, 5, 9):
        assert _raw_radio(dec, data, bad_sig, 10)[0] == -2
    assert _raw_radio(dec, data, sig, 10, buf=0)[0] == -2
    assert _raw_radio(dec, data, sig, 10, buf=(1 << 24) + 1)[0] == -5
    assert _raw_radio(dec, data, sig, 10 ** 6, buf=1 << 24)[0] == 0
    n = C.c_uint64(0)
    assert dec._lib.nfcb200_adaptive_radio(dec._h, data.ctypes.data, 0, sig, 1, len(data), R.RATE, R.BUFFER, (1 << 32) - 10, None, 0, C.byref(n)) == -5
    x = R.logic_input(("t0_direct", R.LOGIC_F32, 4))[0]
    for ch in (0, 3, 9):
        assert dec._lib.nfcb200_adaptive_logic(dec._h, x.ctypes.data, 0, R.LOGIC_F32, ch, 1, 1000, R.RATE, R.BUFFER, 0, None, 0, C.byref(n)) == -2
    assert dec._lib.nfcb200_adaptive_logic(dec._h, x.ctypes.data, 0, R.IQ_F32, 4, 1, 1000, R.RATE, R.BUFFER, 0, None, 0, C.byref(n)) == -2
    assert dec._lib.nfcb200_adaptive_logic(dec._h, x.ctypes.data, 0, R.LOGIC_F32, 4, 1, 1000, R.RATE, 0, 0, None, 0, C.byref(n)) == -2
    assert dec._lib.nfcb200_adaptive_logic(dec._h, x.ctypes.data, 0, R.LOGIC_F32, 4, 1, 1000, R.RATE, (1 << 24) + 1, 0, None, 0, C.byref(n)) == -5


@pytest.mark.gpu
def test_adaptive_calls_leave_decode_state_alone():
    d = N().NfcDecoder(device=0)
    try:
        mag, rate, _ = U.fixture_wav("test_NFC-A_106kbps_001")
        frames = d.decode_batch(mag[None, :], N().SIG_MAG_F32, rate)
        st = d.stats()
        flags = d.block_flags()
        half = len(mag) // 2
        pushed = d.nextFrames(mag[:half], rate)
        d.adaptive_radio(mag, N().SIG_MAG_F32, rate)
        d.adaptive_logic(R.logic_input(("t0_direct", R.LOGIC_F32, 4))[0], R.LOGIC_F32, rate)
        assert d.stats() == st
        assert np.array_equal(d.block_flags(), flags)
        rest = d.nextFrames(mag[half:], rate) + d.nextFrames(None)
        ref = N().NfcDecoder(device=0)
        try:
            assert pushed + rest == ref.nextFrames(mag[:half], rate) + ref.nextFrames(mag[half:], rate) + ref.nextFrames(None)
        finally:
            ref.close()
        assert d.decode_batch(mag[None, :], N().SIG_MAG_F32, rate) == frames
    finally:
        d.close()
