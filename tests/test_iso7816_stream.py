"""Streaming ISO 7816 decode of one logic capture pushed buffer by buffer (nfcb200_iso7816_stream_push, lab::IsoDecoder
fed by LogicDecoderTask).

CPU: the host build of the stream push against the recorded reference output for every case and chunk plan, on every
field and the payload, and against the live chunked oracle where oracle/_ref/libnfcref_iso_stream.so was built; the
reference's call-boundary quirk pinned on warm_reset; the ABI.
GPU: the device push against the recorded output (float and int16), one push against the batch call, the capacity path,
reset, isolation from every other state of the handle both ways, the error paths, and the drop-in shim against the
reference behind the same driver."""
import ctypes as C

import numpy as np
import pytest

import iso_ref as R
import iso_stream_ref as T
import nfcutil as U
import nfc_laboratory_b200 as N

CASE_IDS = [T.case_id(c) for c in T.CASES]
WARM = [c for c in T.CASES if c[0] == "warm_reset" and c[2] is None]


@pytest.mark.parametrize("case", T.CASES, ids=CASE_IDS)
def test_host_stream_equals_golden(case):
    for plan, (x, chunks, rates) in T.plans(case).items():
        assert T.host(x, chunks, rates) == T.expected(case, plan), plan


@pytest.mark.parametrize("case", T.CASES, ids=CASE_IDS)
def test_host_stream_equals_live_oracle(case):
    if T.ref_lib() is None:
        pytest.skip("the chunked reference oracle was not built (oracle/iso_stream.mk needs the reference sources)")
    for plan, (x, chunks, rates) in T.plans(case).items():
        assert T.host(x, chunks, rates) == T.chunked(T.ref_lib(), x, chunks, rates), plan


@pytest.mark.parametrize("case", WARM, ids=[T.case_id(c) for c in WARM])
def test_split_while_reset_is_low_gives_two_more_frames(case):
    """the reference picks its loop afresh at every buffer: a buffer that ends while RST is low after the warm reset, inside
    decodeStreamT0 with the protocol cleared, lets the next buffer detect the reset release and a second ATR"""
    x = T.case_capture(case)
    whole = R.expected(x, case[1])
    assert T.expected(case, "whole") == whole
    windows = T.rst_low_windows(x)
    assert len(windows) == 3  # power-up, warm reset, power-off
    assert len(T.expected(case, "split_rst1")) == len(whole) + 2
    assert T.expected(case, "split_rst0") == T.expected(case, "split_rst2") == whole
    extra = [f for f in T.expected(case, "split_rst1") if f not in whole]
    assert [f[2] for f in extra if f[2] == 0x210] == [0x210] and any(f[13] == "3b00" for f in extra)
    x, chunks, rates = T.plans(case)["split_rst1"]
    assert T.host(x, chunks, rates) == T.expected(case, "split_rst1")


def test_int16_host_stream_equals_float():
    case = ("t1_crc", 25_000_000, None)
    x, chunks, rates = T.plans(case)["random"]
    assert T.host(R.s16(x), chunks, rates, sigtype=6) == T.host(x, chunks, rates) == T.expected(case, "random")


def test_library_exports_the_stream_entry_points():
    header = open(R.os.path.join(R.ROOT, "include", "nfcb200.h")).read()
    lib = C.CDLL(N.library_path())
    for name in ("nfcb200_iso7816_stream_push", "nfcb200_iso7816_stream_pending", "nfcb200_iso7816_stream_reset"):
        assert "int %s(" % name in header
        assert hasattr(lib, name)


# --- GPU ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dec():
    d = N.NfcDecoder(device=0)
    d.setStreamTime(R.STREAM_TIME)
    yield d
    d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", T.CASES, ids=CASE_IDS)
def test_device_stream_equals_golden(dec, case):
    for plan, (x, chunks, rates) in T.plans(case).items():
        want = T.expected(case, plan)
        dec.iso7816_reset()
        assert T.push(dec, x, chunks, rates, N.SIG_LOGIC_F32) == want, plan
        dec.iso7816_reset()
        q = R.s16(x)
        assert T.push(dec, q, chunks, rates, N.SIG_LOGIC_S16) == T.host(q, chunks, rates, sigtype=6), plan


@pytest.mark.gpu
@pytest.mark.parametrize("case", T.CASES, ids=CASE_IDS)
def test_one_push_equals_the_batch_call(dec, case):
    x, rate = T.case_capture(case), case[1]
    dec.iso7816_reset()
    pushed = T.push(dec, x, [len(x)], [rate], N.SIG_LOGIC_F32)
    buf, n = dec.iso7816_decode(x, N.SIG_LOGIC_F32, rate, raw=True)
    assert pushed == R.rows(buf, n) == R.expected(x, rate)


def _raw_push(d, x, rate, cap, sigtype=N.SIG_LOGIC_F32):
    a = np.ascontiguousarray(x, dtype=np.float32)
    buf = (R.CFrame * max(cap, 1))()
    n = C.c_uint64(0)
    rc = d._lib.nfcb200_iso7816_stream_push(d._h, a.ctypes.data, sigtype, len(a), rate, buf, cap, C.byref(n))
    return rc, R.rows(buf, n.value)


@pytest.mark.gpu
def test_capacity_keeps_the_rest_pending():
    case = ("t1_crc", 10_000_000, None)
    x, chunks, rates = T.plans(case)["random"]
    d = N.NfcDecoder(device=0)
    d.setStreamTime(R.STREAM_TIME)
    got, at, saw_capacity = [], 0, False
    for c, r in zip(chunks, rates):
        rc, rows = _raw_push(d, x[at:at + c], r, 1)
        at += c
        assert rc in (0, -4) and len(rows) <= 1
        saw_capacity |= rc == -4
        got += rows
        # drain part of what is pending, the rest rides along to the next push
        buf = (R.CFrame * 2)()
        n, left = C.c_uint64(0), C.c_uint64(0)
        assert d._lib.nfcb200_iso7816_stream_pending(d._h, buf, 2, C.byref(n), C.byref(left)) == 0
        got += R.rows(buf, n.value)
    got += T.push(d, x[:0], [], [], N.SIG_LOGIC_F32)  # the flush drains the rest
    d.close()
    assert saw_capacity
    assert got == T.expected(case, "random")


@pytest.mark.gpu
def test_reset_decodes_as_a_fresh_handle(dec):
    a = R.capture("t0_inverse", 25_000_000)
    b = R.capture("t1_lrc", 10_000_000)
    dec.iso7816_reset()
    dec.iso7816_push(a[: len(a) // 3], N.SIG_LOGIC_F32, 25_000_000)
    dec.iso7816_reset()
    got = T.push(dec, b, [len(b)], [10_000_000], N.SIG_LOGIC_F32)
    fresh = N.NfcDecoder(device=0)
    fresh.setStreamTime(R.STREAM_TIME)
    assert got == T.push(fresh, b, [len(b)], [10_000_000], N.SIG_LOGIC_F32) == R.expected(b, 10_000_000)
    fresh.close()


def _nfc_capture():
    mag, rate, _ = U.fixture_wav("test_NFC-A_106kbps_001")
    return mag, rate


@pytest.mark.gpu
def test_other_calls_leave_the_iso_stream_alone():
    case = ("warm_reset", 10_000_000, None)
    x, chunks, rates = T.plans(case)["random"]
    mag, nrate = _nfc_capture()
    iq = np.random.default_rng(3).normal(size=(1, 1 << 16, 2)).astype(np.float32)
    d = N.NfcDecoder(device=0)
    d.setStreamTime(R.STREAM_TIME)
    got, at = [], 0
    for k, (c, r) in enumerate(zip(chunks, rates)):
        got += d.iso7816_push(x[at:at + c], N.SIG_LOGIC_F32, r, raw=True)
        at += c
        step = k % 4
        if step == 0:
            d.nextFrames(mag[: len(mag) // 2], nrate)
        elif step == 1:
            d.decode_batch(mag[None], N.SIG_MAG_F32, nrate)
        elif step == 2:
            d.iso7816_decode(R.capture("t1_lrc", 10_000_000), N.SIG_LOGIC_F32, 10_000_000)
        else:
            d.spectrum(iq, N.SIG_IQ_F32, 10_000_000)
    got += d.iso7816_flush(raw=True)
    d.close()
    assert R.rows(got, len(got)) == T.expected(case, "random")


@pytest.mark.gpu
def test_iso_pushes_leave_the_other_states_alone():
    mag, rate = _nfc_capture()
    half = len(mag) // 2
    x = R.capture("t0_direct", 10_000_000)
    d = N.NfcDecoder(device=0)
    plain = d.nextFrames(mag[:half], rate) + d.nextFrames(mag[half:], rate) + d.nextFrames(None, rate)
    d.close()
    d = N.NfcDecoder(device=0)
    batch = mag[None]  # one stream, so that carry_before answers
    first = d.decode_batch(batch, N.SIG_MAG_F32, rate)
    flags, stats = d.block_flags(), d.stats()
    carry = d.carry_before(0)
    split = d.nextFrames(mag[:half], rate)
    d.iso7816_push(x[: len(x) // 2], N.SIG_LOGIC_F32, 10_000_000)
    split += d.nextFrames(mag[half:], rate)
    d.iso7816_push(x[len(x) // 2:], N.SIG_LOGIC_F32, 10_000_000)
    split += d.nextFrames(None, rate)
    d.iso7816_flush()
    assert split == plain and len(plain) > 0
    assert np.array_equal(d.block_flags(), flags)
    assert d.stats() == stats
    assert d.carry_before(0) == carry
    assert d.decode_batch(batch, N.SIG_MAG_F32, rate) == first
    d.close()


@pytest.mark.gpu
def test_stream_errors(dec):
    x = R.capture("t0_direct", 10_000_000)[:10_000]
    lib, h = dec._lib, dec._h
    a = np.ascontiguousarray(x)
    buf = (R.CFrame * 4)()
    n = C.c_uint64(0)
    call = lambda ptr, sig, cnt, rate: lib.nfcb200_iso7816_stream_push(h, C.c_void_p(ptr), sig, cnt, rate, buf, 4, C.byref(n))
    dec.iso7816_reset()
    assert call(a.ctypes.data, N.SIG_MAG_F32, len(a), 10_000_000) == -2
    assert call(a.ctypes.data, N.SIG_IQ_S16, len(a), 10_000_000) == -2
    assert call(0, N.SIG_LOGIC_F32, len(a), 10_000_000) == -2
    assert call(a.ctypes.data, N.SIG_LOGIC_F32, len(a), 0) == -2
    assert call(a.ctypes.data, N.SIG_LOGIC_F32, 0xFFFFFFFF, 10_000_000) == -5
    assert lib.nfcb200_iso7816_stream_push(None, C.c_void_p(a.ctypes.data), N.SIG_LOGIC_F32, len(a), 10_000_000, buf, 4, C.byref(n)) == -2
    assert lib.nfcb200_iso7816_stream_push(h, C.c_void_p(a.ctypes.data), N.SIG_LOGIC_F32, len(a), 10_000_000, None, 4, C.byref(n)) == -2
    with pytest.raises(N.NfcB200Error):
        dec.iso7816_push(x, N.SIG_MAG_F32, 10_000_000)
    with pytest.raises(N.NfcB200Error):
        dec.iso7816_push(x[:, :2], N.SIG_LOGIC_F32, 10_000_000)
    # the refused calls left no trace: the stream still decodes as fresh
    assert T.push(dec, x, [len(x)], [10_000_000], N.SIG_LOGIC_F32) == R.host(x, 10_000_000)


@pytest.mark.gpu
@pytest.mark.parametrize("case", T.CASES, ids=CASE_IDS)
def test_shim_equals_reference(case):
    if T.shim_lib() is None or T.ref_lib() is None:
        pytest.skip("the drop-in checker was not built (oracle/iso_stream.mk needs the reference sources)")
    for plan, (x, chunks, rates) in T.plans(case).items():
        assert T.chunked(T.shim_lib(), x, chunks, rates) == T.expected(case, plan), plan
