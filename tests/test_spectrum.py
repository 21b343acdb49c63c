"""nfcb200_spectrum / NfcDecoder.spectrum: the reference's FFT spectrum (lab::FourierProcessTask::process) of IQ captures.

CPU: the frame geometry, the float64 model and the host build of the device transform (tests/native/spectrum_host.cpp)
against the reference's recorded frames, and the selection pattern.  GPU: the device transform against the reference, the
host build (bit for bit), itself across input / output placements, sample formats and batch positions, the error paths, and
that a spectrum call leaves the decode state of the handle alone.
"""
import ctypes as C

import numpy as np
import pytest

import nfcutil as U
import spectrum_ref as R

NAMES = list(R.CASES)
F32, S16 = 1, 4


def N():
    import nfc_laboratory_b200 as mod
    return mod


# --- CPU ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("rate, dec", [(10_000_000, 16), (4_000_000, 6), (2_500_000, 4), (625_000, 1), (1_249_999, 1)])
def test_shape_decimation(rate, dec):
    assert N().spectrum_shape(10 ** 6, rate)[1] == dec


@pytest.mark.parametrize("rate", [10_000_000, 4_000_000])
@pytest.mark.parametrize("hop", [1, 3, 4096, 16384])
def test_shape_frames_at_the_span_boundary(rate, hop):
    span = 1024 * (rate // 625000)
    shape = N().spectrum_shape
    assert shape(span - 1, rate, hop)[0] == 0
    assert shape(span, rate, hop)[0] == 1
    assert shape(span + hop - 1, rate, hop)[0] == 1
    assert shape(span + hop, rate, hop)[0] == 2
    assert shape(span + 7 * hop + hop // 2, rate, hop)[0] == 8
    assert shape(10 ** 7, rate)[0] == (10 ** 7 - span) // span + 1   # hop=None is the span


def test_shape_rejects_low_rates_and_hop_zero():
    with pytest.raises(N().NfcB200Error) as e:
        N().spectrum_shape(10 ** 6, 624_999, 1024)
    assert e.value.code == -5
    with pytest.raises(N().NfcB200Error) as e:
        N().spectrum_shape(10 ** 6, 10_000_000, 0)
    assert e.value.code == -2


def test_every_case_is_recorded():
    assert R.recording(), "tests/golden/ref_spectrum.npz.xz is missing"
    for name in NAMES:
        iq, rate, hop = R.case_input(name)
        rec = R.recording().get(R.key(iq, rate, hop))
        assert rec is not None, name
        assert rec.shape == (R.frames_of(iq.shape[0], rate, hop), 1024) and 20 <= rec.shape[0] <= 50


@pytest.mark.skipif(R.oracle_lib() is None, reason="oracle/_ref/libnfcref_fft.so not built")
@pytest.mark.parametrize("name", NAMES)
def test_live_oracle_equals_recording(name):
    iq, rate, hop = R.case_input(name)
    assert np.array_equal(R.oracle(iq, rate, hop), R.recording()[R.key(iq, rate, hop)])


@pytest.mark.parametrize("name", NAMES)
def test_float64_model_equals_reference(name):
    iq, rate, hop = R.case_input(name)
    assert R.worst(R.model(iq, rate, hop), R.reference(iq, rate, hop)) <= R.TOL


@pytest.mark.parametrize("name", NAMES)
def test_host_build_equals_reference(name):
    iq, rate, hop = R.case_input(name)
    assert R.worst(R.host(iq[None], F32, rate, hop)[0], R.reference(iq, rate, hop)) <= R.TOL


@pytest.mark.parametrize("name", R.S16_CASES)
def test_host_build_int16_equals_float(name):
    iq, rate, hop = R.case_input(name)
    assert np.array_equal(R.host(R.to_s16(iq)[None], S16, rate, hop), R.host(iq[None], F32, rate, hop))


def impulse_input(rate, hop, n_frames, positions):
    """one stream of zeros with one nonzero sample per entry of `positions`, each in its own frame"""
    span = 1024 * (rate // 625000)
    iq = np.zeros((span + (n_frames - 1) * hop, 2), dtype=np.float32)
    for f, p in enumerate(positions):
        iq[f * hop + p] = (0.5, -0.25)
    return iq


def check_impulses(spec, rate, positions):
    """frame f held one nonzero sample at offset positions[f]: its spectrum is flat at |x| w[k] when the selection
    takes that offset as window position k, and all zeros when it does not"""
    sel = {int(o): k for k, o in enumerate(R.selection(rate))}
    w = R.window()
    flat = 0
    for f, p in enumerate(positions):
        m = spec[f]
        if p in sel and w[sel[p]] > 0:
            expect = np.float32(np.hypot(0.5, 0.25)) * w[sel[p]]
            assert np.max(np.abs(m - expect)) <= 2e-6 * expect, (f, p)
            flat += 1
        else:
            assert not m.any(), (f, p)
    assert 0 < flat < len(positions)


def impulse_positions(rate):
    dec = rate // 625000
    # offsets inside a run, right after one, the last of the span, and the first of the next run
    return [1, 2, 3, 4, 5, 4 * dec - 1, 4 * dec, 4 * dec + 3, 4 * dec + 4, 100 * 4 * dec + 2, 255 * 4 * dec - 1,
            255 * 4 * dec + 3, 255 * 4 * dec + 4, 1024 * dec - 1]


@pytest.mark.parametrize("rate", [10_000_000, 4_000_000])
def test_host_build_impulse_selects_the_sse2_runs(rate):
    pos = impulse_positions(rate)
    hop = 1024 * (rate // 625000) + 13
    iq = impulse_input(rate, hop, len(pos), pos)
    check_impulses(R.host(iq[None], F32, rate, hop)[0], rate, pos)


# --- GPU ---------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def dec():
    d = N().NfcDecoder()
    yield d
    d.close()


def gpu_spectrum(d, samples, sigtype, rate, hop, in_dev, out_dev):
    """[streams, n, 2] IQ -> [streams, frames, 1024] through nfcb200_spectrum with each side where the flags say"""
    import torch
    a = np.array(samples, copy=True)    # writable: torch.from_numpy warns on the read-only case inputs
    nf = R.frames_of(a.shape[1], rate, hop)
    src = torch.from_numpy(a).cuda() if in_dev else a
    dst = torch.full((a.shape[0], nf, 1024), -1.0, device="cuda") if out_dev else np.full((a.shape[0], nf, 1024), -1.0, np.float32)
    torch.cuda.synchronize()
    got = d.spectrum_ptr(src.data_ptr() if in_dev else src.ctypes.data, in_dev, sigtype, a.shape[0], a.shape[1], rate, hop,
                         dst.data_ptr() if out_dev else dst.ctypes.data, out_dev, dst.numel() if out_dev else dst.size)
    assert got == nf
    return dst.cpu().numpy() if out_dev else dst


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_gpu_equals_reference_and_host_build_in_every_placement(dec, name):
    iq, rate, hop = R.case_input(name)
    outs = [gpu_spectrum(dec, iq[None], F32, rate, hop, i, o) for i in (False, True) for o in (False, True)]
    for o in outs[1:]:
        assert o.tobytes() == outs[0].tobytes()
    assert R.worst(outs[0][0], R.reference(iq, rate, hop)) <= R.TOL
    assert outs[0].tobytes() == R.host(iq[None], F32, rate, hop).tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("name", R.S16_CASES)
def test_gpu_int16_equals_float_and_reference(dec, name):
    iq, rate, hop = R.case_input(name)
    s16 = R.to_s16(iq)[None]
    outs = [gpu_spectrum(dec, s16, S16, rate, hop, i, o) for i in (False, True) for o in (False, True)]
    for o in outs[1:]:
        assert o.tobytes() == outs[0].tobytes()
    assert outs[0].tobytes() == gpu_spectrum(dec, iq[None], F32, rate, hop, True, True).tobytes()
    assert outs[0].tobytes() == R.host(s16, S16, rate, hop).tobytes()
    assert R.worst(outs[0][0], R.reference(iq, rate, hop)) <= R.TOL


@pytest.mark.gpu
def test_gpu_public_api_keeps_numpy_and_cuda_resident(dec):
    import torch
    iq, rate, hop = R.case_input("nfcb106")
    a = dec.spectrum(iq, N().SIG_IQ_F32, rate, hop)
    assert isinstance(a, np.ndarray) and a.shape == (1, R.frames_of(iq.shape[0], rate, hop), 1024)
    t = dec.spectrum(torch.from_numpy(np.array(iq)).cuda(), N().SIG_IQ_F32, rate, hop)
    assert t.is_cuda and t.device == torch.device("cuda", 0) and t.dtype == torch.float32
    assert t.cpu().numpy().tobytes() == a.tobytes()
    span = dec.spectrum(iq, N().SIG_IQ_F32, rate)        # hop=None: one frame per span
    assert span.shape[1] == N().spectrum_shape(iq.shape[0], rate)[0]
    assert span[0, 1].tobytes() == dec.spectrum(iq[16384:], N().SIG_IQ_F32, rate, 16384)[0, 0].tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("rate", [10_000_000, 4_000_000])
def test_gpu_impulse_selects_the_sse2_runs(dec, rate):
    pos = impulse_positions(rate)
    hop = 1024 * (rate // 625000) + 13
    iq = impulse_input(rate, hop, len(pos), pos)
    check_impulses(gpu_spectrum(dec, iq[None], F32, rate, hop, True, True)[0], rate, pos)


@pytest.mark.gpu
def test_gpu_stream_alone_equals_stream_in_batch(dec):
    iq, rate, hop = R.case_input("mixed")
    batch = np.stack([iq, iq[::-1], iq * np.float32(0.5), R.case_input("nfca106")[0][:iq.shape[0]]])
    hop = 4099
    together = gpu_spectrum(dec, batch, F32, rate, hop, True, True)
    for s in range(batch.shape[0]):
        assert together[s].tobytes() == gpu_spectrum(dec, batch[s:s + 1], F32, rate, hop, True, True)[0].tobytes(), s
        assert together[s].tobytes() == gpu_spectrum(dec, batch[s:s + 1], F32, rate, hop, False, False)[0].tobytes(), s


@pytest.mark.gpu
def test_gpu_large_batch_against_float64_model(dec):
    import torch
    streams, n, rate, hop = 64, 2_000_000, 10_000_000, 1000
    g = torch.Generator(device="cuda")
    g.manual_seed(3)
    t = torch.arange(n, device="cuda", dtype=torch.float64)
    tone = torch.stack([torch.cos(2 * np.pi * 211e3 / rate * t), torch.sin(2 * np.pi * 211e3 / rate * t)], dim=1).float()
    x = 0.01 * torch.randn((streams, n, 2), generator=g, device="cuda") + 0.3 * tone[None]
    out = dec.spectrum(x, N().SIG_IQ_F32, rate, hop)
    nf = R.frames_of(n, rate, hop)
    assert out.shape == (streams, nf, 1024) and streams * nf > 65535
    host_x = x.cpu().numpy()
    host_out = out.cpu().numpy()
    for s in range(streams):
        assert R.worst(host_out[s], R.model(host_x[s], rate, hop)) <= R.TOL, s


def call(d, samples=None, on_dev=0, sigtype=F32, n_streams=1, n_samples=20000, rate=10_000_000, hop=1024, out=None, out_dev=0, cap=0,
         handle=True):
    lib = d._lib
    nf = C.c_uint64(12345)
    rc = lib.nfcb200_spectrum(d._h if handle else None, None if samples is None else C.c_void_p(samples), on_dev, sigtype, n_streams, n_samples,
                              rate, hop, None if out is None else C.c_void_p(out), out_dev, cap, C.byref(nf))
    return rc, nf.value


@pytest.mark.gpu
def test_gpu_error_paths(dec):
    iq = np.zeros((2, 20000, 2), dtype=np.float32)
    out = np.full(2 * 2 * 1024, 7.0, dtype=np.float32)   # 2 frames of hop 1024 per stream at 10 MS/s
    p, o = iq.ctypes.data, out.ctypes.data
    assert call(dec, p, out=o, cap=out.size, handle=False)[0] == -2
    for sig in (0, 5, -1):
        assert call(dec, p, sigtype=sig, out=o, cap=out.size)[0] == -2
    assert call(dec, None, out=o, cap=out.size)[0] == -2
    assert call(dec, p, n_streams=0, out=o, cap=out.size)[0] == -2
    assert call(dec, p, n_samples=0, out=o, cap=out.size)[0] == -2
    assert call(dec, p, hop=0, out=o, cap=out.size)[0] == -2
    assert call(dec, p, out=None, cap=out.size)[0] == -2
    for sig in (N().SIG_MAG_F32, N().SIG_MAG_S16):
        assert call(dec, p, sigtype=sig, out=o, cap=out.size)[0] == -5
    assert call(dec, p, rate=624_999, out=o, cap=out.size)[0] == -5
    # too little room: the frame count comes back, nothing is written
    assert call(dec, p, n_streams=2, out=o, cap=out.size - 1) == (-4, 4)
    assert (out == 7.0).all()
    assert call(dec, p, n_streams=2, out=None, cap=0) == (-4, 4)
    # a stream shorter than the span: no frames
    assert call(dec, p, n_streams=2, n_samples=16383, out=None, cap=0) == (0, 0)
    assert call(dec, p, n_streams=2, n_samples=20000, hop=2000, out=o, cap=out.size) == (0, 2)
    assert (out[:2 * 2 * 1024] != 7.0).any()
    with pytest.raises(N().NfcB200Error) as e:
        dec.spectrum(iq[0, :, 0], N().SIG_MAG_F32, 10_000_000, 1024)
    assert e.value.code == -5


def device_records(d):
    import torch
    from nfc_laboratory_b200.dist import _DevView
    rp, n, ep, ne = d.device_frames()
    rec = torch.as_tensor(_DevView(rp, n * 128), device="cuda").cpu().numpy().tobytes() if n else b""
    ext = torch.as_tensor(_DevView(ep, ne * 128), device="cuda").cpu().numpy().tobytes() if ne else b""
    return (rp, n, ep, ne, rec, ext)


@pytest.mark.gpu
def test_gpu_spectrum_leaves_the_batch_decode_state_alone():
    mag, rate, _ = U.fixture_wav("test_POLL_ABF_001")
    iq = np.stack([mag, np.zeros_like(mag)], axis=1)
    d = N().NfcDecoder()
    try:
        frames = d.decode_batch(iq[None], N().SIG_IQ_F32, rate)
        before = (device_records(d), d.block_flags().tobytes(), d.stats())
        for i_dev, o_dev in ((False, False), (True, True)):
            gpu_spectrum(d, iq[None], F32, rate, 3001, i_dev, o_dev)
        d.spectrum(iq, N().SIG_IQ_F32, rate)
        after = (device_records(d), d.block_flags().tobytes(), d.stats())
        assert after == before
        assert len(frames) > 0
    finally:
        d.close()


@pytest.mark.gpu
def test_gpu_spectrum_between_stream_pushes_changes_no_frame():
    mag, rate, _ = U.fixture_wav("test_NFC-A_106kbps_004")
    iq = np.stack([mag, np.zeros_like(mag)], axis=1).astype(np.float32)
    chunk = 65536

    def run(with_spectrum):
        d = N().NfcDecoder()
        try:
            d.setSampleRate(rate)
            got = []
            for b in range(0, iq.shape[0], chunk):
                got += d.nextFrames(iq[b:b + chunk], rate, N().SIG_IQ_F32)
                if with_spectrum:
                    d.spectrum(iq[b:b + chunk + 20000], N().SIG_IQ_F32, rate, 777)
            got += d.nextFrames(None, rate, N().SIG_IQ_F32)
            return [f.key() for f in got]
        finally:
            d.close()

    plain = run(False)
    assert len(plain) > 0
    assert run(True) == plain
