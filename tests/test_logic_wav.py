"""The reference's 8-bit logic WAVs on the host: the Python writer reproduces the files the reference's RecordDevice writes
(SHA-256 recorded in tests/golden/ref_iso7816_u8.json.xz), read_logic_wav reads them back as RecordDevice does, and the
host build of the ISO 7816 stream, fed b / 255.f in SignalStorageTask::readLogic's 65 536-sample buffers, gives the
reference's frames for them."""
import os

import numpy as np
import pytest

import iso_stream_ref as T
import logic_ref as L
import nfc_laboratory_b200 as N

IDS = [L.case_id(c) for c in L.CASES]


@pytest.mark.parametrize("case", L.CASES, ids=IDS)
def test_writer_matches_recorded_wav(case, tmp_path):
    path = str(tmp_path / "logic.wav")
    L.write(path, case)
    assert L.sha256(path) == L.golden()[L.case_id(case)]["sha256"]


@pytest.mark.parametrize("case", [c for c in L.CASES if c[0][1] == 10_000_000], ids=lambda c: L.case_id(c))
def test_read_logic_wav_round_trip(case, tmp_path):
    path = str(tmp_path / "logic.wav")
    L.write(path, case)
    wav = N.read_logic_wav(path)
    assert wav.sample_rate == case[0][1] and wav.epoch == L.EPOCH
    assert wav.keys == L.KEYS[:case[1]] + (0,) * (8 - case[1])
    assert wav.samples.dtype == np.uint8 and wav.samples.shape == (len(L.samples(case)), case[1])
    assert np.array_equal(wav.samples, L.u8(case))
    lib = L.ref_lib()
    if lib is not None:  # the reference's reader sees the same file
        rate, ch, epoch, keys, x = L.ref_read(lib, path, len(wav.samples))
        assert (rate, ch, epoch, keys) == (wav.sample_rate, case[1], wav.epoch, wav.keys)
        assert np.array_equal(x, L.as_float(wav.samples))


def test_reference_writer_matches(tmp_path):
    lib = L.ref_lib()
    if lib is None:
        pytest.skip("the reference's RecordDevice was not built here")
    for case in L.CASES[::7]:
        a, b = str(tmp_path / "ref.wav"), str(tmp_path / "py.wav")
        L.ref_write(lib, a, case)
        L.write(b, case)
        assert L.sha256(a) == L.sha256(b) == L.golden()[L.case_id(case)]["sha256"]


def test_read_logic_wav_refuses(tmp_path):
    path = str(tmp_path / "x.wav")
    N.write_logic_wav(path, np.zeros((10, 4), dtype=np.uint8), 10_000_000, 1)
    raw = bytearray(open(path, "rb").read())
    raw[34:36] = (16).to_bytes(2, "little")  # 16 bits per sample: a radio file
    open(path, "wb").write(raw)
    with pytest.raises(ValueError):
        N.read_logic_wav(path)
    raw[34:36], raw[20:22] = (8).to_bytes(2, "little"), (3).to_bytes(2, "little")  # not PCM
    open(path, "wb").write(raw)
    with pytest.raises(ValueError):
        N.read_logic_wav(path)
    with pytest.raises(ValueError):
        N.write_logic_wav(path, np.full((4, 4), 1.5, dtype=np.float32), 10_000_000, 1)


def test_read_logic_wav_skips_unknown_chunks_and_defaults_epoch(tmp_path):
    path = str(tmp_path / "x.wav")
    x = np.arange(40, dtype=np.uint8).reshape(8, 5)
    N.write_logic_wav(path, x, 1_000_000, 0)
    raw = open(path, "rb").read()
    # an unknown chunk before the data chunk, as RecordDevice skips it; epoch 0: the file's ctime
    raw = raw[:84] + b"junk" + (6).to_bytes(4, "little") + b"abcdef" + raw[84:]
    open(path, "wb").write(raw)
    wav = N.read_logic_wav(path)
    assert np.array_equal(wav.samples, x) and wav.epoch == int(os.stat(path).st_ctime)


@pytest.mark.parametrize("case", [c for c in L.CASES if c[1] == 4], ids=lambda c: L.case_id(c))
def test_host_stream_equals_golden(case):
    """the host build of the push over b / 255.f at 65 536-sample buffers equals the replayed reference (it reads channels
    0-3, the same bytes at every channel count, whose recorded frames are equal: test_iso7816_u8.py)"""
    iso, ch = case
    x = L.as_float(L.u8(case))[:, :4]
    c = L.chunks(len(x))
    assert T.host(x, c, [iso[1]] * len(c), stream_time=L.EPOCH) == L.expected(case)
