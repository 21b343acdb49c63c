"""The reference's logic capture files: 8-bit PCM WAVs with a META chunk, as hw::RecordDevice writes them for
SignalStorageTask::writeLogic and reads them back for readLogic (RecordDevice.cpp:350-491).  Plain numpy, no device.

    wav = read_logic_wav("logic-20240101.wav")
    frames = dec.iso7816_push(wav.samples, SIG_LOGIC_U8, wav.sample_rate)
"""
import collections
import os
import struct

import numpy as np

HEADER_BYTES = 92  # RIFF 12 + fmt 24 + META 48 + data 8, the header RecordDevice writes (FILEHeader)
META_KEYS = 8

LogicWav = collections.namedtuple("LogicWav", "samples sample_rate epoch keys")
LogicWav.__doc__ = """samples: uint8 [n, channels], a read-only view of the file; sample_rate in S/s; epoch: the capture's start in
seconds since 1970 (the META chunk's, else the file's ctime, as RecordDevice); keys: the META chunk's 8 channel keys"""


def read_logic_wav(path):
    """An 8-bit logic WAV as RecordDevice::readHeader reads it: RIFF / WAVE, then chunks in any order -- `fmt ` (16 bytes,
    PCM only), `META` (40 bytes starting with `meta`: epoch and 8 channel keys; other META chunks are skipped), anything
    else skipped -- up to `data`, whose samples run to the end of the file as RecordDevice reads them.  Anything but 8 bits
    per sample is refused, as SignalStorageTask refuses it as a logic file (16-bit files are radio captures)."""
    size = os.path.getsize(path)
    with open(path, "rb") as f:
        def read(n):
            b = f.read(n)
            if len(b) != n:
                raise ValueError("%s: truncated header" % path)
            return b

        riff, _, wave = struct.unpack("<4sI4s", read(12))
        if riff != b"RIFF" or wave != b"WAVE":
            raise ValueError("%s: not a RIFF / WAVE file" % path)
        fmt, epoch, keys = None, 0, (0,) * META_KEYS
        while True:
            head = f.read(8)
            if len(head) != 8:
                raise ValueError("%s: no data chunk" % path)
            cid, csize = struct.unpack("<4sI", head)
            if cid == b"fmt ":
                if csize != 16:
                    raise ValueError("%s: fmt chunk of %d bytes" % (path, csize))
                fmt = struct.unpack("<HHIIHH", read(16))
                if fmt[0] != 1:
                    raise ValueError("%s: audio format %d is not PCM" % (path, fmt[0]))
                continue
            if cid == b"META" and csize == 4 + 4 + 4 * META_KEYS:
                body = read(csize)
                if body[:4] == b"meta":
                    epoch = struct.unpack_from("<I", body, 4)[0]
                    keys = struct.unpack_from("<%di" % META_KEYS, body, 8)
                continue
            if cid == b"data":
                break
            f.seek(csize, os.SEEK_CUR)
        offset = f.tell()
    if fmt is None:
        raise ValueError("%s: data before a fmt chunk" % path)
    _, channels, rate, _, _, bits = fmt
    if bits != 8:
        raise ValueError("%s: %d bits per sample; logic captures have 8" % (path, bits))
    if channels == 0:
        raise ValueError("%s: 0 channels" % path)
    if epoch == 0:  # RecordDevice: "the file does not have a timestamp stored, it will default to the creation date"
        epoch = int(os.stat(path).st_ctime)
    n = (size - offset) // channels
    if n == 0:
        samples = np.empty((0, channels), dtype=np.uint8)
    else:
        samples = np.memmap(path, dtype=np.uint8, mode="r", offset=offset, shape=(n, channels))
    return LogicWav(samples, int(rate), int(epoch), tuple(int(k) for k in keys))


def logic_bytes(x):
    """float samples in [0, 1] as RecordDevice::writeScaledSamples stores them in 8 bits: (unsigned char) (x * 255.f)"""
    x = np.asarray(x, dtype=np.float32)
    if not np.all((x >= 0) & (x <= 1)):
        raise ValueError("8-bit logic samples are written from values in [0, 1]")
    return (x * np.float32(255)).astype(np.uint8)


def write_logic_wav(path, samples, sample_rate, epoch, keys=()):
    """Write [n, channels] samples (uint8 as they are, float in [0, 1] as RecordDevice converts them) into the file
    RecordDevice writes in Write mode with sample size 8: its 92-byte header, then the samples."""
    a = np.ascontiguousarray(samples if np.asarray(samples).dtype == np.uint8 else logic_bytes(samples), dtype=np.uint8)
    if a.ndim != 2:
        raise ValueError("logic samples must be [n_samples, channels]")
    n, channels = a.shape
    k = [int(v) for v in list(keys)[:channels]]
    k += [0] * (META_KEYS - len(k))
    data = a.size
    header = struct.pack("<4sI4s", b"RIFF", HEADER_BYTES + data - 8, b"WAVE")
    header += struct.pack("<4sIHHIIHH", b"fmt ", 16, 1, channels, sample_rate, channels * sample_rate, channels, 8)
    header += struct.pack("<4sI4sI%di" % META_KEYS, b"META", 4 + 4 + 4 * META_KEYS, b"meta", epoch, *k)
    header += struct.pack("<4sI", b"data", data)
    assert len(header) == HEADER_BYTES
    with open(path, "wb") as f:
        f.write(header)
        f.write(a.tobytes())
