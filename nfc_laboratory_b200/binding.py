"""ctypes binding of include/nfcb200.h.

``NfcDecoder`` mirrors the method names of the reference's ``lab::NfcDecoder``
(src/nfc-lib/lib-lab/lab-radio/src/main/include/lab/nfc/NfcDecoder.h:33-122) so that tests read like the reference's own
harness (src/nfc-test/test-sdr/src/main/cpp/main.cpp:141-180): construct, setEnableNfcX, nextFrames(buffer).
"""
import ctypes as C
import math
import os

import numpy as np

SIG_IQ_F32 = 1
SIG_MAG_F32 = 2
SIG_MAG_S16 = 3
SIG_IQ_S16 = 4
SIG_LOGIC_F32 = 5
SIG_LOGIC_S16 = 6
SIG_LOGIC_U8 = 7

_HERE = os.path.dirname(os.path.abspath(__file__))


class NfcB200Error(RuntimeError):
    def __init__(self, code, message):
        super().__init__("nfcb200 error %d: %s" % (code, message))
        self.code = code


class CFrame(C.Structure):
    _fields_ = [
        ("stream", C.c_uint32), ("tech_type", C.c_uint32), ("frame_type", C.c_uint32), ("frame_flags", C.c_uint32),
        ("frame_phase", C.c_uint32), ("frame_rate", C.c_uint32), ("length", C.c_uint32), ("reserved", C.c_uint32),
        ("sample_start", C.c_uint64), ("sample_end", C.c_uint64), ("sample_rate", C.c_uint64),
        ("time_start", C.c_double), ("time_end", C.c_double), ("date_time", C.c_double),
        ("data", C.c_uint8 * 512),
    ]


class CConfig(C.Structure):
    _fields_ = [
        ("device", C.c_int), ("enabled", C.c_uint32), ("power_level_threshold", C.c_float),
        ("correlation_threshold", C.c_float * 4), ("modulation_min", C.c_float * 4), ("modulation_max", C.c_float * 4),
        ("stream_time", C.c_uint32), ("use_tma", C.c_uint32), ("max_rounds", C.c_uint32), ("segments_per_lane", C.c_uint32),
        ("exact", C.c_uint32), ("reserved", C.c_uint32 * 3),
    ]


class CStats(C.Structure):
    _fields_ = [
        ("samples", C.c_uint64), ("blocks", C.c_uint64), ("active_blocks", C.c_uint64), ("segments", C.c_uint64), ("lanes", C.c_uint64),
        ("live_lanes", C.c_uint64), ("lane_runs", C.c_uint64), ("lane_samples", C.c_uint64), ("rounds", C.c_uint64),
        ("frames", C.c_uint64), ("kernel_launches", C.c_uint64),
        ("ms_h2d", C.c_float), ("ms_screen", C.c_float), ("ms_segment", C.c_float), ("ms_lanes", C.c_float),
        ("ms_gather", C.c_float), ("ms_total", C.c_float), ("ms_wall", C.c_float),
        ("ms_front", C.c_float), ("straggler_lanes", C.c_float), ("feature_samples", C.c_uint64),
    ]


class Frame(tuple):
    """(stream, tech_type, frame_type, frame_flags, frame_phase, frame_rate, sample_start, sample_end, data)"""
    __slots__ = ()

    stream = property(lambda s: s[0])
    tech_type = property(lambda s: s[1])
    frame_type = property(lambda s: s[2])
    frame_flags = property(lambda s: s[3])
    frame_phase = property(lambda s: s[4])
    frame_rate = property(lambda s: s[5])
    sample_start = property(lambda s: s[6])
    sample_end = property(lambda s: s[7])
    data = property(lambda s: s[8])

    def key(self):
        """the fields RawFrame::operator== compares (lab-data RawFrame.cpp:82-98), without the stream index"""
        return tuple(self[1:])


# entry points of include/nfcb200.h whose names are letters and underscores; nfcb200_iso7816_decode_batch is bound below
EXPORTS = [
    "nfcb200_config_default", "nfcb200_create", "nfcb200_destroy", "nfcb200_configure", "nfcb200_decode_batch",
    "nfcb200_stream_push", "nfcb200_stream_reset", "nfcb200_get_stats", "nfcb200_get_block_flags", "nfcb200_pack_frames",
    "nfcb200_last_error", "nfcb200_version", "nfcb200_device_frames", "nfcb200_emit_records", "nfcb200_stream_pending", "nfcb200_debug_trace", "nfcb200_carry_size", "nfcb200_set_carry",
    "nfcb200_carry_before", "nfcb200_default_carry", "nfcb200_spectrum", "nfcb200_spectrum_shape",
    "nfcb200_adaptive_radio", "nfcb200_adaptive_logic",
]

# nfcb200_signal_point: one point of the adaptive signal (NfcDecoder.adaptive_radio / adaptive_logic)
SIGNAL_POINT_DTYPE = np.dtype([("stream", "<u4"), ("channel", "<u4"), ("sample", "<u8"), ("value", "<f4"), ("reserved", "<u4")])
ADAPTIVE_BUFFER = 65536  # samples per buffer of a replayed file (SignalStorageTask.cpp:323-437)

SPECTRUM_BINS = 1024


def library_path():
    return os.path.join(_HERE, "libnfcb200.so")


_lib = None


def load_library():
    """load libnfcb200.so (built in-tree by __graft_entry__.build() / csrc/Makefile); fails loudly when it is missing"""
    global _lib
    if _lib is not None:
        return _lib
    path = library_path()
    if not os.path.exists(path):
        raise NfcB200Error(-1, "CUDA library %s is missing: run `python -c 'import __graft_entry__ as g; g.build()'`; "
                               "there is no CPU fallback" % path)
    lib = C.CDLL(path)
    lib.nfcb200_last_error.restype = C.c_char_p
    lib.nfcb200_version.restype = C.c_char_p
    lib.nfcb200_config_default.argtypes = [C.POINTER(CConfig)]
    lib.nfcb200_create.argtypes = [C.POINTER(CConfig), C.POINTER(C.c_void_p)]
    lib.nfcb200_destroy.argtypes = [C.c_void_p]
    lib.nfcb200_configure.argtypes = [C.c_void_p, C.POINTER(CConfig)]
    lib.nfcb200_decode_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_uint32, C.c_uint64, C.c_uint32,
                                         C.POINTER(CFrame), C.c_uint64, C.POINTER(C.c_uint64)]
    lib.nfcb200_stream_push.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_uint64, C.c_uint32, C.POINTER(CFrame), C.c_uint64,
                                        C.POINTER(C.c_uint64)]
    lib.nfcb200_stream_reset.argtypes = [C.c_void_p]
    lib.nfcb200_get_stats.argtypes = [C.c_void_p, C.POINTER(CStats)]
    lib.nfcb200_get_block_flags.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    lib.nfcb200_pack_frames.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    lib.nfcb200_carry_size.restype = C.c_int
    lib.nfcb200_default_carry.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    lib.nfcb200_set_carry.argtypes = [C.c_void_p, C.c_char_p, C.c_uint64, C.c_uint32]
    lib.nfcb200_carry_before.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    lib.nfcb200_device_frames.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64), C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
    lib.nfcb200_emit_records.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.POINTER(CFrame),
                                         C.c_uint64, C.POINTER(C.c_uint64)]
    lib.nfcb200_spectrum.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint64, C.c_void_p, C.c_int,
                                     C.c_uint64, C.POINTER(C.c_uint64)]
    lib.nfcb200_iso7816_decode_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_uint32, C.c_uint64, C.c_uint32,
                                                 C.POINTER(CFrame), C.c_uint64, C.POINTER(C.c_uint64)]
    lib.nfcb200_iso7816_stream_push.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_uint64, C.c_uint32, C.POINTER(CFrame), C.c_uint64,
                                                C.POINTER(C.c_uint64)]
    lib.nfcb200_iso7816_decode_batch_ch.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint32,
                                                    C.POINTER(CFrame), C.c_uint64, C.POINTER(C.c_uint64)]
    lib.nfcb200_iso7816_stream_push_ch.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_uint32, C.c_uint64, C.c_uint32, C.POINTER(CFrame),
                                                   C.c_uint64, C.POINTER(C.c_uint64)]
    lib.nfcb200_iso7816_stream_pending.argtypes = [C.c_void_p, C.POINTER(CFrame), C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    lib.nfcb200_iso7816_stream_reset.argtypes = [C.c_void_p]
    lib.nfcb200_adaptive_radio.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint64,
                                           C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    lib.nfcb200_adaptive_logic.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint32,
                                           C.c_uint64, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    lib.nfcb200_spectrum_shape.argtypes = [C.c_uint64, C.c_uint32, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
    _lib = lib
    return lib


def _check(lib, rc):
    if rc != 0:
        raise NfcB200Error(rc, lib.nfcb200_last_error().decode("utf-8", "replace"))


def spectrum_shape(n_samples, sample_rate, hop=None):
    """(frames per stream, decimation) of NfcDecoder.spectrum for streams of n_samples; hop=None is the span, 1024 x decimation"""
    lib = load_library()
    nf, dec = C.c_uint64(0), C.c_uint32(0)
    _check(lib, lib.nfcb200_spectrum_shape(int(n_samples), int(sample_rate), 1, None, C.byref(dec)))
    hop = SPECTRUM_BINS * dec.value if hop is None else int(hop)
    _check(lib, lib.nfcb200_spectrum_shape(int(n_samples), int(sample_rate), hop, C.byref(nf), None))
    return int(nf.value), int(dec.value)


_SIG_DTYPE = {SIG_IQ_F32: (np.float32, 2), SIG_MAG_F32: (np.float32, 1), SIG_MAG_S16: (np.int16, 1), SIG_IQ_S16: (np.int16, 2),
              SIG_LOGIC_F32: (np.float32, 4), SIG_LOGIC_S16: (np.int16, 4), SIG_LOGIC_U8: (np.uint8, 4)}
LOGIC_CHANNELS = range(4, 9)  # channels per logic sample the ISO 7816 calls take (include/nfcb200.h)


def _logic_dtype(samples, sigtype):
    """refuse 8-bit samples with another logic format, and anything but uint8 with SIG_LOGIC_U8: a conversion would read
    the bytes b as b, not as b / 255.f"""
    if _SIG_DTYPE.get(sigtype, (None, 0))[1] != 4:
        raise NfcB200Error(-2, "signal type %d is not a logic format" % sigtype)
    dt = str(getattr(samples, "dtype", ""))
    if (sigtype == SIG_LOGIC_U8) != dt.endswith("uint8"):
        raise NfcB200Error(-2, "signal type %d takes %s samples, got %s" % (sigtype, np.dtype(_SIG_DTYPE[sigtype][0]).name, dt or type(samples).__name__))


class NfcDecoder:
    """GPU decoder handle.  Method names follow lab::NfcDecoder; batch decoding is the GPU-native addition."""

    def __init__(self, device=0, use_tma=True, segments_per_lane=0, exact=False):
        self._lib = load_library()
        self._cfg = CConfig()
        self._lib.nfcb200_config_default(C.byref(self._cfg))
        self._cfg.device = device
        self._cfg.use_tma = 1 if use_tma else 0
        self._cfg.segments_per_lane = segments_per_lane
        self._cfg.exact = 1 if exact else 0
        self._h = C.c_void_p()
        _check(self._lib, self._lib.nfcb200_create(C.byref(self._cfg), C.byref(self._h)))
        self._rate = 0
        self._frames = None
        self._cap = 0

    # --- lifecycle -------------------------------------------------------------------------------------------------
    def close(self):
        if self._h:
            self._lib.nfcb200_destroy(self._h)
            self._h = C.c_void_p()

    cleanup = close

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def initialize(self):
        """NfcDecoder::initialize: forget stream state, re-derive parameters at the next buffer"""
        self._apply()
        _check(self._lib, self._lib.nfcb200_stream_reset(self._h))

    def _apply(self):
        _check(self._lib, self._lib.nfcb200_configure(self._h, C.byref(self._cfg)))

    # --- setters / getters of lab::NfcDecoder ------------------------------------------------------------------------
    def _enable(self, bit, on):
        if on:
            self._cfg.enabled |= bit
        else:
            self._cfg.enabled &= ~bit
        self._apply()

    def setEnableNfcA(self, on): self._enable(1, on)
    def setEnableNfcB(self, on): self._enable(2, on)
    def setEnableNfcF(self, on): self._enable(4, on)
    def setEnableNfcV(self, on): self._enable(8, on)
    def isNfcAEnabled(self): return bool(self._cfg.enabled & 1)
    def isNfcBEnabled(self): return bool(self._cfg.enabled & 2)
    def isNfcFEnabled(self): return bool(self._cfg.enabled & 4)
    def isNfcVEnabled(self): return bool(self._cfg.enabled & 8)

    def setSampleRate(self, rate): self._rate = int(rate)
    def sampleRate(self): return self._rate
    def setStreamTime(self, t): self._cfg.stream_time = int(t); self._apply()
    def streamTime(self): return int(self._cfg.stream_time)
    def setPowerLevelThreshold(self, v): self._cfg.power_level_threshold = float(v); self._apply()
    def powerLevelThreshold(self): return float(self._cfg.power_level_threshold)

    def _set_thr(self, t, corr=None, mn=None, mx=None):
        # NaN leaves a value unchanged, like the reference setters (NfcA.cpp:2027-2045)
        if corr is not None and not math.isnan(corr):
            self._cfg.correlation_threshold[t] = corr
        if mn is not None and not math.isnan(mn):
            self._cfg.modulation_min[t] = mn
        if mx is not None and not math.isnan(mx):
            self._cfg.modulation_max[t] = mx
        self._apply()

    def setCorrelationThresholdNfcA(self, v): self._set_thr(0, corr=v)
    def setCorrelationThresholdNfcB(self, v): self._set_thr(1, corr=v)
    def setCorrelationThresholdNfcF(self, v): self._set_thr(2, corr=v)
    def setCorrelationThresholdNfcV(self, v): self._set_thr(3, corr=v)
    def setModulationThresholdNfcA(self, mn, mx): self._set_thr(0, mn=mn, mx=mx)
    def setModulationThresholdNfcB(self, mn, mx): self._set_thr(1, mn=mn, mx=mx)
    def setModulationThresholdNfcF(self, mn, mx): self._set_thr(2, mn=mn, mx=mx)
    def setModulationThresholdNfcV(self, mn, mx): self._set_thr(3, mn=mn, mx=mx)
    def correlationThresholdNfcA(self): return float(self._cfg.correlation_threshold[0])
    def correlationThresholdNfcB(self): return float(self._cfg.correlation_threshold[1])
    def correlationThresholdNfcF(self): return float(self._cfg.correlation_threshold[2])
    def correlationThresholdNfcV(self): return float(self._cfg.correlation_threshold[3])

    # --- decode ------------------------------------------------------------------------------------------------------
    def _buffer(self, cap):
        if cap > self._cap:
            self._frames = (CFrame * cap)()
            self._cap = cap
        return self._frames

    @staticmethod
    def _convert(buf, n):
        out = []
        for i in range(n):
            f = buf[i]
            out.append(Frame((f.stream, f.tech_type, f.frame_type, f.frame_flags, f.frame_phase, f.frame_rate,
                              int(f.sample_start), int(f.sample_end), bytes(f.data[:f.length]))))
        return out

    def _with_room(self, call, cap, raw):
        """call(buf, cap, byref(n)) of a C entry point that returns frames, again with room for all of them when the first
        buffer was too small"""
        while True:
            buf = self._buffer(cap)
            n = C.c_uint64(0)
            rc = call(buf, cap, C.byref(n))
            if rc == -4 and n.value > cap:
                cap = int(n.value) + 16
                continue
            _check(self._lib, rc)
            return (buf, n.value) if raw else self._convert(buf, n.value)

    def _batch(self, samples, sigtype):
        """(array, address, on_device) of a batch [n_streams, n_samples(, components)], or of one stream without the first
        axis, made contiguous: a numpy array is converted to the signal type's dtype; a torch tensor must have that dtype
        and lie on the host or on this decoder's device.  The library reads a CUDA tensor on its own stream, so torch's
        current stream is waited for first."""
        dtype, comps = _SIG_DTYPE[sigtype]
        one_stream = 1 if comps == 1 else 2
        if isinstance(samples, np.ndarray):
            a = np.ascontiguousarray(samples, dtype=dtype)
            a = a[None] if a.ndim == one_stream else a
            return a, a.ctypes.data, False
        import torch
        if samples.is_cuda and samples.device.index != self._cfg.device:
            raise NfcB200Error(-2, "tensor on %s, decoder on cuda:%d" % (samples.device, self._cfg.device))
        want = {np.float32: torch.float32, np.int16: torch.int16, np.uint8: torch.uint8}[dtype]
        if samples.dtype != want:
            raise NfcB200Error(-2, "signal type %d takes %s samples, got a %s tensor" % (sigtype, want, samples.dtype))
        t = samples.contiguous()
        t = t[None] if t.dim() == one_stream else t
        if t.is_cuda:
            torch.cuda.current_stream(t.device).synchronize()
        return t, t.data_ptr(), t.is_cuda

    def decode_batch_ptr(self, ptr, on_device, sigtype, n_streams, n_samples, sample_rate, cap=1 << 16, raw=False):
        """decode [n_streams][n_samples] samples at `ptr` (host or device address)"""
        return self._with_room(lambda buf, cap, n: self._lib.nfcb200_decode_batch(self._h, C.c_void_p(ptr), 1 if on_device else 0, sigtype, n_streams,
                                                                               n_samples, sample_rate, buf, cap, n), cap, raw)

    def set_carry(self, blob, clock_shift=0):
        """carry in front of the next single-stream decode (a time shard continuing a capture); None clears"""
        if blob is None:
            _check(self._lib, self._lib.nfcb200_set_carry(self._h, None, 0, 0))
        else:
            b = bytes(blob)
            _check(self._lib, self._lib.nfcb200_set_carry(self._h, b, len(b), int(clock_shift)))

    def carry_size(self):
        return int(self._lib.nfcb200_carry_size())

    def default_carry(self):
        """the carry a cold-started lane assumes in front of it (power-on protocol state, carrier on)"""
        n = self.carry_size()
        buf = C.create_string_buffer(n)
        _check(self._lib, self._lib.nfcb200_default_carry(self._h, buf, n))
        return buf.raw

    def carry_before(self, sample):
        """(carry blob, lane_begin) of the last single-stream decode: the decoder's carry in front of the first lane that
        begins at or after `sample`; lane_begin is None when no lane begins there"""
        n = self._lib.nfcb200_carry_size()
        buf = C.create_string_buffer(n)
        size, begin = C.c_uint64(0), C.c_uint64(0)
        _check(self._lib, self._lib.nfcb200_carry_before(self._h, int(sample), buf, n, C.byref(size), C.byref(begin)))
        return buf.raw, (None if begin.value == 0xFFFFFFFFFFFFFFFF else int(begin.value))

    def device_frames(self):
        """(records_ptr, n_records, ext_ptr, n_ext_chunks): the frames of the last decode_batch as they sit in device memory,
        ordered by (stream, time) -- 128-byte records + 128-byte payload extension chunks (include/nfcb200.h)"""
        rp, ep = C.c_void_p(), C.c_void_p()
        n, ne = C.c_uint64(0), C.c_uint64(0)
        _check(self._lib, self._lib.nfcb200_device_frames(self._h, C.byref(rp), C.byref(n), C.byref(ep), C.byref(ne)))
        return rp.value or 0, int(n.value), ep.value or 0, int(ne.value)

    def emit_records(self, records_ptr, n_records, ext_ptr, n_ext_chunks, stream_offset, sample_rate, raw=False):
        """gathered device-format records (HOST memory) -> frames, stream index raised by stream_offset"""
        buf = (CFrame * max(1, n_records))()
        n = C.c_uint64(0)
        _check(self._lib, self._lib.nfcb200_emit_records(self._h, C.c_void_p(records_ptr), n_records, C.c_void_p(ext_ptr), n_ext_chunks,
                                                         int(stream_offset), int(sample_rate), buf, max(1, n_records), C.byref(n)))
        return (buf, int(n.value)) if raw else self._convert(buf, int(n.value))

    def decode_batch(self, samples, sigtype, sample_rate, cap=1 << 16):
        """samples: numpy array [n_streams, n_samples(, 2)] or torch tensor of the same shape"""
        a, ptr, on_device = self._batch(samples, sigtype)
        return self.decode_batch_ptr(ptr, on_device, sigtype, int(a.shape[0]), int(a.shape[1]), sample_rate, cap)

    def spectrum(self, samples, sigtype, sample_rate, hop=None):
        """FFT spectrum of the reference's frequency view (lab::FourierProcessTask) every `hop` samples of every stream
        (hop=None: one frame per span of 1024 x decimation samples).  samples: IQ as numpy [n_streams, n_samples, 2] (or one
        stream [n_samples, 2]) -> numpy float32 [n_streams, frames, 1024]; a CUDA tensor of the same shape -> a CUDA tensor
        on the same device.  Bins run from the most negative frequency up (include/nfcb200.h nfcb200_spectrum)."""
        a, ptr, on_device = self._batch(samples, sigtype)
        n_streams, n_samples = int(a.shape[0]), int(a.shape[1])
        if hop is None:
            hop = SPECTRUM_BINS * spectrum_shape(n_samples, sample_rate)[1]
        n_frames = spectrum_shape(n_samples, sample_rate, hop)[0]
        if on_device:
            import torch
            out = torch.empty((n_streams, n_frames, SPECTRUM_BINS), dtype=torch.float32, device=a.device)
            self.spectrum_ptr(ptr, True, sigtype, n_streams, n_samples, sample_rate, hop, out.data_ptr(), True, out.numel())
        else:
            out = np.empty((n_streams, n_frames, SPECTRUM_BINS), dtype=np.float32)
            self.spectrum_ptr(ptr, False, sigtype, n_streams, n_samples, sample_rate, hop, out.ctypes.data, False, out.size)
        return out

    def spectrum_ptr(self, ptr, on_device, sigtype, n_streams, n_samples, sample_rate, hop, out_ptr, out_on_device, cap):
        """nfcb200_spectrum on raw addresses (host or device, each side as its flag says); returns the frames per stream"""
        nf = C.c_uint64(0)
        _check(self._lib, self._lib.nfcb200_spectrum(self._h, C.c_void_p(ptr), 1 if on_device else 0, sigtype, n_streams, n_samples, int(sample_rate),
                                                     int(hop), C.c_void_p(out_ptr), 1 if out_on_device else 0, int(cap), C.byref(nf)))
        return int(nf.value)

    def adaptive_radio(self, samples, sigtype, sample_rate, buffer=ADAPTIVE_BUFFER, offset=0):
        """the reference's adaptive signal of radio captures (lab::SignalResamplingTask, the GUI's signal view): numpy
        [n_streams, n_samples] magnitude or [n_streams, n_samples, 2] IQ (or one stream without the first axis), or a torch
        tensor of that shape, cut into buffers of `buffer` samples, the stream's first sample at position `offset`.
        Returns a SIGNAL_POINT_DTYPE array ordered by (stream, emission order) (include/nfcb200.h nfcb200_adaptive_radio)."""
        a, ptr, on_device = self._batch(samples, sigtype)
        n_streams, n_samples = int(a.shape[0]), int(a.shape[1])
        return self._points(lambda out, cap, n: self._lib.nfcb200_adaptive_radio(self._h, C.c_void_p(ptr), 1 if on_device else 0, sigtype, n_streams,
                                                                                 n_samples, int(sample_rate), int(buffer), int(offset), out, cap, n),
                            n_streams * n_samples)

    def adaptive_logic(self, samples, sigtype, sample_rate, channels=None, buffer=ADAPTIVE_BUFFER, offset=0):
        """the adaptive signal of logic captures [n_streams, n_samples, C] (or one stream [n_samples, C]), C = 4-8 channels
        in a logic format as iso7816_decode takes them; channels=None takes C from the shape.  Every channel but 1 (CLK) has
        points.  Returns a SIGNAL_POINT_DTYPE array ordered by (stream, channel, emission order)."""
        _logic_dtype(samples, sigtype)
        a, ptr, on_device = self._batch(samples, sigtype)
        if len(a.shape) != 3 or (channels is not None and int(channels) != a.shape[2]):
            raise NfcB200Error(-2, "logic samples must be [n_streams, n_samples, channels], got %s" % (tuple(a.shape),))
        n_streams, n_samples, ch = int(a.shape[0]), int(a.shape[1]), int(a.shape[2])
        return self._points(lambda out, cap, n: self._lib.nfcb200_adaptive_logic(self._h, C.c_void_p(ptr), 1 if on_device else 0, sigtype, ch,
                                                                                 n_streams, n_samples, int(sample_rate), int(buffer), int(offset),
                                                                                 out, cap, n),
                            n_streams * n_samples * max(1, ch - 1))

    def _points(self, call, n_in):
        """call(out, cap, byref(n)) of an adaptive entry point, again with room for every point when the first guess (a
        quiet signal keeps about one sample in 255) was too small"""
        cap = n_in // 128 + 1024
        while True:
            out = np.empty(cap, dtype=SIGNAL_POINT_DTYPE)
            n = C.c_uint64(0)
            rc = call(C.c_void_p(out.ctypes.data), cap, C.byref(n))
            if rc == -4 and n.value > cap:
                cap = int(n.value)
                continue
            _check(self._lib, rc)
            return out[: n.value]

    def iso7816_decode(self, samples, sigtype, sample_rate, cap=1 << 16, raw=False):
        """ISO 7816 contact smart-card frames (lab::IsoDecoder) of logic captures of C = 4-8 channels, IO, CLK, RST, VCC first:
        numpy [n_streams, n_samples, C] (or one stream [n_samples, C]), float32 for SIG_LOGIC_F32, int16 for SIG_LOGIC_S16,
        uint8 for SIG_LOGIC_U8 (read_logic_wav), or a torch tensor of the same shape (a CUDA tensor is decoded where it
        lies).  Channels 4 and up are read past.  Frames are ordered by (stream, time).  raw=True returns (CFrame buffer,
        count) with every field, time_start / time_end / date_time included."""
        _logic_dtype(samples, sigtype)
        a, ptr, on_device = self._batch(samples, sigtype)
        if len(a.shape) != 3 or a.shape[2] not in LOGIC_CHANNELS:
            raise NfcB200Error(-2, "logic samples must be [n_streams, n_samples, 4-8], got %s" % (tuple(a.shape),))
        n_streams, n_samples, channels = int(a.shape[0]), int(a.shape[1]), int(a.shape[2])
        return self._with_room(lambda buf, cap, n: self._lib.nfcb200_iso7816_decode_batch_ch(self._h, C.c_void_p(ptr), 1 if on_device else 0, sigtype,
                                                                                          channels, n_streams, n_samples, int(sample_rate), buf, cap, n),
                               cap, raw)

    def iso7816_push(self, samples, sigtype, sample_rate, cap=4096, raw=False):
        """lab::IsoDecoder::nextFrames(SignalBuffer) of one buffer of a live logic capture [n_samples, C], C = 4-8 channels
        (numpy, float32 for SIG_LOGIC_F32, int16 for SIG_LOGIC_S16, uint8 for SIG_LOGIC_U8): the frames it completes,
        every pending one included.  The decoder carries over to the next push, whatever its format and channel count; a
        push at another sample rate restarts it.  Frames as iso7816_decode returns them; raw=True gives a list of CFrame
        with every field."""
        _logic_dtype(samples, sigtype)
        a = np.ascontiguousarray(samples, dtype=_SIG_DTYPE[sigtype][0])
        if a.ndim != 2 or a.shape[1] not in LOGIC_CHANNELS:
            raise NfcB200Error(-2, "logic samples must be [n_samples, 4-8], got %s" % (a.shape,))
        if a.shape[0] == 0:
            return self.iso7816_flush(cap, raw)
        return self._iso_stream(lambda buf, cap, n: self._lib.nfcb200_iso7816_stream_push_ch(self._h, a.ctypes.data, sigtype, a.shape[1], a.shape[0],
                                                                                             int(sample_rate), buf, cap, n), cap, raw)

    def iso7816_flush(self, cap=4096, raw=False):
        """nextFrames({}) on the ISO stream: it decodes nothing (IsoTech.cpp:31-32); frames still pending are returned"""
        return self._iso_stream(lambda buf, cap, n: self._lib.nfcb200_iso7816_stream_push(self._h, None, SIG_LOGIC_F32, 0, 0, buf, cap, n), cap, raw)

    def iso7816_reset(self):
        """forget the ISO stream: the next push decodes as on a fresh decoder"""
        _check(self._lib, self._lib.nfcb200_iso7816_stream_reset(self._h))

    def _iso_stream(self, call, cap, raw):
        """call(buf, cap, byref(n)) of an ISO stream push, then its pending frames until none is left"""
        buf = (CFrame * cap)()
        n = C.c_uint64(0)
        rc = call(buf, cap, C.byref(n))
        if rc != -4:
            _check(self._lib, rc)
        frames = [CFrame.from_buffer_copy(f) for f in buf[:n.value]] if raw else self._convert(buf, n.value)
        left = C.c_uint64(1 if rc == -4 else 0)
        while left.value:
            _check(self._lib, self._lib.nfcb200_iso7816_stream_pending(self._h, buf, cap, C.byref(n), C.byref(left)))
            frames += [CFrame.from_buffer_copy(f) for f in buf[:n.value]] if raw else self._convert(buf, n.value)
        return frames

    def nextFrames(self, samples, sample_rate=None, sigtype=SIG_MAG_F32, cap=4096):
        """NfcDecoder::nextFrames(SignalBuffer): streaming decode of one capture.  samples=None (an invalid buffer in the
        reference, NfcDecoder.cpp:449-463) flushes.  Every frame the buffer completes is returned, however many: `cap` is
        only the size of each copy out of the library."""
        rate = int(sample_rate or self._rate or 0)
        cap = max(1, int(cap))
        buf = self._buffer(cap)
        n = C.c_uint64(0)
        if samples is None:
            rc = self._lib.nfcb200_stream_push(self._h, None, sigtype, 0, rate, buf, cap, C.byref(n))
        else:
            dtype, comps = _SIG_DTYPE[sigtype]
            a = np.ascontiguousarray(samples, dtype=dtype)
            count = a.size // comps
            rc = self._lib.nfcb200_stream_push(self._h, a.ctypes.data, sigtype, count, rate, buf, cap, C.byref(n))
        if rc != -4:
            _check(self._lib, rc)
        self._rate = rate
        # more frames than cap: the push delivered cap of them, the rest wait in nfcb200_stream_pending
        frames = self._convert(buf, n.value)
        left = C.c_uint64(1 if rc == -4 else 0)
        while left.value:
            _check(self._lib, self._lib.nfcb200_stream_pending(self._h, buf, cap, C.byref(n), C.byref(left)))
            frames += self._convert(buf, n.value)
        return frames

    def stats(self):
        s = CStats()
        _check(self._lib, self._lib.nfcb200_get_stats(self._h, C.byref(s)))
        return {name: getattr(s, name) for name, _ in CStats._fields_}

    def block_flags(self):
        nb = C.c_uint64(0)
        _check(self._lib, self._lib.nfcb200_get_block_flags(self._h, None, 0, C.byref(nb)))
        st = self.stats()
        streams = int(st["blocks"] // max(1, nb.value))
        out = np.zeros((streams, nb.value), dtype=np.uint8)
        _check(self._lib, self._lib.nfcb200_get_block_flags(self._h, out.ctypes.data, out.size, C.byref(nb)))
        return out
