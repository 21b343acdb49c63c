"""nfc_laboratory_b200 -- H100-native NFC IQ demodulation path (drop-in for lab::NfcDecoder of josevcm/nfc-laboratory).

The product is the C-ABI shared library ``libnfcb200.so`` (hand-written sm_90a CUDA, see ``csrc/`` and
``include/nfcb200.h``).  This package is the thin Python binding used by the tests and the benchmark; it holds no
decoding logic and there is no CPU fallback: importing works anywhere, decoding needs the library and a CUDA device.
"""
from .binding import (  # noqa: F401
    Frame,
    NfcB200Error,
    NfcDecoder,
    SIGNAL_POINT_DTYPE,
    SIG_IQ_F32,
    SIG_IQ_S16,
    SIG_LOGIC_F32,
    SIG_LOGIC_S16,
    SIG_LOGIC_U8,
    SIG_MAG_F32,
    SIG_MAG_S16,
    library_path,
    load_library,
    spectrum_shape,
)
from .logic_wav import LogicWav, read_logic_wav, write_logic_wav  # noqa: F401

__all__ = ["Frame", "NfcB200Error", "NfcDecoder", "SIG_IQ_F32", "SIG_MAG_F32", "SIG_MAG_S16", "SIG_IQ_S16", "SIG_LOGIC_F32", "SIG_LOGIC_S16",
           "SIG_LOGIC_U8", "SIGNAL_POINT_DTYPE", "LogicWav", "read_logic_wav", "write_logic_wav", "library_path",
           "load_library", "spectrum_shape"]
