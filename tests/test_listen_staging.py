"""The locked NFC-A 106 kbps listen decoder reads its ring taps from the stage (nfc_core.h Machine::stage_advance), and
every staged tap it uses equals the ring word it stands for.  Host build of the lane machine with NFCB200_CHECK_TAPS
(tests/native/listen_taps.cpp), run over the NFC-A 106 kbps captures.  Without the first check the staging could
silently never fire while every decode still matched the reference."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import nfcutil as U

NAMES = [n for n in U.fixture_names() if n.startswith("test_NFC-A_106kbps")]


@pytest.fixture(scope="module")
def taps_lib(tmp_path_factory):
    src = os.path.join(U.ROOT, "tests", "native", "listen_taps.cpp")
    so = str(tmp_path_factory.mktemp("listen_taps") / "liblistentaps.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-msse2", "-mfpmath=sse", "-ffp-contract=off", "-shared", "-fPIC", src, "-o", so])
    lib = C.CDLL(so)
    lib.hostsim_run.restype = C.c_long
    lib.hostsim_run.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                C.c_void_p, C.c_void_p, C.POINTER(U.SimFrame), C.c_long, C.POINTER(U.SimResult), C.c_void_p, C.c_uint32]
    lib.hostsim_taps.argtypes = [C.POINTER(C.c_ulonglong)]
    return lib


def run_counted(lib, mag, rate, cap=65536):
    """one lane over the whole capture; (frames, staged taps used, differing, used by stage kind)"""
    mag = np.ascontiguousarray(mag, dtype=np.float32)
    buf = (U.SimFrame * cap)()
    res = U.SimResult()
    lib.hostsim_taps_clear()
    n = lib.hostsim_run(mag.ctypes.data, mag.size, rate, 0xF, 0, 0, 0, None, None, buf, cap, C.byref(res), None, 256)
    assert 0 <= n <= cap
    counts = (C.c_ulonglong * 10)()
    lib.hostsim_taps(counts)
    frames = [U.frame_tuple(f.tech, f.type, f.flags, f.phase, f.rate, f.start, f.end, bytes(f.data[:f.len])) for f in buf[:n]]
    return frames, counts[0], counts[1], list(counts[2:])


def test_there_are_nfca_106k_captures():
    assert len(NAMES) >= 4


@pytest.mark.parametrize("name", NAMES)
def test_listen_taps_are_staged_and_equal_the_ring(taps_lib, name):
    mag, rate, _ = U.fixture_wav(name)
    frames, used, differ, by_kind = run_counted(taps_lib, mag, rate)

    listen = by_kind[taps_lib.hostsim_kind_listen106()]
    assert listen > 0, "the 106 kbps listen decoder never read a staged tap"
    assert by_kind[taps_lib.hostsim_kind_poll106()] > 0
    assert differ == 0, "%d of %d staged taps differ from the ring" % (differ, used)

    # the check build decodes what the plain host build decodes
    assert frames == U.sim_run(mag, rate)[0]
