"""Torch tensors as batch input of NfcDecoder.decode_batch, spectrum and iso7816_decode.

A tensor is passed to the library by address, so its dtype must be the one the signal type names (float32 or int16) and
it must lie on the host or on the decoder's device; anything else is refused before the library reads a byte."""
import pytest

import nfc_laboratory_b200 as N

RATE = 10_000_000


def _inputs():
    """(method, signal type, sample shape, the dtype the signal type takes, a dtype it does not take)"""
    import torch
    f32, s16, f64 = torch.float32, torch.int16, torch.float64
    return [
        ("decode_batch", N.SIG_MAG_F32, (2, 4096), f32, f64),
        ("decode_batch", N.SIG_MAG_S16, (2, 4096), s16, f32),
        ("decode_batch", N.SIG_IQ_F32, (2, 4096, 2), f32, s16),
        ("spectrum", N.SIG_IQ_F32, (2, 32768, 2), f32, f64),
        ("spectrum", N.SIG_IQ_S16, (2, 32768, 2), s16, f32),
        ("iso7816_decode", N.SIG_LOGIC_F32, (2, 4096, 4), f32, s16),
        ("iso7816_decode", N.SIG_LOGIC_S16, (2, 4096, 4), s16, f32),
    ]


@pytest.mark.gpu
@pytest.mark.parametrize("device", ["cpu", "cuda:0"])
def test_tensor_of_the_wrong_dtype_is_refused(device):
    import torch
    d = N.NfcDecoder(device=0)
    try:
        for method, sigtype, shape, right, wrong in _inputs():
            with pytest.raises(N.NfcB200Error, match="takes torch"):
                getattr(d, method)(torch.zeros(shape, dtype=wrong, device=device), sigtype, RATE)
            getattr(d, method)(torch.zeros(shape, dtype=right, device=device), sigtype, RATE)
    finally:
        d.close()


@pytest.mark.gpu
def test_tensor_on_another_device_is_refused():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    d = N.NfcDecoder(device=0)
    try:
        for method, sigtype, shape, right, _ in _inputs():
            with pytest.raises(N.NfcB200Error, match="decoder on cuda:0"):
                getattr(d, method)(torch.zeros(shape, dtype=right, device="cuda:1"), sigtype, RATE)
    finally:
        d.close()
