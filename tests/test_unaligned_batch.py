"""Batches whose stream pitch is not a multiple of 16 bytes.

The screening kernel stages tiles with cp.async.bulk only when the batch's base pointer and stream pitch are 16-byte
aligned; otherwise it stages them with plain loads, and a stream after the first then starts off a 16-byte boundary.
Those loads must not assume alignment: each stream of such a batch decodes as it does alone."""
import numpy as np
import pytest

import nfcutil as U
import nfc_laboratory_b200 as N


@pytest.mark.gpu
def test_unaligned_stream_pitch_decodes_each_stream_as_alone():
    mag, rate, _ = U.fixture_wav("test_NFC-A_106kbps_001")
    n = len(mag) - len(mag) % 4 + 3           # float samples: the pitch is 4 bytes past a multiple of 16
    assert (n * 4) % 16
    batch = np.stack([mag[:n], mag[:n][::-1].copy(), mag[:n]])
    d = N.NfcDecoder(device=0)
    together = d.decode_batch(batch, N.SIG_MAG_F32, rate)
    alone = []
    for i in range(len(batch)):
        alone += [N.Frame((i,) + tuple(f[1:])) for f in d.decode_batch(batch[i], N.SIG_MAG_F32, rate)]
    d.close()
    assert together == alone
    assert {f.stream for f in together} == {0, 1, 2}
