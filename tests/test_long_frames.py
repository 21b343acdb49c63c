"""Long frames against the reference on every frame field: NFC-A I-blocks of 1 to 513 bytes at 106 / 212 / 424 kbps (the
edges of the 80-byte inline payload, of each 128-byte extension chunk and of the 512-byte frame buffer), frames around the
frame-size limit a RATS, ATQB or ATTRIB negotiates (in the RATS's lane and in a later lane, which starts from the default
limit until the carry chain corrects it), the limit 0 of FSDI 13, NFC-F frames up to 257 bytes, a dense batch of such
streams, and pushes that overflow the stream's initial frame pool.

CPU: the recorded reference output equals the live reference; the captures decode to what they were built with; the host
build of the lane machine, the segment pipeline and the warp-lane pipeline equal the reference; the record parser.
GPU: decode_batch in thread lanes, exact warp lanes and through the straggler hand-over, float and int16; the dense batch,
its packed device records and their conversion (emit_records, a two-rank gather); the stream in whole, 65 536-sample and
1-63-sample pushes; single pushes of more than 2^14 frames and of more than 2^12 extension chunks; a frame past 512 bytes."""
import json
import os

import numpy as np
import pytest

import long_frames as L
import nfc_stream_ref as T
import nfcutil as U
import screen_ref as S

NAMES = L.NAMES
needs_ref = pytest.mark.skipif(T.ref_lib() is None, reason="oracle/_ref/libnfcref.so was not built (needs the reference sources)")

SIG_MAG_F32, SIG_MAG_S16 = 2, 3


def want(name):
    return L.expected("case/" + name, L.case(name)[0])


def chunks_of(n):
    return (n - 80 + L.CHUNK - 1) // L.CHUNK if n > 80 else 0


# --- CPU -----------------------------------------------------------------------------------------------------------------
@needs_ref
def test_golden_equals_live_reference():
    """tests/golden/ref_long_frames.json.xz is what the reference answers today, input for input"""
    inputs = L.golden_inputs()
    assert sorted(L.golden()) == sorted(inputs)
    for name, build in inputs.items():
        g, live = L.golden()[name], json.loads(json.dumps(L.golden_entry(name, build())))
        if "frames" in g:
            # past a 1-byte RATS the reference's answer depends on the process's history (long_frames.comparable)
            g, live = dict(g, frames=L.comparable(g["frames"])), dict(live, frames=L.comparable(live["frames"]))
        assert g == live, name


@pytest.mark.parametrize("name", NAMES)
def test_capture_decodes_to_what_it_was_built_with(name):
    """the generator: every poll / listen frame decodes to its payload, unless a frame passes the negotiated limit"""
    x, built = L.case(name)
    got = [(r[1], bytes.fromhex(r[7])) for r in want(name) if r[1] in (L.POLL, L.LISTEN)]
    if built is not None:
        assert got == built
    else:
        # the reference cuts the frame that reaches the limit there and flags it Truncated (0x08)
        assert any(r[2] & 0x08 for r in want(name)) or name == "a0/fsdi13"


def test_golden_pins_the_limits():
    """what the recorded runs show: lengths at the limits, Truncated | CrcError past them, nothing after FSDI 13"""
    frames = lambda name: [(r[1], r[2], len(r[7]) // 2) for r in want(name) if r[1] in (L.POLL, L.LISTEN)]
    for rate in (0, 1, 2):
        assert frames("a%d/n256" % rate)[-2:] == [(L.POLL, 0, 256), (L.LISTEN, 0, 256)]
        assert frames("a%d/n257" % rate)[0] == (L.POLL, 0x28, 256)
        assert frames("a%d/fsdi9/n512" % rate)[-2:] == [(L.POLL, 0, 512), (L.LISTEN, 0, 512)]
        assert frames("a%d/fsdi9/n513" % rate)[2] == (L.POLL, 0x28, 512)
    for fsdi in L.RATS_FSDI:
        limit = L.FDS[fsdi]
        for where in ("same", "later"):
            assert frames("a0/fsdi%d/%s/n%d" % (fsdi, where, limit + 1))[2] == (L.POLL, 0x28, limit)
    assert frames("a0/fsdi0/same/n300")[2] == (L.POLL, 0x28, 16) and len(frames("a0/fsdi0/same/n300")) > 20
    assert frames("a0/fsdi13") == [(L.POLL, 0, 4)]
    assert frames("b/atqb0/n17")[2:] == [(L.POLL, 0x28, 16), (L.LISTEN, 0x28, 16)]
    assert frames("f2/n254") == [(L.POLL, 0x28, 254)]


@pytest.mark.parametrize("name", NAMES)
def test_host_model_equals_reference(name):
    """the host build of the lane machine: one lane, the segment pipeline and the warp-lane pipeline (fast paths on), the
    last two fed the screen model's flags"""
    x = L.case(name)[0]
    ref = L.comparable(T.keys(want(name))[:-1])
    trig = S.block_flags_device_model(x, S.ScreenParams(L.FS))
    c = L.comparable
    assert c(U.sim_run(x, L.FS)[0]) == ref
    assert c(U.sim_pipeline(x, trig, L.FS)[0]) == ref
    assert c(U.sim_pipeline2(x, trig, L.FS)[0]) == ref
    assert c(U.sim_pipeline2(x, trig, L.FS, group=1, exact_int=True)[0]) == ref


def test_record_parser_round_trip():
    """the packed layout: 80 payload bytes inline, the rest in 128-byte chunks, at the inline and chunk edges"""
    rng = np.random.default_rng(5)
    lengths = [0, 1, 79, 80, 81, 208, 209, 336, 337, 464, 465, 511, 512]
    frames = [(k % 3, 0x101, 0x102 + k % 2, k, 0x104, 105937, 1000 * k, 1000 * k + 900, rng.integers(0, 256, n, dtype=np.uint8).tobytes())
              for k, n in enumerate(lengths)]
    rec, ext = L.pack_records(frames)
    assert rec.nbytes == 128 * len(frames) and ext.size == 128 * sum(chunks_of(n) for n in lengths)
    got = L.parse_records(rec, ext, stream_offset=5)
    assert got == [(f[0] + 5,) + f[1:] for f in frames]
    assert [len(f[-1]) for f in got] == lengths


# --- GPU -----------------------------------------------------------------------------------------------------------------
def _decoder(**kw):
    import nfc_laboratory_b200 as N
    return N.NfcDecoder(device=0, **kw)


@pytest.fixture(scope="module")
def dec():
    d = _decoder()
    yield d
    d.close()


@pytest.fixture(scope="module")
def dec_exact():
    d = _decoder(exact=True)
    yield d
    d.close()


@pytest.fixture(scope="module")
def dec_straggler():
    """every thread lane goes to the warp-lane straggler pass (NFCB200_STRAGGLER=-1, read at nfcb200_create)"""
    old = os.environ.get("NFCB200_STRAGGLER")
    os.environ["NFCB200_STRAGGLER"] = "-1"
    try:
        d = _decoder()
    finally:
        if old is None:
            del os.environ["NFCB200_STRAGGLER"]
        else:
            os.environ["NFCB200_STRAGGLER"] = old
    yield d
    d.close()


def batch_streams(d, x, sigtype):
    """records of decode_batch of x [streams, n] with each frame's stream: [(stream,) + record]"""
    a = np.ascontiguousarray(x)
    buf, n = d.decode_batch_ptr(a.ctypes.data, False, sigtype, a.shape[0], a.shape[1], L.FS, raw=True)
    return [(int(buf[i].stream),) + r for i, r in enumerate(T.records(buf, n))]


def fresh_stream(d):
    st = T.Stream(d)
    st.reset()
    return st


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_batch_equals_reference(dec, dec_exact, dec_straggler, name):
    x = L.case(name)[0]
    ref = L.comparable(want(name)[:-1])
    first = T.batch_records(dec, x, SIG_MAG_F32, L.FS)
    assert L.comparable(first) == ref
    for d in (dec, dec_exact, dec_straggler):
        assert T.batch_records(d, x, SIG_MAG_F32, L.FS) == first
        assert T.batch_records(d, L.s16(x), SIG_MAG_S16, L.FS) == first


def tiny_plan(name, n, frames):
    """65 536-sample buffers, and 1-63-sample buffers over 6 000 samples at the start and at the end of the longest frame"""
    longest = max((f for f in frames if f[1] in (L.POLL, L.LISTEN)), key=lambda f: len(f[7]))
    rng = T._rng("long", name)
    out, at = [], 0
    for a, b in ((longest[5] - 3000, longest[5] + 3000), (longest[6] - 3000, longest[6] + 3000)):
        a, b = max(a, at), min(b, n)
        out += T._fixed(a - at, 65536) + T._random_chunks(rng, b - a, 1, 63)
        at = b
    return [c for c in out if c] + T._fixed(n - at, 65536)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_stream_equals_reference(dec, name):
    """whole, 65 536-sample and 1-63-sample pushes around the longest frame, each plus the flush frame"""
    x = L.case(name)[0]
    ref = want(name)
    plans = [[len(x)], T._fixed(len(x), 65536), tiny_plan(name, len(x), ref)]
    got = [fresh_stream(dec).plan(x, chunks, SIG_MAG_F32, L.FS) for chunks in plans]
    assert all(sum(p) == len(x) for p in plans)
    assert got[1] == got[0] and got[2] == got[0]
    if L.comparable(ref) == ref:
        assert got[0] == ref
    else:
        assert L.comparable(got[0]) == L.comparable(ref) and got[0][:-1] == T.batch_records(dec, x, SIG_MAG_F32, L.FS)


def device_records(d):
    """(records, chunks) of the last decode_batch, copied from device memory"""
    import torch
    from nfc_laboratory_b200.dist import _DevView
    rp, n, ep, ne = d.device_frames()
    host = lambda p, k: torch.as_tensor(_DevView(p, k * 128), device="cuda").cpu().numpy() if k else np.zeros(0, np.uint8)
    return host(rp, n), host(ep, ne)


@pytest.mark.gpu
def test_dense_batch_equals_reference(dec):
    """every stream of the dense batch equals the reference, up to a 1-byte RATS in the noise where there is one
    (long_frames.comparable; test_dense_batch_records_convert checks the lane modes against each other past it)"""
    x = L.dense_batch()
    got = batch_streams(dec, x, SIG_MAG_F32)
    cut = 0
    for s in range(L.DENSE_STREAMS):
        ref = L.comparable(L.expected("dense/%d" % s, x[s])[:-1])
        mine = [r[1:] for r in got if r[0] == s]
        assert L.comparable(mine) == ref, s
        cut += len(mine) > len(ref)
    assert cut < L.DENSE_STREAMS // 2


@pytest.mark.gpu
def test_dense_batch_records_convert(dec, dec_exact):
    """the dense batch in both lane modes and from int16 gives the same frames; its packed device records hold one record
    per frame and one chunk per 128 payload bytes past 80; emit_records and the Python parser give decode_batch's frames
    back, byte for byte"""
    x = L.dense_batch()
    got = batch_streams(dec, x, SIG_MAG_F32)
    assert len([r for r in got if len(r[8]) > 160]) > 50
    assert batch_streams(dec_exact, x, SIG_MAG_F32) == got
    assert batch_streams(dec, L.s16(x), SIG_MAG_S16) == got

    rec, ext = device_records(dec)
    assert rec.size == 128 * len(got)
    assert ext.size == 128 * sum(chunks_of(len(r[8]) // 2) for r in got)
    buf, n = dec.emit_records(rec.ctypes.data, len(got), ext.ctypes.data, ext.size // 128, 5, L.FS, raw=True)
    assert [(int(buf[i].stream),) + r for i, r in enumerate(T.records(buf, n))] == [(r[0] + 5,) + r[1:] for r in got]
    parsed = L.parse_records(rec, ext, stream_offset=5)
    assert [(p[0],) + p[1:8] + (p[8].hex(),) for p in parsed] == [(r[0] + 5,) + r[1:9] for r in got]


@pytest.mark.gpu
def test_two_rank_gather_equals_whole_batch(dec):
    """two halves of the dense batch on two handles, their packed records gathered as rank 0 holds them
    (dist.GatheredRecords) and converted: the whole batch's frames"""
    import torch
    from nfc_laboratory_b200.dist import GatheredRecords
    x = L.dense_batch()
    half = L.DENSE_STREAMS // 2
    whole = dec.decode_batch(x, SIG_MAG_F32, L.FS)
    parts = []
    for lo, hi in ((0, half), (half, L.DENSE_STREAMS)):
        d = _decoder()
        try:
            d.decode_batch(x[lo:hi], SIG_MAG_F32, L.FS)
            parts.append(device_records(d))
        finally:
            d.close()
    spans, pr, pe = [], 0, 0
    for rec, ext in parts:
        spans.append((pr, rec.size // 128, pe, ext.size // 128))
        pr, pe = pr + rec.size, pe + ext.size
    records = torch.from_numpy(np.concatenate([p[0] for p in parts]))
    ext = torch.from_numpy(np.concatenate([p[1] for p in parts]))
    got = GatheredRecords(records, ext, spans, lambda r: (r - 1) * half, L.FS).frames(dec)
    assert [f.key() for f in got] == [f.key() for f in whole]
    assert [f.stream for f in got] == [f.stream for f in whole]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["records", "chunks"])
def test_push_past_the_initial_frame_pool_loses_nothing(dec, kind):
    """one push of more than 2^14 frames ("records") or of more than 2^12 extension chunks ("chunks") gives exactly the
    frames of 65 536-sample pushes of the same capture, and those are the reference's"""
    pcm = L.overflow_capture(kind)
    count, dig = L.expected("overflow/" + kind, pcm.astype(np.float32) / np.float32(L.PCM))
    one = fresh_stream(dec).plan(pcm, [len(pcm)], SIG_MAG_S16, L.FS)
    if kind == "records":
        assert len(one) > 1 << 14
    else:
        assert sum(chunks_of(len(r[7]) // 2) for r in one) > 1 << 12
    many = fresh_stream(dec).plan(pcm, T._fixed(len(pcm), 65536), SIG_MAG_S16, L.FS)
    assert len(one) == len(many) == count
    assert one == many
    assert L.digest(one) == dig


@pytest.mark.gpu
def test_frame_past_512_bytes_is_capped(dec, dec_exact):
    """RATS with FSDI 10 (limit 1024) and a 600-byte I-block pair: the reference writes past its 512-byte buffer there,
    so only the device's own answer is pinned -- the frame cut at 512 bytes with its first 512 bytes, the same in both lane
    modes and in the stream (DESIGN.md section 2)"""
    x, _ = L.nfca_case(600, 0, 10)
    poll = L.iblock(600, 0x02, 0, 10)
    got = T.batch_records(dec, x, SIG_MAG_F32, L.FS)
    assert T.batch_records(dec_exact, x, SIG_MAG_F32, L.FS) == got
    assert fresh_stream(dec).plan(x, T._fixed(len(x), 65536), SIG_MAG_F32, L.FS)[:-1] == got
    ex = [(r[1], r[2], bytes.fromhex(r[7])) for r in got if r[1] in (L.POLL, L.LISTEN)]
    assert ex[:2] == [(L.POLL, 0, L.rats(10)), (L.LISTEN, 0, L.ATS)]
    listen = L.iblock(600, 0x03, 0, 10)
    # longer than the 512-byte frame buffer: cut to its first 512 bytes, CRC error (the CRC is not checked past the buffer)
    assert ex[2:] == [(L.POLL, 0x20, poll[:512]), (L.LISTEN, 0x20, listen[:512])]
    assert all(len(p) <= 512 for _, _, p in ex)
