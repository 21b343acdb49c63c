"""The protocol layer against the reference on every frame field: when the listen search runs (responses swept across the
guard and waiting edges of every window a command or a negotiated value sets, and across every position of a 32-sample
chunk), windows that outlast an idle stretch (a response, a new poll or the end of the capture after more than one lane's
worth of silence inside a negotiated FWT), the chained Encrypted flag of Mifare sessions, and the parity, CRC and
short-frame flags.

CPU: the recorded reference output equals the live reference; the captures decode to what they were built with; every
sweep straddles its edge; the flags the error cases were built to carry; the host build of the lane machine, the segment
pipeline and the warp-lane pipeline equal the reference; the carry exchange of long session captures.
GPU: decode_batch in exact warp lanes, thread lanes and through the straggler hand-over, float and int16; the stream in
whole, 65 536-sample pushes and with buffer ends next to each window edge; the carry exchange through the C ABI."""
import json
import os

import numpy as np
import pytest

import long_frames as L
import nfc_stream_ref as T
import nfcutil as U
import protocol_sessions as P
import screen_ref as S

NAMES = P.names()
EDGE = [n for n in NAMES if n.startswith("edge/")]
CHUNK = sorted({n.rsplit("/", 1)[0] for n in NAMES if n.startswith("chunk/")})
SINGLE = [n for n in NAMES if not n.startswith("chunk/")]
needs_ref = pytest.mark.skipif(T.ref_lib() is None, reason="oracle/_ref/libnfcref.so was not built (needs the reference sources)")

SIG_MAG_F32, SIG_MAG_S16 = 2, 3
GUARD = int(P.STU * 1024)


def want(name):
    return P.expected("case/" + name, P.case(name)[0])


def pl(recs):
    """(type, flags, payload) of the poll / listen frames of records"""
    return [(r[1], r[2], bytes.fromhex(r[7])) for r in recs if r[1] in (P.POLL, P.LISTEN)]


def ctx_of(name):
    return name.split("/d")[0].split("/", 1)[1]


# --- CPU -----------------------------------------------------------------------------------------------------------------
@needs_ref
def test_golden_equals_live_reference():
    """tests/golden/ref_protocol.json.xz is what the reference answers today, input for input"""
    inputs = P.golden_inputs()
    runs = P.golden()["runs"]
    assert sorted(runs) == sorted(inputs)
    for name, build in inputs.items():
        g, live = runs[name], json.loads(json.dumps(P.golden_entry(name, build())))
        g, live = dict(g, frames=L.comparable(g["frames"])), dict(live, frames=L.comparable(live["frames"]))
        assert g == live, name


@pytest.mark.parametrize("name", [n for n in SINGLE if not n.startswith("err/")])
def test_capture_decodes_to_what_it_was_built_with(name):
    """edge sweeps: the exchanges before the one under test, its poll and, where the reference finds it, its response;
    the late responses and encrypted sessions: every frame they were built with"""
    got = [(t, p) for t, _, p in pl(want(name))]
    if name.startswith("edge/"):
        c = P.contexts()[ctx_of(name)]
        if P.responds(want(name), ctx_of(name)):
            assert got == c.frames()
        else:
            # a response that starts before the guard edge is missed or read from its middle (a garbled listen frame)
            assert got[:len(c.frames()) - 1] == c.frames()[:-1] and all(t == P.LISTEN for t, _ in got[len(c.frames()) - 1:])
    else:
        built = P.case(name)[1]
        if built is not None:
            assert got == built


@pytest.mark.parametrize("ctx", P.CONTEXTS)
def test_edge_sweeps_straddle(ctx):
    """every capture of a context has the same noise before its response, so the poll frame ends at the same sample at
    every delay, and the sweep is monotone: the response decodes at guard d* ... d* + 3 and wait d* - 3 ... d*, not at
    guard d* - 3 ... d* - 1 nor wait d* + 1 ... d* + 3, nor 1.2 x the window.  An NFC-V response decodes even when its
    sub-carrier starts right after the poll (its guard edge lies earlier than any well-formed response can start)"""
    e = P.edges()[ctx]
    names = ["edge/%s/d%d" % (ctx, d) for d in P.sweep_delays(ctx)]
    ok = {d: P.responds(want(n), ctx) for d, n in zip(P.sweep_delays(ctx), names)}
    ends = {[r[6] for r in want(n) if r[1] == P.POLL][-1] for n in names}
    assert len(ends) == 1
    assert all(ok[e["wait"] - k] and not ok[e["wait"] + 1 + k] for k in range(3))
    if e["guard"] is None:
        assert ctx == "v/inventory" and all(ok[d] for d in ok if d <= e["wait"])
    else:
        assert all(ok[e["guard"] + k] and not ok[e["guard"] - 1 - k] for k in range(3))
    assert not ok[max(ok)]


@pytest.mark.parametrize("group", CHUNK)
def test_chunk_shifts_cover_every_position(group):
    """the 32 shifts move the poll end (and with it guardEnd and waitingEnd) through all 32 positions mod 32, and the
    response decodes at the waiting edge d* for every shift and at d* + 1 for none"""
    ctx = ctx_of(group)
    d = int(group.rsplit("/d", 1)[1])
    ends = [[r[6] for r in want("%s/s%d" % (group, s)) if r[1] == P.POLL][-1] - s for s in range(32)]
    assert len(set(ends)) == 1
    hit = [P.responds(want("%s/s%d" % (group, s)), ctx) for s in range(32)]
    assert all(hit) if d == P.edges()[ctx]["wait"] else not any(hit)


def test_negotiated_windows_order_the_waiting_edges():
    """the waiting edge follows the window each FWI / time slot sets: FWI 15 reads as 4 (the default FWT), every FWI
    step doubles it, an ATS without TB keeps the default (within a few samples: contexts differ in their payloads and
    their noise, which moves the end of the poll frame the window counts from and the point where the response is found)"""
    e = {c: P.edges()[c]["wait"] for c in P.CONTEXTS}
    near = lambda a, b: abs(a - b) <= 16
    assert near(e["a0/i/fwi15"], e["a0/i/fwi4"]) and near(e["a0/i/notb"], e["a0/i"]) and near(e["a0/i/fwi4"], e["a0/i"])
    for a, b in ((0, 1), (1, 4), (4, 7), (7, 9)):
        assert near(e["a0/i/fwi%d" % b] - e["a0/i/fwi%d" % a], P.xgt(b) - P.xgt(a))
    assert near(e["b/i/fwi8"] - e["b/i/fwi4"], P.xgt(8) - P.xgt(4))
    for rate in (1, 2):
        # an NFC-F response is found somewhere in its 48-bit preamble, wherever the noise lets it
        assert abs(e["f%d/tsn15" % rate] - e["f%d/tsn0" % rate] - int(P.STU * 15 * 256 * 64)) < 64


def test_late_responses_need_the_carried_window():
    """a response 100 000 and 300 000 samples after an I-block behind ATS FWI 7 (longer than the default FWT of 48 332),
    1 000 000 behind FWI 9 and 400 000 behind ATQB FWI 8 decode; a poll during the wait ends it"""
    for name in ("late/a/fwi7/100000", "late/a/fwi7/300000", "late/a/fwi9/1000000", "late/b/fwi8"):
        assert [(t, p) for t, _, p in pl(want(name))] == P.case(name)[1], name
    assert [(t, p) for t, _, p in pl(want("late/a/fwi7/poll"))] == P.case("late/a/fwi7/poll")[1]


@pytest.mark.parametrize("variant,seed", P.ENC_VARIANTS)
def test_encrypted_sessions_carry_the_flag(variant, seed):
    """the first listen frame after AUTH (the nonce, or without one the answer to the next poll) starts the Encrypted
    state: from it on every frame is Encrypted, and from the one after it parity errors are cleared, across idle gaps of
    1, 2 and 5 lanes and through a 6-byte encrypted frame starting 50 00, until WUPA / REQA; the I-block after that is
    clear.  An AUTH with a bad CRC still starts the state; a CRC-failed HLTA before it does not stop the session"""
    name = "enc/%s/%d" % (variant, seed)
    got = pl(want(name))
    wake = max(i for i, f in enumerate(got) if f[2] in (P.REQA, P.WUPA))
    assert got[-2:] == [(P.POLL, 0, P.case(name)[1][-2][1]), (P.LISTEN, 0, P.case(name)[1][-1][1])]
    auth = next(i for i, f in enumerate(got) if f[0] == P.POLL and f[2][:1] in (b"\x60", b"\x61"))
    first = next(i for i in range(auth + 1, len(got)) if got[i][0] == P.LISTEN)
    assert first == auth + (2 if variant == "auth_no_answer" else 1)
    assert all(f[1] & P.FL_ENCRYPTED for f in got[first:wake])
    assert not any(f[1] & P.FL_PARITY for f in got[first + 1:wake])
    assert len(got[first:wake]) >= 17 and any(f[2][:2] == b"\x50\x00" for f in got[first:wake])
    assert not any(f[1] & P.FL_ENCRYPTED for f in got[:first] + got[wake:])
    if variant == "auth_no_answer":
        assert got[auth + 1][1] & P.FL_PARITY


@pytest.mark.parametrize("name", sorted(n for n, (_, k, _) in P.error_cases().items() if k is not None))
def test_error_cases_carry_their_flag(name):
    """the frame built with a flipped parity or CRC bit carries ParityError / CrcError, the other frames do not"""
    _, k, flag = P.error_cases()[name]
    got = pl(want("err/" + name))
    assert got[k][1] & flag, got
    assert not any(f[1] & flag for i, f in enumerate(got) if i != k and not (name == "crc/a0/hlta" and i > k)), got


def test_partial_bytes_and_short_frames():
    """anticollision frames with a partial last byte: 7 bits keep the byte, fewer drop it; no short frame but a 1-byte
    7-bit poll is flagged ShortFrame"""
    for nbytes in range(2, 7):
        for nbits in range(1, 8):
            got = pl(want("err/sdd/nvb%02x" % ((nbytes << 4) | nbits)))
            poll = got[2]
            assert poll[0] == P.POLL and len(poll[2]) == nbytes + (nbits == 7)
            assert not poll[1] & P.FL_SHORT
    for b in (0x35, 0x40, 0x43, 0x7F, 0x00):
        got = pl(want("err/short/%02x" % b))
        assert got[0] == (P.POLL, P.FL_SHORT, bytes([b]))


def host_model(x):
    trig = S.block_flags_device_model(x, S.ScreenParams(P.FS))
    return [U.sim_run(x, P.FS)[0], U.sim_pipeline(x, trig, P.FS)[0], U.sim_pipeline2(x, trig, P.FS)[0],
            U.sim_pipeline2(x, trig, P.FS, group=1, exact_int=True)[0]]


@pytest.mark.parametrize("name", SINGLE)
def test_host_model_equals_reference(name):
    """the host build of the lane machine: one lane, the segment pipeline and the warp-lane pipeline (fast paths on), the
    last two fed the screen model's flags"""
    x = P.case(name)[0]
    ref = L.comparable(T.keys(want(name))[:-1])
    for k, got in enumerate(host_model(x)):
        assert L.comparable(got) == ref, k


@pytest.mark.parametrize("group", CHUNK)
def test_host_model_at_every_chunk_position(group):
    """the waiting edge d* and d* + 1 of a context, shifted by 0 ... 31 leading samples"""
    for shift in range(32):
        name = "%s/s%d" % (group, shift)
        x = P.case(name)[0]
        ref = L.comparable(T.keys(want(name))[:-1])
        for k, got in enumerate(host_model(x)):
            assert L.comparable(got) == ref, (name, k)


@pytest.mark.parametrize("ranks", [False, True], ids=["serial", "rank-protocol"])
@pytest.mark.parametrize("k", range(P.LONG_CAPTURES))
def test_carry_exchange_with_the_lane_pipeline(k, ranks):
    """dist.decode_long_capture_carry over the host build of the lane pipeline with 2 ... 5 shards: the stitched decode of
    a long session capture equals the reference's uncut decode"""
    from nfc_laboratory_b200 import dist as ND
    x = P.long_capture(k)
    full = L.comparable(T.keys(P.expected("long/%d" % k, x))[:-1])
    d = U.HostWindowDecoder(P.FS)
    for shards in (2, 3, 4, 5):
        st = {}
        got = ND.decode_long_capture_carry(d, lambda b, e: x[None, b:e], x.size, shards, None, P.FS, overlap=1 << 18, left=8192, stats=st,
                                           model_ranks=ranks, step=1 << 18)
        assert L.comparable(got) == full, (shards, st)


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


FAMILIES = P.families()


def want_batch(name):
    """the reference's records of the capture as its family's batch holds it (protocol_sessions.padded)"""
    x = P.padded(name)
    return P.expected("case/" + name if len(x) == len(P.case(name)[0]) else "padded/" + name, x)


def batch_streams(d, x, sigtype):
    a = np.ascontiguousarray(x)
    buf, n = d.decode_batch_ptr(a.ctypes.data, False, sigtype, a.shape[0], a.shape[1], P.FS, raw=True)
    recs = T.records(buf, n)
    out = [[] for _ in range(a.shape[0])]
    for i, r in enumerate(recs):
        out[int(buf[i].stream)].append(r)
    return out


def family_batch(d, family, sigtype):
    x = np.stack([P.padded(n) for n in FAMILIES[family]])
    return batch_streams(d, x if sigtype == SIG_MAG_F32 else L.s16(x), sigtype)


@pytest.mark.gpu
@pytest.mark.parametrize("family", list(FAMILIES))
def test_batch_equals_reference(dec, dec_exact, dec_straggler, family):
    """each stream of the family's batch equals the reference's decode of that padded stream on every field, in exact
    warp lanes, thread lanes and the straggler hand-over, float and int16"""
    names = FAMILIES[family]
    first = family_batch(dec_exact, family, SIG_MAG_F32)
    for n, got in zip(names, first):
        assert L.comparable(got) == L.comparable(want_batch(n)[:-1]), n
    for d in (dec, dec_exact, dec_straggler):
        for sigtype in (SIG_MAG_F32, SIG_MAG_S16):
            assert family_batch(d, family, sigtype) == first


def window_cuts(name, recs):
    """buffer ends at guardEnd - 1, 0, + 1 and waitingEnd - 1, 0, + 1 of the window the poll under test opens: its
    reported end plus the guard time and the window, plus the symbol detection delay of its tech and rate (minus for
    NFC-V)"""
    ctx = ctx_of(name)
    c = P.contexts()[ctx]
    polls = [r for r in recs if r[1] == P.POLL and bytes.fromhex(r[7]) == c.poll]
    if not polls:
        return []
    end = polls[-1][6]
    tech, rate = ctx[0], int(ctx[1]) if ctx[1].isdigit() else 0
    p1 = [94, 47, 24]
    sdd = {"a": sum(p1[:rate]), "b": 0, "f": 0, "v": -int(round(P.STU * 512))}[tech]
    out = []
    for edge in (end + GUARD + sdd, end + c.fwt + sdd):
        out += [edge + k for k in (-1, 0, 1)]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("ctx", P.CONTEXTS)
def test_stream_equals_reference(dec, ctx):
    """the edge sweep of each context pushed whole, in 65 536-sample buffers and with buffer ends next to the guard and
    waiting edges of its window, each plus the flush frame"""
    for name in [n for n in EDGE if ctx_of(n) == ctx]:
        x = P.case(name)[0]
        ref = want(name)
        plans = [[len(x)], T._fixed(len(x), 65536), T._cuts(len(x), window_cuts(name, ref))]
        for chunks in plans:
            st = T.Stream(dec)
            st.reset()
            got = st.plan(x, chunks, SIG_MAG_F32, P.FS)
            assert L.comparable(got) == L.comparable(ref), (name, len(chunks))


@pytest.mark.gpu
@pytest.mark.parametrize("k", range(P.LONG_CAPTURES))
def test_carry_exchange_on_the_device(dec, k):
    """the long session captures time-sharded through the C ABI with the decoder's carry handed from shard to shard, serial
    and as one process per GPU would run it: the uncut decode"""
    import nfc_laboratory_b200 as N
    from nfc_laboratory_b200 import dist as ND
    x = P.long_capture(k)
    full = [f.key() for f in dec.decode_batch(x[None], N.SIG_MAG_F32, P.FS)]
    assert L.comparable(full) == L.comparable(T.keys(P.expected("long/%d" % k, x))[:-1])
    for ranks, shards in ((False, 2), (False, 4), (True, 3), (True, 5)):
        st = {}
        got = ND.decode_long_capture_carry(dec, lambda b, e: x[None, b:e], x.size, shards, N.SIG_MAG_F32, P.FS, overlap=1 << 18, left=8192,
                                           stats=st, model_ranks=ranks, step=1 << 18)
        assert got == full, (shards, ranks, st)
