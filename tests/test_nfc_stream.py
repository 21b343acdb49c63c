"""Streaming NFC decode of one capture pushed buffer by buffer (nfcb200_stream_push, lab::NfcDecoder::nextFrames as
RadioDecoderTask and test-sdr call it) and the decoder settings, against the reference on every frame field: the times,
the sample rate and the flush frame included.

CPU: the recorded reference output equals the live reference; the reference's frames do not depend on its buffer plan;
the host build of the lane machine, the segment pipeline and the warp-lane pipeline at every setting of the matrix.
GPU: every capture in buffer plans of 65 536, 4 096, 256, 255, 257 samples, random sizes, 1-63 samples around an exchange
and cuts next to every frame edge; int16 magnitude, float2 IQ, int16 IQ and the synthetic workloads; the pending, reset
and flush calls and a sample-rate change; the settings matrix on the stream and on the batch call in both lane modes."""
import numpy as np
import pytest

import nfc_stream_ref as T
import nfcutil as U
import screen_ref as S

NAMES = U.fixture_names()
MATRIX = T.matrix_cases()
MATRIX_IDS = ["%s-%s" % (T.settings_id(s), name) for s, name in MATRIX]
needs_ref = pytest.mark.skipif(T.ref_lib() is None, reason="oracle/_ref/libnfcref.so was not built (needs the reference sources)")

SIG_IQ_F32, SIG_MAG_F32, SIG_MAG_S16, SIG_IQ_S16 = 1, 2, 3, 4


def s16(mag):
    """the fixtures quantised back to the int16 PCM they were read from (x / 32768.f is exact)"""
    pcm = np.round(mag * 32768.0).astype(np.int16)
    assert np.array_equal(pcm.astype(np.float32) / np.float32(32768.0), mag)
    return pcm


# --- CPU -----------------------------------------------------------------------------------------------------------------
@needs_ref
def test_golden_equals_live_reference():
    """tests/golden/ref_nfc_stream.json.xz is what the reference answers today, input for input"""
    entries = T.golden_entries()
    assert sorted(T.golden()) == sorted(name for name, _, _ in entries)
    for name, steps, s in entries:
        g = T.golden()[name]
        assert g["key"] == T.steps_key(steps, s), name
        assert [tuple(r) for r in g["frames"]] == T.ref_run(steps, s), name


def test_golden_pins_the_flush_and_settings_effects():
    """what the recorded runs show about the reference: the flush frames, date_time, and settings that change frames"""
    g = {k: [tuple(r) for r in v["frames"]] for k, v in T.golden().items()}
    # nextFrames({}) on a fresh decoder: carrier off at clock -1, divided by a sample rate of 0
    assert g["flush/fresh"] == [(0x100, 0x100, 0, 0x101, 0, 0xFFFFFFFF, 0xFFFFFFFF, "", 0, "inf", "inf", "inf")]
    a = g["%s/default" % T.A106]
    assert g["flush/twice"] == a + [a[-1]]
    assert len(g["flush/again"]) == len(a) + 1 and g["flush/again"][-1] == a[-1]
    t = g["%s/stream_time=1.7e+09" % T.A106]
    assert [r[:10] for r in t] == [r[:10] for r in a]
    assert all(float.fromhex(r[11]) == T.STREAM_TIME + float.fromhex(r[9]) for r in t)
    assert all(float.fromhex(r[9]) == r[5] / r[8] for r in a)
    assert len(g["test_NFC-A_424kbps_001/corr=0.2,0.5,0.5,0.5"]) > len(g["test_NFC-A_424kbps_001/default"])
    assert len(g["%s/power=0.003" % T.A106]) != len(a)
    for m in (0x1, 0x2, 0x4, 0x8):
        got = g["test_POLL_ABF_001/enabled=%d" % m]
        assert {r[0] for r in got} <= {0x100, 0x101 + (m.bit_length() - 1)}
    assert {r[0] for r in g["test_POLL_ABF_001/enabled=0"]} == {0x100}
    assert [r[8] for r in g["rate/up"] if r[5] > 0][-1] == T.OTHER_RATE
    # at a sample-rate change the reference re-initialises without the start-of-stream carrier frames a fresh decoder gives
    for o in ("up", "down"):
        first, second = g["rate/%s/first" % o], g["rate/%s/second" % o]
        assert g["rate/%s" % o][:len(first)] == first
        assert [r[:7] for r in second[:2]] == [(0x100, 0x100, 0, 0x101, 0, 0, 0), (0x100, 0x100, 0, 0x101, 0, 1, 1)]
        assert g["rate/%s" % o][len(first):] != second


@needs_ref
@pytest.mark.parametrize("name", NAMES)
def test_reference_frames_do_not_depend_on_the_buffer_plan(name):
    """why one expected list stands for every buffer plan of the device tests"""
    x = T.capture(name)
    want = T.capture_expected(name)
    for plan, chunks in T.plans(name, len(x), want).items():
        if len(set(chunks[:-1])) == 1:
            steps = [("push", x, T.RATE, chunks[0]), ("flush",)]
        else:
            at = np.cumsum([0] + chunks)
            steps = [("push", x[a:b], T.RATE, b - a) for a, b in zip(at[:-1], at[1:])] + [("flush",)]
        assert T.ref_run(steps) == want, plan


@pytest.mark.parametrize("s,name", MATRIX, ids=MATRIX_IDS)
def test_host_model_settings_equal_reference(s, name):
    """the host build of the lane machine with the same thresholds and power level: one lane, the segment pipeline and the
    warp-lane pipeline, both fed the screen model's flags at the same settings"""
    x = T.capture(name)
    want = T.keys(T.capture_expected(name, s))[:-1]
    sp = S.ScreenParams(T.RATE, corrA=s["corr"][0], corrF=s["corr"][2], corrV=s["corr"][3], modMinB=s["mod_min"][1], power=s["power"])
    trig = S.block_flags_device_model(x, sp)
    with T.host_settings(s):
        assert U.sim_run(x, T.RATE, enabled=s["enabled"])[0] == want
        assert U.sim_pipeline(x, trig, T.RATE, enabled=s["enabled"])[0] == want
        assert U.sim_pipeline2(x, trig, T.RATE, enabled=s["enabled"])[0] == want
        assert U.sim_pipeline2(x, trig, T.RATE, enabled=s["enabled"], group=1, exact_int=True)[0] == want


def test_host_settings_reach_the_model():
    """the settings hook changes the host model's frames where the reference's change, and is off outside the block"""
    name = "test_NFC-A_424kbps_001"
    x = T.capture(name)
    low = T.settings(corr={0: 0.2})
    with T.host_settings(low):
        a = U.sim_run(x, T.RATE)[0]
    b = U.sim_run(x, T.RATE)[0]
    assert len(a) > len(b) and b == T.keys(T.capture_expected(name))[:-1]


# --- GPU -----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dec():
    import nfc_laboratory_b200 as N
    d = N.NfcDecoder(device=0)
    yield d
    d.close()


@pytest.fixture(scope="module")
def dec_exact():
    import nfc_laboratory_b200 as N
    d = N.NfcDecoder(device=0, exact=True)
    yield d
    d.close()


def fresh(dec, s=T.DEFAULT, cap=4096):
    """the handle's stream forgotten, settings `s` applied: a new lab::NfcDecoder with its setters called"""
    T.configure(dec, s)
    st = T.Stream(dec, cap)
    st.reset()
    return st


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_buffer_plans_equal_reference(dec, name):
    x = T.capture(name)
    want = T.capture_expected(name)
    got = {}
    for plan, chunks in T.plans(name, len(x), want).items():
        got[plan] = fresh(dec).plan(x, chunks, SIG_MAG_F32, T.RATE)
    # the device alone: every plan gives the same list
    first = next(iter(got.values()))
    assert all(g == first for g in got.values()), [p for p, g in got.items() if g != first]
    for plan, g in got.items():
        assert g == want, plan


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_int16_stream_equals_reference(dec, name):
    x = T.capture(name)
    want = T.capture_expected(name)
    chunks = T.plans(name, len(x), want)["random"]
    assert fresh(dec).plan(s16(x), chunks, SIG_MAG_S16, T.RATE) == want


@pytest.mark.gpu
@pytest.mark.parametrize("name", T.IQ_CAPTURES)
def test_iq_stream_equals_reference(dec, name):
    iq = T.iq_of(T.capture(name))
    want = T.expected("%s/iq" % name, T.whole_steps(T.ref_iq_magnitude(iq)))
    chunks = T._random_chunks(T._rng(name, "iq"), len(iq), 1_000, 300_000)
    assert fresh(dec).plan(iq, chunks, SIG_IQ_F32, T.RATE) == want


@pytest.mark.gpu
@pytest.mark.parametrize("name", T.IQ16_CAPTURES)
def test_int16_iq_stream_equals_reference(dec, name):
    pcm = T.iq16_of(T.capture(name))
    want = T.expected("%s/iq16" % name, T.whole_steps(T.ref_iq_magnitude(pcm)))
    chunks = T._random_chunks(T._rng(name, "iq16"), len(pcm), 1_000, 300_000)
    assert fresh(dec).plan(pcm, chunks, SIG_IQ_S16, T.RATE) == want


@pytest.mark.gpu
@pytest.mark.parametrize("config", T.SYNTH)
def test_synthetic_stream_equals_reference(dec, config):
    iq = T.synth_iq(config)
    for k in range(T.SYNTH_STREAMS):
        want = T.expected("synth/%s/%d" % (config, k), T.whole_steps(T.ref_iq_magnitude(iq[k])))
        assert sum(1 for r in want if r[1] in (0x102, 0x103)) >= 10
        chunks = T._random_chunks(T._rng(config, k), iq.shape[1], 1_000, 300_000)
        assert fresh(dec).plan(iq[k], chunks, SIG_IQ_F32, T.RATE) == want, k


@pytest.mark.gpu
def test_pending_drains_an_overflowing_push_in_order(dec):
    name = "test_NFC-F_212kbps_003"
    x = T.capture(name)
    want = T.capture_expected(name)
    assert len(want) > 40
    for cap in (0, 1):
        st = fresh(dec)
        rc, got, n_out = st.raw_push(x, SIG_MAG_F32, T.RATE, cap)
        assert rc == -4 and n_out == cap and len(got) == cap
        # cap 0 delivers nothing and reports every frame as left
        rc, none, n0, left = st.pending(0)
        assert rc == 0 and none == [] and n0 == 0 and left == len(want) - 1 - cap
        while left:
            rc, more, n, left2 = st.pending(1 if cap == 1 else 7)
            assert rc == 0 and n == len(more) and left2 == left - n
            got += more
            left = left2
        assert st.pending(4)[1:] == ([], 0, 0)
        got += st.push(None, SIG_MAG_F32, T.RATE)
        assert got == want, cap


@pytest.mark.gpu
def test_reset_then_push_equals_a_fresh_handle(dec):
    import nfc_laboratory_b200 as N
    x = T.capture("test_NFC-B_106kbps_002")
    y = T.capture(T.A106)
    st = fresh(dec)
    st.plan(x[:300_000], [100_000] * 3, SIG_MAG_F32, T.RATE, flush=False)
    st.reset()
    a = st.plan(y, T._fixed(len(y), 65536), SIG_MAG_F32, T.RATE)
    other = N.NfcDecoder(device=0)
    try:
        b = T.Stream(other).plan(y, T._fixed(len(y), 65536), SIG_MAG_F32, T.RATE)
    finally:
        other.close()
    assert a == b == T.capture_expected(T.A106)


@pytest.mark.gpu
@pytest.mark.parametrize("seq", ["flush/fresh", "flush/twice", "flush/again"])
def test_flush_sequences_equal_reference(dec, seq):
    steps = T.flush_sequences()[seq]
    want = T.expected(seq, steps)
    st = fresh(dec)
    got = []
    for step in steps:
        if step[0] == "push":
            got += st.plan(step[1], T._fixed(len(step[1]), step[3]), SIG_MAG_F32, step[2], flush=False)
        else:
            got += st.push(None, SIG_MAG_F32, T.RATE)
    assert got == want


@pytest.mark.gpu
@pytest.mark.parametrize("order", ["up", "down"])
def test_sample_rate_change_equals_reference(dec, order):
    steps = T.rate_change_steps(order)
    want = T.expected("rate/%s" % order, steps)
    st = fresh(dec)
    got = []
    for step in steps[:-1]:
        chunks = T._random_chunks(T._rng("rate", order, step[2]), len(step[1]), 1_000, 300_000)
        got += st.plan(step[1], chunks, SIG_MAG_F32, step[2], flush=False)
    got += st.push(None, SIG_MAG_F32, T.RATE)
    # the device restarts as a fresh decoder at the change, start-of-stream carrier frames included; the reference's
    # initialize() does not emit those (DESIGN.md section 2)
    halves = {k: T.expected("rate/%s/%s" % (order, k), v) for k, v in T.restart_steps(order).items()}
    assert got == halves["first"] + halves["second"]
    assert got[:len(halves["first"])] == want[:len(halves["first"])]


@pytest.mark.gpu
@pytest.mark.parametrize("s,name", MATRIX, ids=MATRIX_IDS)
def test_settings_equal_reference(dec, dec_exact, s, name):
    """settings set before the first buffer: the stream, and the batch call with thread lanes and with exact warp lanes"""
    x = T.capture(name)
    want = T.capture_expected(name, s)
    assert fresh(dec, s).plan(x, T._fixed(len(x), 65536), SIG_MAG_F32, T.RATE) == want
    assert T.batch_records(dec, x, SIG_MAG_F32, T.RATE) == want[:-1]
    T.configure(dec_exact, s)
    assert T.batch_records(dec_exact, x, SIG_MAG_F32, T.RATE) == want[:-1]
    T.configure(dec, T.DEFAULT)


@pytest.mark.gpu
def test_nextframes_returns_every_frame_past_cap():
    """NfcDecoder.nextFrames with more frames in one buffer than its copy holds: nothing is lost or reordered"""
    import nfc_laboratory_b200 as N
    name = "test_NFC-F_212kbps_003"
    x = T.capture(name)
    d = N.NfcDecoder(device=0)
    try:
        got = d.nextFrames(x, T.RATE, cap=3) + d.nextFrames(None, cap=3)
    finally:
        d.close()
    want = T.capture_expected(name)
    assert len(want) > 3 * 10
    assert [f.key() for f in got] == T.keys(want)
