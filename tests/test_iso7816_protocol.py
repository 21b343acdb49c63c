"""The ISO 7816 decoder's protocol layer against the reference on every frame field: characters swept across the guard
and waiting edges of ATR, T=0 and T=1 contexts (TB3 CWI 0 / 1 / 5 / 9, TC1 0 / 1 / 254 / 255) at 10, 25 and 50 MS/s and
shifted by 0 ... 31 samples, bit boundaries on the decoder's sampling sample in both conventions, ATR parameters (TC2,
TA3 with blocks at the IFSC cut, TD chains to T=15, right and wrong TCK), PPS variants (no PPS1, PPS2 / PPS3, Fi x Di,
RFU values, no response, a counter-proposal), error signals and T=1 parity errors, and the clock: drift at 4.9 / 5.1 %,
ramps, jitter, stops, the device walk's 32-wide clock batch stopping at every lane, and clock measurements on the sample
of an IO edge or a timer.  Captures from tests/iso_sessions.py; the reference's frames in
tests/golden/ref_iso_protocol.json.xz (make_iso_protocol_golden.py).

CPU: the recorded output equals the live reference; the sweeps are monotone around their edges; the shifts cover 0 ...
31; the edges agree with the decoder's arithmetic; no ATR or PPS announces a byte it does not carry; the host build of
the walk and of the stream push equals the reference on every case and plan.
GPU: nfcb200_iso7816_decode_batch per family on float32, int16 and 8-bit input against each row's padded reference,
a stream alone against the same stream in its batch, and nfcb200_iso7816_stream_push whole, in 65 536-sample buffers and
with buffer ends next to the edges and on the clock measurements of a step."""
import json
import os
import sys

import numpy as np
import pytest

import iso_ref as R
import iso_sessions as P
import iso_stream_ref as T

needs_ref = pytest.mark.skipif(R.ref_lib() is None or T.ref_lib() is None,
                               reason="oracle/_ref/libnfcref_iso*.so were not built (need the reference sources)")


def runs():
    return P.golden()["runs"]


NAMES = [n for n in P.names() if n in runs()]
FAMILIES = {f: ns for f, ns in ((f, [n for n in ns if n in runs()]) for f, ns in P.families().items()) if ns}


def want(name):
    g = runs()[name]
    assert g["key"] == P.key(P.case(name), P.rate_of(name)), "the capture differs from the recorded one"
    return g["frames"]


def want_padded(name):
    g = runs()[name]
    return g.get("padded", g["frames"])


def iso_frames(rows):
    return [r for r in rows if r[1] == 0x201]


# --- CPU -----------------------------------------------------------------------------------------------------------------
@needs_ref
@pytest.mark.parametrize("fam", sorted(FAMILIES))
def test_golden_equals_live_reference(fam):
    """tests/golden/ref_iso_protocol.json.xz is what the reference answers today, case for case, padded and chunked"""
    sys.path.insert(0, os.path.join(P.ROOT, "tests", "golden"))
    import make_iso_protocol_golden as M
    got = M.family_entries((fam, FAMILIES[fam], P.edges()))
    for n in FAMILIES[fam]:
        assert json.loads(json.dumps(got[n])) == runs()[n], n


def test_nothing_dropped_but_what_is_named():
    assert sorted(set(P.names()) - set(runs())) == sorted(P.golden()["dropped"])


@pytest.mark.parametrize("ctx", P.CONTEXTS)
def test_edge_sweeps_are_monotone(ctx):
    """the swept character decodes at guard d* ... d* + 3 and not at d* - 3 ... d* - 1; at wait d* - 3 ... d* and not at
    d* + 1 ... d* + 3; in T=0 and in the ATR the waiting time never governs (decodeFrameT0 clears searchEndTime after
    every byte that is not a TPDU's last)"""
    c = P.contexts()[ctx]
    for rate in c.rates:
        e = P.edges()["%s/r%d" % (ctx, rate // 1_000_000)]
        ok = {d: P.responds(want(P.edge_name(ctx, rate, d)), ctx) for d in P.sweep(P.edges(), ctx, rate)}
        if e["guard"] is not None:
            assert all(ok[e["guard"] + k] for k in range(4)) and not any(ok[e["guard"] - k] for k in (1, 2, 3)), (rate, ok)
        if c.t1:
            assert all(ok[e["wait"] - k] for k in range(4)) and not any(ok[e["wait"] + k] for k in (1, 2, 3)), (rate, ok)
            assert not ok[max(ok)]
        else:
            assert e["wait"] is None and ok[max(ok)]


@pytest.mark.parametrize("ctx", P.SHIFT_CONTEXTS)
def test_shifts_cover_every_position(ctx):
    """0 ... 31 leading samples move the swept character through every position mod 32, and at d* - 1, d*, d* + 1 the
    outcome does not depend on the shift"""
    for kind in ("guard", "wait"):
        g = P.edges()["%s/r%d" % (ctx, P.SHIFT_RATE // 1_000_000)][kind]
        if g is None:
            continue
        for d in (g - 1, g, g + 1):
            names = ["shift/%s/%s/d%d/s%d" % (ctx, kind, d, s) for s in range(32)]
            starts = [iso_frames(want(n))[0][7] for n in names]
            assert sorted(x % 32 for x in starts) == list(range(32))
            hit = {P.responds(want(n), ctx) for n in names}
            assert hit == {d != (g - 1 if kind == "guard" else g + 1)}, (kind, d)


def _d2u(x):
    return int(x) & 0xFFFFFFFF if abs(x) < 2 ** 63 else 0


@pytest.mark.parametrize("ctx", P.CONTEXTS)
def test_edges_follow_the_decoders_arithmetic(ctx):
    """d* within one sample of updateProtocol / decodeCharacter: the guard edge at the previous character's start +
    guardTime, the waiting edge one sample before its start + waitingTime, with the ETU of the clock TS gives"""
    c = P.contexts()[ctx]
    for rate in c.rates:
        e = P.edges()["%s/r%d" % (ctx, rate // 1_000_000)]
        s = c.build(rate, 0)
        if not s.starts:
            s.frame(c.frame)
        fclk = P.ts_clock(s)
        fi, di = (1, 1) if ctx == "atr" or ctx.startswith("t0_tc1") else (1, 3)
        et = rate * P.FI[fi] / (P.DI[di] * fclk)
        cgt = _d2u(round(et * 12))
        tc1_255 = ctx.endswith("tc1_255")
        guard = _d2u((10.5 if c.t1 else 11.5) * et) if tc1_255 else _d2u(cgt - 0.5 * et)
        if e["guard"] is not None:
            assert abs(e["guard"] - guard) <= 1, (rate, e, guard)
        if c.t1:
            cwi = int(ctx[6:]) if ctx.startswith("t1_cwi") else 5
            wait = _d2u(_d2u(round(et * (11 + 2 ** cwi))) + 0.5 * et)
            assert abs(e["wait"] - (wait - 1)) <= 1, (rate, e, wait)
        else:
            assert e["guard"] is not None


def test_atr_and_pps_carry_every_announced_byte():
    """processATR / processPPS read only inside the frame for every case: the bytes past a frame's end are a recorded
    deviation (the reference reads its buffer there, the port 0), so no case may depend on them"""
    for n in NAMES:
        for r in iso_frames(want(n)):
            b = bytes.fromhex(r[13])
            if r[2] == P.ATR:
                i, k = 1, 2
                while True:
                    y = b[i]
                    k += bin(y & 0x70).count("1")
                    assert k <= len(b), (n, r[13])
                    if not y & 0x80:
                        break
                    i, k = k, k + 1
                    assert i < len(b), (n, r[13])
            elif b[:1] == b"\xff" and len(b) > 1 and b[1] & 0x10:
                assert len(b) > 2, (n, r[13])


def test_cases_reach_what_they_were_built_for():
    """the parameters under test show in the reference's frames"""
    fr = lambda n: iso_frames(want(n))
    assert any(r[3] & P.FLAG_CRC for r in fr("atr/t1_t15/tck_wrong")) and not any(r[3] & P.FLAG_CRC for r in fr("atr/t1_t15/tck_right"))
    assert any(r[3] & P.FLAG_PARITY for r in fr("err/t1_parity_2"))
    # a clock step moves the protocol clock: the frame after it has another rate than the ATR
    for k in range(P.BATCH_K):
        rows = fr("clk/batch/k%02d" % k)
        assert rows[0][2] == P.ATR and rows[-1][5] != rows[0][5], k
    rates = {fr(n)[-1][5] for n in NAMES if n.startswith("pps/fidi/")}
    assert len(rates) >= 10


@pytest.mark.parametrize("fam", sorted(FAMILIES))
def test_host_equals_golden(fam):
    """the host build of the walk on every case, and of the stream push on every chunk plan"""
    for n in FAMILIES[fam]:
        x, rate = P.case(n), P.rate_of(n)
        assert R.host(x, rate, stream_time=P.STREAM_TIME) == want(n), n
        for plan, chunks in P.chunk_plans(n, x).items():
            if plan in runs()[n].get("plans", {}):
                assert T.host(x, chunks, [rate] * len(chunks), stream_time=P.STREAM_TIME) == runs()[n]["plans"][plan], (n, plan)


# --- GPU -----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dec():
    import nfc_laboratory_b200 as N
    d = N.NfcDecoder(device=0)
    d.setStreamTime(P.STREAM_TIME)
    yield d
    d.close()


def _batch(d, x, sigtype, rate):
    buf, n = d.iso7816_decode(x, sigtype, rate, raw=True)
    rows = R.rows(buf, n)
    out = [[] for _ in range(x.shape[0] if x.ndim == 3 else 1)]
    for r in rows:
        out[r[0]].append([0] + r[1:])
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("fam", sorted(FAMILIES))
def test_batch_equals_reference(dec, fam):
    """one batch call per family and input type; each row against the reference's decode of the padded stream"""
    import nfc_laboratory_b200 as N
    names = FAMILIES[fam]
    rate = P.rate_of(names[0])
    xs = [P.case(n) for n in names]
    n = max(len(x) for x in xs)
    x = np.stack([P.padded(v, n) for v in xs])
    for sigtype, a in ((N.SIG_LOGIC_F32, x), (N.SIG_LOGIC_S16, R.s16(x)), (N.SIG_LOGIC_U8, (x * 255).astype(np.uint8))):
        got = _batch(dec, a, sigtype, rate)
        for name, rows in zip(names, got):
            assert rows == want_padded(name), (name, sigtype)


@pytest.mark.gpu
def test_stream_alone_equals_stream_in_batch(dec):
    import nfc_laboratory_b200 as N
    for fam in ("clk/batch/r25", "edge/t1_cwi1/r50"):
        names = FAMILIES[fam]
        xs = [P.case(n) for n in names]
        n = max(len(x) for x in xs)
        x = np.stack([P.padded(v, n) for v in xs])
        rate = P.rate_of(names[0])
        together = _batch(dec, x, N.SIG_LOGIC_F32, rate)
        for i in range(len(names)):
            assert _batch(dec, x[i], N.SIG_LOGIC_F32, rate)[0] == together[i], names[i]


@pytest.mark.gpu
@pytest.mark.parametrize("fam", sorted(f for f in FAMILIES if f.startswith(("edge/", "clk/batch"))))
def test_stream_push_equals_reference(dec, fam):
    """whole, 65 536-sample buffers and buffer ends at d* - 1, d*, d* + 1 of the edges or on the step's clock
    measurements: the walk's carry across calls"""
    import nfc_laboratory_b200 as N
    for n in FAMILIES[fam]:
        x, rate = P.case(n), P.rate_of(n)
        for plan, chunks in P.chunk_plans(n, x).items():
            dec.iso7816_reset()
            got = T.push(dec, x, chunks, [rate] * len(chunks), N.SIG_LOGIC_F32)
            assert got == (want(n) if plan == "whole" else runs()[n]["plans"][plan]), (n, plan)
