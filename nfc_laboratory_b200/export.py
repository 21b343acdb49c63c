"""Frame lists in the reference's own output formats (the step right after the hot path, SURVEY.md 8f rows N1 / N3).
Host-side plumbing, no device code:

  trz_entry / write_frames_json   the `{"frames": [...]}` document of TraceStorageTask::writeFrameEntry
                                  (lab-tasks/src/main/cpp/tasks/TraceStorageTask.cpp:458-520), which is also the golden
                                  format of the regression tool (nfc-test/test-sdr/src/main/cpp/main.cpp writeFrames)
  write_trz / read_trz            the .trz container: tar + gzip with the member `frame.json` (README.md:378-448,
                                  readable by tools/py_nfclab/readers.py and by TraceStorageTask::readFrameEntry :380-455),
                                  and with radio= / logic= the adaptive signal's `logic-<id>.apcm` and `radio-<id>.apcm`
                                  members of TraceStorageTask::writeLogicEntry / writeRadioEntry (:643-758, :881-1003)
  read_trz_signals                those members read back as TraceStorageTask::readLogicEntry / readRadioEntry do
  rx_json_line / rx_text_line     one line per frame as `nfc-rx` prints them (nfc-app/app-rx/src/main/cpp/main.cpp:350-470)

A frame is anything with the fields of binding.Frame / include/nfcb200.h: tech_type, frame_type, frame_flags, frame_phase,
frame_rate, sample_start, sample_end, data -- plus sample_rate and stream_time passed by the caller (time_start =
double(sample_start) / double(sample_rate), date_time = stream_time + time_start, lab-radio NfcA.cpp:539-547).

ISO 7816 frames (tech 0x0200 / 0x0201, NfcDecoder.iso7816_decode) carry their own date_time: the reference sets it to
stream_time alone for ATR, T=0 and T=1 frames (Iso7816.cpp:529-530, 618-619, 670-671).  Given a frame record that has a
date_time field (binding.CFrame, a FRAME_DTYPE record), the writers below use it for those frames.
"""
import io
import json
import math
import struct
import tarfile

import numpy as np

FT_CARRIER_OFF, FT_CARRIER_ON, FT_POLL, FT_LISTEN = 0x0100, 0x0101, 0x0102, 0x0103
FLAG_ENCRYPTED, FLAG_TRUNCATED, FLAG_PARITY, FLAG_CRC, FLAG_SYNC = 0x02, 0x08, 0x10, 0x20, 0x40

TECH_ISO_ANY, TECH_ISO7816 = 0x0200, 0x0201

FRAME_TYPE_NAMES = {FT_CARRIER_OFF: "CarrierOff", FT_CARRIER_ON: "CarrierOn", FT_POLL: "Poll", FT_LISTEN: "Listen",
                    0x0200: "VccLow", 0x0201: "VccHigh", 0x0202: "RstLow", 0x0203: "RstHigh",
                    0x0210: "ATR", 0x0211: "Request", 0x0212: "Response", 0x0213: "Exchange"}
FRAME_TECH_NAMES = {0x0000: "None", 0x0101: "NfcA", 0x0102: "NfcB", 0x0103: "NfcF", 0x0104: "NfcV",
                    TECH_ISO_ANY: "IsoAny", TECH_ISO7816: "ISO7816"}


def _fields(frame):
    """(tech, type, flags, phase, rate, start, end, payload) of a binding.Frame or CFrame, a tuple key, or a FRAME_DTYPE record"""
    if hasattr(frame, "tech_type"):
        data = bytes(frame.data)
        if hasattr(frame, "length"):  # binding.CFrame: the payload is the first `length` bytes of data[512]
            data = data[: int(frame.length)]
        return (int(frame.tech_type), int(frame.frame_type), int(frame.frame_flags), int(frame.frame_phase), int(frame.frame_rate),
                int(frame.sample_start), int(frame.sample_end), data)
    if hasattr(frame, "dtype") and frame.dtype.names:
        return (int(frame["tech_type"]), int(frame["frame_type"]), int(frame["frame_flags"]), int(frame["frame_phase"]), int(frame["frame_rate"]),
                int(frame["sample_start"]), int(frame["sample_end"]), bytes(frame["data"][: int(frame["length"])]))
    t = tuple(frame)
    if len(t) == 9:  # leading stream index
        t = t[1:]
    return (int(t[0]), int(t[1]), int(t[2]), int(t[3]), int(t[4]), int(t[5]), int(t[6]), bytes(t[7]))


def _date_time(frame, tech, stream_time, time_start):
    """an ISO frame's own date_time when the record has one, else stream_time + time_start"""
    if tech in (TECH_ISO_ANY, TECH_ISO7816):
        if hasattr(frame, "date_time"):
            return float(frame.date_time)
        if hasattr(frame, "dtype") and frame.dtype.names and "date_time" in frame.dtype.names:
            return float(frame["date_time"])
    return float(stream_time) + time_start


def trz_entry(frame, sample_rate, stream_time=0.0, range_start=0.0):
    """one element of frame.json["frames"] (TraceStorageTask.cpp:462-498; key set and value types as nlohmann dumps them)"""
    tech, ftype, flags, phase, rate, start, end, payload = _fields(frame)
    time_start = float(start) / float(sample_rate)
    time_end = float(end) / float(sample_rate)
    offset = int(sample_rate * range_start)
    e = {
        "sampleStart": start - offset,
        "sampleEnd": end - offset,
        "sampleRate": int(sample_rate),
        "timeStart": time_start - range_start,
        "timeEnd": time_end - range_start,
        "techType": tech,
        "frameType": ftype,
        "frameRate": rate,
        "frameFlags": flags,
        "framePhase": phase,
        "dateTime": _date_time(frame, tech, stream_time, time_start),
    }
    if payload:
        e["frameData"] = ":".join("%02X" % b for b in payload)
        e["length"] = len(payload)
    return e


def frames_document(frames, sample_rate, stream_time=0.0, range_start=0.0, range_end=math.inf, with_length=True):
    out = []
    for f in frames:
        e = trz_entry(f, sample_rate, stream_time, range_start)
        if e["timeStart"] + range_start < range_start or e["timeEnd"] + range_start > range_end:
            continue  # TraceStorageTask.cpp:466
        if not with_length:
            e.pop("length", None)  # the regression tool's writer has no length key (test-sdr main.cpp writeFrames)
        out.append(e)
    return {"frames": out}


def write_frames_json(path, frames, sample_rate, stream_time=0.0, carrier=False):
    """the regression tool's golden file: poll / listen frames only unless carrier=True (test-sdr main.cpp:171-174)"""
    keep = [f for f in frames if carrier or _fields(f)[1] in (FT_POLL, FT_LISTEN)]
    with open(path, "w") as f:
        json.dump(frames_document(keep, sample_rate, stream_time, with_length=False), f, sort_keys=True)


def write_trz(path, frames, sample_rate, stream_time=0.0, radio=None, logic=None, range_start=0.0, range_end=math.inf):
    """.trz = tar + gzip with the member frame.json (ustar headers: microtar, which the reference reads TRZ with, knows
    nothing else), then, in the order of TraceStorageTask::writeTraceFile (:322-350), one logic-<channel>.apcm per channel
    of `logic` and one radio-<stream>.apcm per stream of `radio`: SIGNAL_POINT_DTYPE arrays as NfcDecoder.adaptive_logic /
    adaptive_radio return them (logic points of one capture).  Only signal points with sample_rate x range_start <= sample
    <= sample_rate x range_end are stored, and frames inside the range.  The reference's Write command without timeStart /
    timeEnd uses 0.0 for both (TraceStorageTask.cpp:228-229), which keeps only the points at sample 0 and the frames that
    end at 0; range_start=0.0, range_end=0.0 gives that trace, the default range_end keeps the whole capture."""
    content = json.dumps(frames_document(frames, sample_rate, stream_time, range_start, range_end), separators=(",", ":")).encode()
    members = [("frame.json", content)]
    if logic is not None and len(logic):
        if len(np.unique(logic["stream"])) > 1:
            raise ValueError("logic points of more than one capture: the .trz names logic entries by channel alone")
        for ch in np.unique(logic["channel"]):
            members.append(("logic-%d.apcm" % ch, apcm_entry(logic[logic["channel"] == ch], sample_rate, int(ch), True, range_start, range_end)))
    if radio is not None and len(radio):
        for st in np.unique(radio["stream"]):
            members.append(("radio-%d.apcm" % st, apcm_entry(radio[radio["stream"] == st], sample_rate, int(st), False, range_start, range_end)))
    with tarfile.open(path, "w:gz", format=tarfile.USTAR_FORMAT) as tar:
        for name, data in members:
            info = tarfile.TarInfo(name)
            info.size = len(data)
            info.mode = 0o664
            tar.addfile(info, io.BytesIO(data))


APCM_MAGIC, APCM_VERSION = b"APCM", 2
INFO_FLAGS, INFO_START_OFFSET, INFO_TOTAL_SAMPLES, INFO_STREAM_ID, INFO_SAMPLE_RATE = range(5)  # TraceStorageTask.cpp:35-39


def _trunc_u32(x):
    """static_cast<unsigned int>(double) of a sample position; None past any position (an infinite range end)"""
    return None if math.isinf(x) else int(x)


def _short(values):
    """static_cast<short>(float): x86 converts to a 32-bit integer (0x80000000 where it does not fit) and keeps 16 bits"""
    v = np.asarray(values, dtype=np.float32).astype(np.float64)
    ok = np.isfinite(v) & (v > -2147483649.0) & (v < 2147483648.0)
    i = np.where(ok, np.trunc(np.where(ok, v, 0.0)), -2147483648.0).astype(np.int64)
    return ((i & 0xFFFF) ^ 0x8000) - 0x8000


def apcm_entry(points, sample_rate, stream_id, logic, range_start=0.0, range_end=math.inf):
    """the bytes of one .apcm member: SampleHdr {'APCM', version 2, info[6]}, then per point in the range the offset delta
    as u8 and, logic, value > 0.5 as u8 (:714-744); radio, the delta of short(value * 32768) as 16-bit little endian
    (:953-986).  Deltas start from the range's first sample and sample 0."""
    start, end = _trunc_u32(sample_rate * range_start), _trunc_u32(sample_rate * range_end)
    pos = np.asarray(points["sample"], dtype=np.int64)
    keep = pos >= start
    if end is not None:
        keep &= pos <= end
    pos, val = pos[keep], np.asarray(points["value"], dtype=np.float32)[keep]
    info = [0] * 6
    info[INFO_START_OFFSET] = max(int(points["sample"][0]) & 0xFFFFFFFF, start) if logic and len(points) else 0
    info[INFO_TOTAL_SAMPLES] = len(pos)
    info[INFO_STREAM_ID] = stream_id
    info[INFO_SAMPLE_RATE] = int(sample_rate)
    hdr = APCM_MAGIC + struct.pack("<I6I", APCM_VERSION, *info)
    doff = (np.diff(pos, prepend=start) & 0xFF).astype(np.uint8)
    if logic:
        rec = np.stack([doff, (val > 0.5).astype(np.uint8)], axis=1)
    else:
        dq = np.diff(_short(val * np.float32(32768.0)), prepend=0) & 0xFFFF
        rec = np.stack([doff, (dq & 0xFF).astype(np.uint8), (dq >> 8).astype(np.uint8)], axis=1)
    return hdr + rec.tobytes()


def read_trz_signals(path):
    """{member name: (header info[6], points)} of the .apcm members of a .trz, points a structured array (sample, value)
    as TraceStorageTask::readLogicEntry / readRadioEntry rebuild them (:526-641, :760-879): positions from
    info[START_OFFSET] plus the running sum of the offset deltas; logic values the stored byte, radio values the running
    16-bit sum of the deltas times 1 / 32768"""
    out = {}
    with tarfile.open(path, "r:gz") as tar:
        for m in tar.getmembers():
            if not (m.name.startswith("logic") or m.name.startswith("radio")):
                continue
            data = tar.extractfile(m).read()
            if data[:4] != APCM_MAGIC:
                raise ValueError("%s: not an APCM entry" % m.name)
            version, *info = struct.unpack_from("<I6I", data, 4)
            if version != APCM_VERSION:
                raise ValueError("%s: APCM version %d" % (m.name, version))
            width = 2 if m.name.startswith("logic") else 3
            rec = np.frombuffer(data, dtype=np.uint8, offset=32)
            if rec.size != info[INFO_TOTAL_SAMPLES] * width:
                raise ValueError("%s: %d bytes for %d samples" % (m.name, rec.size, info[INFO_TOTAL_SAMPLES]))
            rec = rec.reshape(-1, width)
            pts = np.empty(len(rec), dtype=[("sample", "<u8"), ("value", "<f4")])
            pts["sample"] = info[INFO_START_OFFSET] + np.cumsum(rec[:, 0].astype(np.uint64))
            if width == 2:
                pts["value"] = rec[:, 1].astype(np.float32)
            else:
                q = np.cumsum(rec[:, 1].astype(np.int64) | rec[:, 2].astype(np.int64) << 8)
                pts["value"] = (((q & 0xFFFF) ^ 0x8000) - 0x8000).astype(np.float32) * np.float32(1.0 / 32768)
            out[m.name] = (info, pts)
    return out


def read_trz(path):
    """-> list of (tech, type, flags, phase, rate, sample_start, sample_end, payload) like binding.Frame.key()"""
    with tarfile.open(path, "r:gz") as tar:
        doc = json.load(tar.extractfile(tar.getmember("frame.json")))
    out = []
    for e in doc["frames"]:
        data = bytes(int(x, 16) for x in e["frameData"].split(":")) if e.get("frameData") else b""
        out.append((e["techType"], e["frameType"], e["frameFlags"], e["framePhase"], e["frameRate"], e["sampleStart"], e["sampleEnd"], data))
    return out


def rx_json_line(frame, sample_rate, stream_time=0.0):
    """nfc-rx --json line of one frame (main.cpp printFrameJSON :350-437), as compact JSON text"""
    tech, ftype, flags, phase, rate, start, end, payload = _fields(frame)
    time_start = float(start) / float(sample_rate)
    time_end = float(end) / float(sample_rate)
    date_time = _date_time(frame, tech, stream_time, time_start)
    o = {
        "timestamp": start,
        "tech": FRAME_TECH_NAMES.get(tech, "UNKNOWN"),
        "type": FRAME_TYPE_NAMES.get(ftype, "UNKNOWN"),
        "tech_type": tech,
        "frame_type": ftype,
        "time_start": 0 if time_start == 0.0 else time_start,
        "time_end": 0 if time_end == 0.0 else time_end,
        "sample_start": start,
        "sample_end": end,
        "sample_rate": int(sample_rate),
        "date_time": int(date_time) if date_time == math.floor(date_time) else date_time,
    }
    if rate > 0:
        o["rate"] = rate
    if payload:
        o["data"] = ":".join("%02x" % b for b in payload)
        o["length"] = len(payload)
    fl = []
    if flags & FLAG_CRC:
        fl.append("crc-error")
    if flags & FLAG_PARITY:
        fl.append("parity-error")
    if flags & FLAG_SYNC:
        fl.append("sync-error")
    if flags & FLAG_TRUNCATED:
        fl.append("truncated")
    if flags & FLAG_ENCRYPTED:
        fl.append("encrypted")
    if ftype == FT_POLL:
        fl.append("request")
    elif ftype == FT_LISTEN:
        fl.append("response")
    if fl:
        o["flags"] = fl
    return json.dumps(o, sort_keys=True, separators=(",", ":"))  # nlohmann::json objects dump with sorted keys


def rx_text_line(frame, sample_rate):
    """nfc-rx default line of one frame (main.cpp printFrame :439-465)"""
    tech, ftype, flags, phase, rate, start, end, payload = _fields(frame)
    s = "%010.3f (%s) " % (float(start) / float(sample_rate), FRAME_TYPE_NAMES.get(ftype, "UNKNOWN"))
    if ftype in (FT_POLL, FT_LISTEN):
        import numpy as np
        khz = float(np.round(np.float32(rate) / np.float32(1000.0)))  # roundf(float(rate) / 1000.0f)
        s += "[%s@%.0f]: " % (FRAME_TECH_NAMES.get(tech, "UNKNOWN"), khz)
        s += "".join("%02X " % b for b in payload)
    return s
