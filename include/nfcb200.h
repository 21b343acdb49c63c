/*
 * nfcb200.h -- C ABI of the H100-native NFC IQ demodulation path (libnfcb200.so).
 *
 * This is the drop-in boundary: the reference has no FFI on this path, its seam is link-time -- whoever provides
 * liblab-radio provides lab::NfcDecoder (lab-radio/src/main/include/lab/nfc/NfcDecoder.h:33-122).  The shim in
 * nfc_laboratory_b200/shim/ implements that class on top of the entry points below (INTEGRATION.md); every entry point
 * names the reference interface it replaces.  Plain pointers and sizes only, no torch / CUDA types.
 *
 * All functions return 0 on success or a negative nfcb200_status; nfcb200_last_error() gives the text.  A handle is
 * single-caller like the reference decoder (RadioDecoderTask.cpp:92-151); CUDA streams and events are internal.
 * There is no CPU fallback: without a CUDA device nfcb200_create() fails with NFCB200_ERR_NO_DEVICE.
 */
#ifndef NFCB200_H
#define NFCB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct nfcb200_handle nfcb200_handle;

typedef enum nfcb200_status
{
   NFCB200_OK = 0,
   NFCB200_ERR_NO_DEVICE = -1,   /* no CUDA device / driver: the product has no CPU path        */
   NFCB200_ERR_INVALID = -2,     /* bad argument (reference: RadioDecoderTask InvalidConfig = -2) */
   NFCB200_ERR_CUDA = -3,        /* CUDA runtime error, see nfcb200_last_error                    */
   NFCB200_ERR_CAPACITY = -4,    /* output or internal pool too small; call again with more room  */
   NFCB200_ERR_UNSUPPORTED = -5  /* sample rate / signal type outside what the kernels implement  */
} nfcb200_status;

/* sample formats.  1 and 2 are hw::SignalType values (hw-dev SignalType.h:27-36); 3 and 4 are the WAV ingest formats
 * of hw::RecordDevice (RecordDevice.cpp:281-311: int16 / 32768.f) decoded on the device */
typedef enum nfcb200_sigtype
{
   NFCB200_SIG_IQ_F32 = 1,   /* SIGNAL_TYPE_RADIO_IQ: interleaved float32 I,Q (RadioDeviceTask.cpp:547-655 fused in) */
   NFCB200_SIG_MAG_F32 = 2,  /* SIGNAL_TYPE_RADIO_SAMPLES: float32 magnitude (NfcDecoder::nextFrames input)          */
   NFCB200_SIG_MAG_S16 = 3,  /* mono int16 PCM                                                                       */
   NFCB200_SIG_IQ_S16 = 4,   /* interleaved int16 I,Q                                                                */
   NFCB200_SIG_LOGIC_F32 = 5,/* SIGNAL_TYPE_LOGIC_SAMPLES, stride 4: float32 IO, CLK, RST, VCC (IsoDecoder input)   */
   NFCB200_SIG_LOGIC_S16 = 6,/* the same 4 channels as int16 (4-channel 16-bit WAV), read as s / 32768.f              */
   NFCB200_SIG_LOGIC_U8 = 7  /* 8-bit unsigned logic samples, the reference's logic WAVs (SignalStorageTask.cpp:485),
                                read as b / 255.f (RecordDevice.cpp:244-245); only the _ch ISO 7816 calls take them     */
} nfcb200_sigtype;

enum { NFCB200_TECH_A = 0, NFCB200_TECH_B = 1, NFCB200_TECH_F = 2, NFCB200_TECH_V = 3 };

/* frame tech and frame types of the ISO 7816 decoder (lab-data RawFrame.h:41-61) */
enum
{
   NFCB200_TECH_ISO_ANY = 0x0200, NFCB200_TECH_ISO7816 = 0x0201,
   NFCB200_FRAME_ISO_VCC_LOW = 0x0200, NFCB200_FRAME_ISO_VCC_HIGH = 0x0201, NFCB200_FRAME_ISO_RST_LOW = 0x0202,
   NFCB200_FRAME_ISO_RST_HIGH = 0x0203, NFCB200_FRAME_ISO_ATR = 0x0210, NFCB200_FRAME_ISO_REQUEST = 0x0211,
   NFCB200_FRAME_ISO_RESPONSE = 0x0212, NFCB200_FRAME_ISO_EXCHANGE = 0x0213
};

/* POD mirror of lab::RawFrame (lab-data RawFrame.cpp:26-39); `stream` is the index of the capture in the batch */
typedef struct nfcb200_frame
{
   uint32_t stream;
   uint32_t tech_type;    /* FrameTech  0x0100 any, 0x0101 A, 0x0102 B, 0x0103 F, 0x0104 V        */
   uint32_t frame_type;   /* FrameType  0x0100 carrier off, 0x0101 carrier on, 0x0102 poll, 0x0103 listen */
   uint32_t frame_flags;  /* FrameFlags: ShortFrame 1, Encrypted 2, Truncated 8, ParityError 0x10, CrcError 0x20, SyncError 0x40 */
   uint32_t frame_phase;  /* FramePhase: 0x0101 carrier, 0x0102 selection, 0x0103 application      */
   uint32_t frame_rate;   /* symbols per second                                                    */
   uint32_t length;       /* payload bytes                                                         */
   uint32_t reserved;
   uint64_t sample_start;
   uint64_t sample_end;
   uint64_t sample_rate;
   double time_start;     /* double(sample_start) / double(sample_rate)                            */
   double time_end;
   double date_time;      /* streamTime + time_start                                               */
   uint8_t data[512];     /* `length` payload bytes, zero padded to the next 64-byte boundary; the rest is not written */
} nfcb200_frame;

/* decoder configuration: the NfcDecoder setters (NfcDecoder.h:47-117) / RadioDecoderTask JSON keys
 * (RadioDecoderTask.cpp:207-366).  nfcb200_config_default() fills the reference defaults. */
typedef struct nfcb200_config
{
   int device;                    /* CUDA device ordinal                                                          */
   uint32_t enabled;              /* bit t enables tech t: setEnableNfcA/B/F/V                                    */
   float power_level_threshold;   /* setPowerLevelThreshold, default 0.01                                         */
   float correlation_threshold[4];/* setCorrelationThresholdNfcX: 0.75 0.50 0.50 0.50                             */
   float modulation_min[4];       /* setModulationThresholdNfcX min: 0.90 0.10 0.10 0.90                          */
   float modulation_max[4];       /* setModulationThresholdNfcX max: 1.00 0.90 0.90 1.00                          */
   uint32_t stream_time;          /* setStreamTime                                                                */
   uint32_t use_tma;              /* 1: stage screening tiles with cp.async.bulk (default); 0: plain loads (debug) */
   uint32_t max_rounds;           /* bound on speculation rounds (0 = default)                                    */
   uint32_t segments_per_lane;    /* 0 = choose from the batch size; >= 1 forces the lane grouping                */
   uint32_t exact;                /* 1: one warp lane per stream carries the reference's float state across the whole
                                     capture (running sums included): bit-exact on float input, slower.  0 (default): lanes
                                     cold-start their running sums -- exact on 16-bit input, sums within 2e-6 on float input */
   uint32_t reserved[3];
} nfcb200_config;

/* counters and device timings of the last nfcb200_decode_batch call */
typedef struct nfcb200_stats
{
   uint64_t samples;          /* n_streams * n_samples                          */
   uint64_t blocks;           /* screening blocks                               */
   uint64_t active_blocks;    /* blocks handed to lanes                         */
   uint64_t segments;         /* segments found by the screen                   */
   uint64_t lanes;            /* lanes (groups of consecutive segments)         */
   uint64_t live_lanes;       /* segments not swallowed by a predecessor        */
   uint64_t lane_runs;        /* lane executions over all rounds                */
   uint64_t lane_samples;     /* samples stepped by lanes over all rounds       */
   uint64_t rounds;           /* speculation rounds                             */
   uint64_t frames;           /* frames returned                                */
   uint64_t kernel_launches;  /* kernels of this library launched by the call   */
   float ms_h2d;              /* host -> device copy of the samples (0 when the input is device resident) */
   float ms_screen;           /* K1 screening kernel                            */
   float ms_segment;          /* segment construction + front pass              */
   float ms_lanes;            /* all lane + chain kernels                       */
   float ms_gather;           /* frame gather incl. device -> host copy         */
   float ms_total;            /* whole call, device events                      */
   float ms_wall;             /* whole call, host clock                         */
   float ms_front;            /* front pass (part of ms_segment .. ms_lanes: own event pair) */
   float straggler_lanes;     /* thread lanes that held the launch and were decoded again by a warp lane (a count)  */
   uint64_t feature_samples;  /* samples the front pass wrote to the feature pool */
} nfcb200_stats;

void nfcb200_config_default(nfcb200_config *cfg);

/* replaces `new NfcDecoder()` + setters (RadioDecoderTask.cpp:67, 224-341; test-sdr main.cpp:149-156) */
int nfcb200_create(const nfcb200_config *cfg, nfcb200_handle **out);

/* replaces the NfcDecoder destructor / cleanup() (NfcDecoder.cpp:365-369) */
void nfcb200_destroy(nfcb200_handle *h);

/* re-configure; takes effect at the next decode (NfcDecoder::initialize, NfcDecoder.cpp:295-360) */
int nfcb200_configure(nfcb200_handle *h, const nfcb200_config *cfg);

/*
 * Batch decode: n_streams independent captures of n_samples each, laid out [n_streams][n_samples] in `sigtype`
 * format.  Replaces one NfcDecoder instance per stream fed by nextFrames() until exhausted (NfcDecoder.cpp:374-467),
 * preceded by the IQ -> magnitude step of RadioDeviceTask (RadioDeviceTask.cpp:547-655) when sigtype is an IQ format.
 *   samples_on_device != 0: `samples` is a device pointer on the handle's device (no copy)
 *   samples_on_device == 0: `samples` is host memory (pinned memory copies asynchronously)
 * Frames are written to out[0 .. min(*n_out, cap)) ordered by (stream, decode order); *n_out is the number of frames
 * decoded (if it exceeds cap the call returns NFCB200_ERR_CAPACITY after filling cap frames).  Carrier on/off frames
 * are included (filter on frame_type like test-sdr main.cpp:171-174 if not wanted).
 */
int nfcb200_decode_batch(nfcb200_handle *h, const void *samples, int samples_on_device, int sigtype, uint32_t n_streams, uint64_t n_samples,
                         uint32_t sample_rate, nfcb200_frame *out, uint64_t cap, uint64_t *n_out);

/*
 * Streaming decode of ONE capture in arbitrary chunks: replaces NfcDecoder::nextFrames(SignalBuffer) called per
 * buffer by RadioDecoderTask::signalDecode (RadioDecoderTask.cpp:377-401) and test-sdr (main.cpp:163-176).  Frames
 * whose decode is complete are returned; state is carried across calls.  n == 0 flushes: the pending tail is decoded
 * as end of stream and, like nextFrames({}) (NfcDecoder.cpp:449-463), one carrier frame at the current clock is added.
 */
int nfcb200_stream_push(nfcb200_handle *h, const void *samples, int sigtype, uint64_t n, uint32_t sample_rate, nfcb200_frame *out, uint64_t cap,
                        uint64_t *n_out);

/*
 * Frames of the stream that did not fit the buffer of an earlier nfcb200_stream_push (which then returned
 * NFCB200_ERR_CAPACITY after delivering `cap` frames): delivers up to cap of them, *n_left = how many remain.  Nothing is
 * lost on overflow; the stream state has advanced regardless.
 */
int nfcb200_stream_pending(nfcb200_handle *h, nfcb200_frame *out, uint64_t cap, uint64_t *n_out, uint64_t *n_left);

/*
 * Per-sample value tap on the device (debug / test): ONE lane of the decoder over a host capture, one row of 8 floats per
 * sample from `first` on -- [x, w, deviation, average, channel 4, channel 5, lock state, 0], the channels of the
 * reference's signal debugger (NfcTech.h:32-37, NfcDecoder::setEnableDebug), NaN where a channel was not written.
 * first = 0: the exact stream start; otherwise a cold start with `warm` warm-up samples.  rows must hold (n - first) * 8
 * floats.  Slow by design (one GPU thread); the product kernels compile the taps away.
 */
int nfcb200_debug_trace(const nfcb200_config *cfg, const void *samples, int sigtype, uint64_t n, uint32_t sample_rate, uint32_t first,
                        uint32_t warm, float *rows);

/* forget the streaming state (NfcDecoder::initialize on a sample-rate change, NfcDecoder.cpp:383-388) */
int nfcb200_stream_reset(nfcb200_handle *h);

int nfcb200_get_stats(nfcb200_handle *h, nfcb200_stats *stats);

/* debug tap: per-block screening flags of the last batch, [n_streams][n_blocks] bytes (bit0 trigger, bit1 active) */
int nfcb200_get_block_flags(nfcb200_handle *h, uint8_t *out, uint64_t cap, uint64_t *n_blocks_per_stream);

/*
 * Time shards of ONE long capture (BASELINE.json configs[4]): a shard that does not start at the capture's first sample
 * continues its predecessor's decoder.  After a single-stream nfcb200_decode_batch, nfcb200_carry_before returns the carry
 * of the decoder in front of the first lane that begins at or after `sample` (*lane_begin: that lane's begin, an idle point
 * of the capture; ~0 when there is none).  nfcb200_set_carry hands such a carry to the NEXT single-stream decode of a handle
 * (one shot; clock_shift is subtracted from the absolute sample times it holds: the next window counts from its own first
 * sample).  The blob is opaque, nfcb200_carry_size() bytes: protocol state (FSD / FWT / SFGT from RATS / ATS / ATTRIB, the
 * Encrypted flag, lastCommand -- NfcA.cpp:1592-1790, NfcB.cpp:1153-1258), carrier flags, the carrier edge time.
 * A window decoded from an injected carry is a CONTINUATION, not a decoder start: the reference's start-of-stream
 * behaviour (two carrier-off frames at samples 0 and 1, detectors held off for 1 024 samples) does not apply, its first
 * 2 048 samples are warm-up only (start the window that far, or further, in front of the idle point the carry belongs
 * to: nfc_laboratory_b200/dist.py decode_long_capture_carry uses 6 144).
 */
int nfcb200_carry_size(void);
int nfcb200_default_carry(nfcb200_handle *h, void *blob, uint64_t cap); /* what a cold-started lane assumes: power-on state, carrier on */
int nfcb200_set_carry(nfcb200_handle *h, const void *blob, uint64_t size, uint32_t clock_shift);
int nfcb200_carry_before(nfcb200_handle *h, uint64_t sample, void *blob, uint64_t cap, uint64_t *size, uint64_t *lane_begin);

/*
 * Multi-GPU frame gather (SURVEY.md 8e; no counterpart in the reference, which has no second device): the frames of the
 * last nfcb200_decode_batch call as they sit in DEVICE memory -- ordered by (stream, time), 128-byte records (stream,
 * header fields, the first 80 payload bytes) plus 128-byte extension chunks for longer payloads -- so that a rank can hand
 * them to NCCL without a host round trip; nfcb200_emit_records converts gathered records (host memory) into ABI frames
 * on the receiving rank, adding stream_offset to the stream index.  The pointers stay valid until the next decode.
 */
int nfcb200_device_frames(nfcb200_handle *h, const void **records, uint64_t *n_records, const void **ext, uint64_t *n_ext_chunks);
int nfcb200_emit_records(nfcb200_handle *h, const void *records, uint64_t n_records, const void *ext, uint64_t n_ext_chunks, uint32_t stream_offset,
                         uint32_t sample_rate, nfcb200_frame *out, uint64_t cap, uint64_t *n_out);

/*
 * Wire format of the multi-GPU frame gather (no reference counterpart: the reference is one decoder per process).
 * Writes [u64 count][count x 80-byte frame headers, stream index raised by stream_offset][payload bytes back to back]
 * to `out`; *n_bytes is the size needed (call with out == NULL to size the buffer).  Host-only, no CUDA call.
 */
int nfcb200_pack_frames(const nfcb200_frame *frames, uint64_t n, uint32_t stream_offset, uint8_t *out, uint64_t cap, uint64_t *n_bytes);

/*
 * FFT spectrum of IQ captures: lab::FourierProcessTask::process (FourierProcessTask.cpp:223-352, the frequency view of the
 * reference's GUI, topic "signal.fft") at every hop of every stream.  n_streams captures of n_samples each, laid out
 * [n_streams][n_samples] in `sigtype` format (NFCB200_SIG_IQ_F32 or NFCB200_SIG_IQ_S16; int16 enters as s / 32768.f).
 * Frame f of stream s is the reference's frame of a buffer that begins at sample f * hop: decimation d = sample_rate / 625000,
 * 1024 window positions taken as runs of 4 consecutive samples every 4 d samples (the reference's SSE2 selection), the
 * sin^2 window, a 1024-point forward FFT, magnitudes sqrt(re^2 + im^2), negative frequencies first.  Frames per stream:
 * n_samples < 1024 d ? 0 : (n_samples - 1024 d) / hop + 1.
 *   samples_on_device / out_on_device: `samples` / `out` are device pointers on the handle's device, else host memory
 *   out: [n_streams][*n_frames][1024] float32; cap counts floats.  If it is too small the call returns NFCB200_ERR_CAPACITY
 *        with *n_frames set and writes nothing.
 * A magnitude sigtype or a sample rate below 625 000 S/s returns NFCB200_ERR_UNSUPPORTED.  The call returns when `out` is
 * complete and changes no decode state of the handle (streaming state, carry, stats, block flags, device frames).
 */
int nfcb200_spectrum(nfcb200_handle *h, const void *samples, int samples_on_device, int sigtype, uint32_t n_streams, uint64_t n_samples,
                     uint32_t sample_rate, uint64_t hop, float *out, int out_on_device, uint64_t cap, uint64_t *n_frames);

/* frames per stream and decimation of nfcb200_spectrum for a shape; host only, no CUDA call */
int nfcb200_spectrum_shape(uint64_t n_samples, uint32_t sample_rate, uint64_t hop, uint64_t *n_frames, uint32_t *decimation);

/*
 * ISO 7816 contact smart-card decode: n_streams 4-channel logic captures (IO, CLK, RST, VCC) of n_samples each, laid out
 * [n_streams][n_samples][4] in `sigtype` format (NFCB200_SIG_LOGIC_F32 or NFCB200_SIG_LOGIC_S16).  Replaces one
 * lab::IsoDecoder per stream fed the whole capture by one nextFrames() call, then nextFrames({}) (IsoDecoder.cpp:164-215).
 * Conventions as nfcb200_decode_batch: samples_on_device, frames ordered by (stream, decode order) with `stream` the batch
 * index, NFCB200_ERR_CAPACITY after filling cap frames with *n_out the number decoded, date_time from config.stream_time.
 * VCC / RST changes come as tech 0x0200 frames; ATR, PPS, T=0 TPDUs and T=1 blocks as tech 0x0201.  Payloads over 512
 * bytes are cut there and flagged Truncated (0x08).  A non-logic sigtype or a sample rate of 0 returns NFCB200_ERR_INVALID,
 * n_samples >= 2^32 - 1 NFCB200_ERR_UNSUPPORTED (the reference's sample clock is 32-bit).  The call changes no NFC decode
 * state of the handle (streaming state, carry, stats, block flags, device frames).
 */
int nfcb200_iso7816_decode_batch(nfcb200_handle *h, const void *samples, int samples_on_device, int sigtype, uint32_t n_streams, uint64_t n_samples,
                                 uint32_t sample_rate, nfcb200_frame *out, uint64_t cap, uint64_t *n_out);

/*
 * Streaming ISO 7816 decode of ONE logic capture in arbitrary buffers: replaces lab::IsoDecoder::nextFrames(SignalBuffer)
 * called per buffer by LogicDecoderTask (LogicDecoderTask.cpp:300), and nextFrames({}) on stop (:186, :261).  Input is
 * host memory, n samples of 4 channels in `sigtype` format (NFCB200_SIG_LOGIC_F32 or NFCB200_SIG_LOGIC_S16).  The decoder
 * state, the last sample included, carries from buffer to buffer, and so does the reference's call boundary: a buffer
 * picks its loop afresh (detect unless an ATR locked the protocol), so where buffers end can change the frames, as it does
 * in the reference (DESIGN.md section 13).  A buffer at another sample rate restarts the sample clock at 0 and resets the
 * protocol.  date_time uses config.stream_time as it is at the push.  n == 0 is nextFrames({}): it decodes nothing and
 * delivers what is pending.  More frames than cap: NFCB200_ERR_CAPACITY after delivering cap, the rest wait in
 * nfcb200_iso7816_stream_pending (nothing is lost).  A stream whose sample clock would pass 2^32 - 1 samples is refused
 * with NFCB200_ERR_UNSUPPORTED.  The ISO stream leaves every other state of the handle alone (NFC stream, batch decode
 * state, spectrum, ISO batch), and they leave it alone.
 */
int nfcb200_iso7816_stream_push(nfcb200_handle *h, const void *samples, int sigtype, uint64_t n, uint32_t sample_rate, nfcb200_frame *out,
                                uint64_t cap, uint64_t *n_out);

/*
 * The two calls above for logic captures of `channels` channels (4-8), laid out [n_streams][n_samples][channels] and
 * [n][channels], in any logic format: NFCB200_SIG_LOGIC_F32, NFCB200_SIG_LOGIC_S16 or NFCB200_SIG_LOGIC_U8.  The reference
 * reads a buffer's stride() channels per sample and decodes channels 0-3 (IO, CLK, RST, VCC: IsoTech.cpp:37-58,
 * Iso7816.cpp:39-42); channels 4 and up are read past and never affect a frame.  channels outside 4-8 returns
 * NFCB200_ERR_INVALID: with fewer than 4 the reference reads channels the sample does not have, with more than 8 it
 * writes past its 8-channel sample (IsoTech.h:230-236).  Device samples of the batch call must be aligned to one channel
 * (4 / 2 / 1 bytes); stream pitch and base need no other alignment.  A stream keeps its state, the last sample's channels
 * 0-3 included, across pushes of different formats and channel counts.  Every other convention is that of
 * nfcb200_iso7816_decode_batch and nfcb200_iso7816_stream_push, which mean channels = 4 and take float32 and int16 only.
 */
int nfcb200_iso7816_decode_batch_ch(nfcb200_handle *h, const void *samples, int samples_on_device, int sigtype, uint32_t channels, uint32_t n_streams,
                                    uint64_t n_samples, uint32_t sample_rate, nfcb200_frame *out, uint64_t cap, uint64_t *n_out);
int nfcb200_iso7816_stream_push_ch(nfcb200_handle *h, const void *samples, int sigtype, uint32_t channels, uint64_t n, uint32_t sample_rate,
                                   nfcb200_frame *out, uint64_t cap, uint64_t *n_out);

/* frames of the ISO stream that did not fit an earlier push's buffer: up to cap of them, *n_left = how many remain */
int nfcb200_iso7816_stream_pending(nfcb200_handle *h, nfcb200_frame *out, uint64_t cap, uint64_t *n_out, uint64_t *n_left);

/* forget the ISO stream: the next push decodes as on a fresh handle (the sample before it is 0) */
int nfcb200_iso7816_stream_reset(nfcb200_handle *h);

/* one point of the reference's adaptive signal (lab::SignalResamplingTask): the sample at stream position `sample` kept
 * with its value.  `stream` is the batch index, `channel` 0 for radio and the logic channel for logic. */
typedef struct nfcb200_signal_point
{
   uint32_t stream;
   uint32_t channel;
   uint64_t sample;
   float value;
   uint32_t reserved;
} nfcb200_signal_point;

/*
 * The adaptive signal of radio captures: lab::SignalResamplingTask::processRadioSignal (lab-tasks
 * SignalResamplingTask.cpp:168-229), the waveform of the reference GUI's signal view (QtControl.cpp:238, 296) and the
 * radio signal TraceStorageTask stores in a .trz (TraceStorageTask.cpp:881-1003).  n_streams captures of n_samples each,
 * laid out [n_streams][n_samples] in `sigtype` format (any radio format; IQ enters as its magnitude sqrtf(I*I + Q*Q),
 * int16 as s / 32768.f), are cut into buffers of buffer_len samples (the last one of a stream shorter), each resampled on
 * its own as the reference resamples each buffer it is handed: replayed files come in buffers of 65 536 samples
 * (SignalStorageTask.cpp:323-437).  A live capture is one call per buffer with n_streams = 1, buffer_len = n_samples and
 * `offset` the position of its first sample: the reference keeps no state across buffers.
 *   points: ordered by (stream, emission order of the reference); sample = offset + buffer start + (unsigned) float(i),
 *           the index i stored as float as the reference stores it.  More points than cap: NFCB200_ERR_CAPACITY after
 *           filling cap, *n_out the total.  `out` is host memory.
 *   where the reference is undefined: a buffer shorter than 25 samples reads past its end in the reference's initial sum,
 *           here those samples are 0; a buffer yields at most buffer_len + 1 points, which is more than the reference's
 *           output buffer holds (:170, it writes past it) for a buffer under 255 samples whose samples all deviate,
 *           here every point is returned.
 * Invalid sigtype, a null handle, an empty batch, buffer_len 0 or a sample rate of 0: NFCB200_ERR_INVALID.  buffer_len
 * over 2^24 (indices would not be exact as float) or a stream reaching position 2^32 (the .trz's 32-bit offsets):
 * NFCB200_ERR_UNSUPPORTED.  The call changes no decode state of the handle.
 */
int nfcb200_adaptive_radio(nfcb200_handle *h, const void *samples, int samples_on_device, int sigtype, uint32_t n_streams, uint64_t n_samples,
                           uint32_t sample_rate, uint64_t buffer_len, uint64_t offset, nfcb200_signal_point *out, uint64_t cap, uint64_t *n_out);

/*
 * The adaptive signal of logic captures: lab::SignalResamplingTask::processLogicSignal (SignalResamplingTask.cpp:231-274),
 * stored by TraceStorageTask as logic-<channel>.apcm (TraceStorageTask.cpp:643-758).  Captures of `channels` channels (4-8)
 * laid out [n_streams][n_samples][channels] in NFCB200_SIG_LOGIC_F32, _S16 (s / 32768.f) or _U8 (b / 255.f), cut into
 * buffers as nfcb200_adaptive_radio cuts them.  Every channel but 1 (CLK) gets its points: the first sample of each buffer,
 * each sample that differs from the one before it, and one sample 255 after each point kept.  Points are ordered by
 * (stream, channel, emission order), `channel` the channel number.  Device samples must be aligned to one element.
 * Every other convention is nfcb200_adaptive_radio's; channels outside 4-8 returns NFCB200_ERR_INVALID.
 */
int nfcb200_adaptive_logic(nfcb200_handle *h, const void *samples, int samples_on_device, int sigtype, uint32_t channels, uint32_t n_streams,
                           uint64_t n_samples, uint32_t sample_rate, uint64_t buffer_len, uint64_t offset, nfcb200_signal_point *out, uint64_t cap,
                           uint64_t *n_out);

const char *nfcb200_last_error(void);

/* library / build identification, e.g. "nfcb200 0.1 sm_90a" */
const char *nfcb200_version(void);

#ifdef __cplusplus
}
#endif

#endif
