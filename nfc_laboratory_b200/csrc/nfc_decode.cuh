/*
 * nfc_decode.cuh -- K2..K4: segment construction, the exact decoder lanes and the carry chain, on the device.
 *
 *   segment_*_kernel : one thread per stream; finishes the screening flags at block granularity (level shifts,
 *                      carrier on/off band, dilation) and cuts the stream into segments (nfc_chain.h)
 *   lanes_kernel     : persistent warps; every thread is one lane = one exact per-sample decoder (nfc_core.h) running
 *                      over one segment.  The 32 lanes of a warp step in lock step and address their history rings with
 *                      the same relative slot, so ring traffic is fully coalesced (scratch words interleaved by lane).
 *   chain_kernel     : one thread per stream; chain_walk() -> list of lanes whose speculated carry was wrong
 *   frame_*_kernel   : frames of the final generation of the live lanes, ordered and packed on the device
 *   stream_kernel    : single-lane sequential decode for the streaming entry point (nfcb200_stream_push)
 *
 * No kernel here has a counterpart in the reference: the reference runs this logic on one CPU thread per stream.
 */
#ifndef NFCB200_DECODE_CUH
#define NFCB200_DECODE_CUH

#include "nfc_screen.cuh"
#include "nfc_wlane.h"

namespace nfcb200 {

// decoder parameters travel as a __grid_constant__ kernel argument (constant bank, per launch): handles with different
// configurations can decode concurrently

// one decoded frame in the device pool (128 bytes); payloads longer than 80 bytes continue in the extension pool
struct FrameRec
{
   u32 lane;  // global lane index
   u32 gen;   // generation of the lane run that produced it
   u32 seq;   // order within the run
   u32 tech, type, flags, phase, rate, start, end, len;
   u32 ext;   // first 128-byte extension chunk, 0xFFFFFFFF if none
   u8 data[80];
};

struct FramePool
{
   FrameRec *recs;
   u32 cap;
   u32 *count;  // device counter (may exceed cap: overflow is reported, excess frames are dropped)
   u8 *ext;     // extension chunks of 128 bytes
   u32 extCap;  // in chunks
   u32 *extCount;
};

struct DeviceSink
{
   FramePool pool;
   u32 lane, gen, seq;

   __device__ void frame(const FrameOut &f, const u8 *payload)
   {
      u32 idx = atomicAdd(pool.count, 1u);
      u32 s = seq++;

      if (idx >= pool.cap)
         return;

      FrameRec &r = pool.recs[idx];
      r.lane = lane;
      r.gen = gen;
      r.seq = s;
      r.tech = f.tech;
      r.type = f.type;
      r.flags = f.flags;
      r.phase = f.phase;
      r.rate = f.rate;
      r.start = f.start;
      r.end = f.end;
      r.len = f.len;
      r.ext = 0xFFFFFFFFu;

      u32 inl = f.len < 80 ? f.len : 80;
      for (u32 i = 0; i < inl; i++)
         r.data[i] = payload[i];

      if (f.len > 80)
      {
         u32 rest = f.len - 80;
         u32 chunks = (rest + 127) / 128;
         u32 e = atomicAdd(pool.extCount, chunks);
         if (e + chunks <= pool.extCap)
         {
            r.ext = e;
            u8 *dst = pool.ext + (size_t) e * 128;
            for (u32 i = 0; i < rest; i++)
               dst[i] = payload[80 + i];
         }
         else
         {
            r.len = 80; // extension pool exhausted: reported through the counter, payload truncated
         }
      }
   }
};

__device__ __forceinline__ float load_sample(const void *samples, int sigtype, uint64_t idx)
{
   switch (sigtype)
   {
      case SIG_IQ_F32:
      {
         float2 v = __ldg(((const float2 *) samples) + idx);
         return sqrtf(v.x * v.x + v.y * v.y);
      }
      case SIG_MAG_F32:
         return __ldg(((const float *) samples) + idx);
      case SIG_MAG_S16:
         return (float) __ldg(((const short *) samples) + idx) / 32768.0f;
      default:
      {
         short2 v = __ldg(((const short2 *) samples) + idx);
         float I = (float) v.x / 32768.0f, Q = (float) v.y / 32768.0f;
         return sqrtf(I * I + Q * Q);
      }
   }
}

// the same in two halves: the raw load can be issued a whole step before the value is needed (the IEEE square root
// would otherwise wait for it on the spot)
__device__ __forceinline__ float2 load_raw(const void *samples, int sigtype, uint64_t idx)
{
   switch (sigtype)
   {
      case SIG_IQ_F32:
      {
         // a volatile load keeps its place in the instruction stream: the compiler would otherwise sink a read-only load
         // to its use one step later, which defeats the point of requesting the sample early
         float2 v;
         asm volatile("ld.global.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(((const float2 *) samples) + idx));
         return v;
      }
      case SIG_MAG_F32:
         return make_float2(__ldg(((const float *) samples) + idx), 0.0f);
      case SIG_MAG_S16:
         return make_float2((float) __ldg(((const short *) samples) + idx), 0.0f);
      default:
      {
         short2 v = __ldg(((const short2 *) samples) + idx);
         return make_float2((float) v.x, (float) v.y);
      }
   }
}

__device__ __forceinline__ float mag_from_raw(int sigtype, float2 raw)
{
   switch (sigtype)
   {
      case SIG_IQ_F32:
         return sqrtf(raw.x * raw.x + raw.y * raw.y);
      case SIG_MAG_F32:
         return raw.x;
      case SIG_MAG_S16:
         return raw.x / 32768.0f;
      default:
      {
         float I = raw.x / 32768.0f, Q = raw.y / 32768.0f;
         return sqrtf(I * I + Q * Q);
      }
   }
}

// ---------------------------------------------------------------------------------------------------------------------
// segments
// ---------------------------------------------------------------------------------------------------------------------
struct SegmentConfig
{
   uint8_t *flags;      // [n_streams][n_blocks]
   const float *bsum;   // [n_streams][n_blocks]
   uint32_t n_streams, n_blocks;
   uint64_t n_samples;
   uint32_t *counts;    // [n_streams] segments per stream
   const uint32_t *offsets; // [n_streams] exclusive prefix of counts
   LaneRec *lanes;
   uint32_t *queue;     // dirty lane indices
   float low, high;     // carrier thresholds (NfcDecoder.cpp:328-329)
   float meanW;         // per-block decay of the carrier average: signalMeanW0 ^ 256
   uint32_t group;      // segments per lane
   uint32_t *segTotal;  // total number of segments (statistics / group sizing)
   uint32_t shortHalo;  // lanes may use the short warm-up (nfc_chain.h lane_first_sample)
   const uint32_t *segCounts;  // [n_streams] segments per stream (counts[] holds LANES per stream once grouped)
   const uint32_t *segOffsets; // [n_streams] exclusive prefix of segCounts
   SegRec *segs;               // segment table, ordered by (stream, time)
   unsigned long long *featTotal; // feature samples allocated so far (every segment takes end - first)
   uint32_t *activeTotal;         // active blocks (statistics), may be null
   const Carry *carryIn;          // carry in front of the first lane of stream 0 (a time shard continuing a capture), or null
};

// ---- block-granular part of the screen, parallel over all blocks ---------------------------------------------------------
// level shifts (the reference's gated envelope goes stale, NfcTech.cpp:39-53) and the carrier on/off band
// (NfcDecoder.cpp:472-523).  The carrier average entering a block is the exponentially weighted sum of the previous block
// means; with meanW = signalMeanW0^256 = 0.277 eight terms reproduce the recursion to 3e-5, far inside the band margins.
__global__ void segment_flags_kernel(SegmentConfig c)
{
   const uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
   const uint64_t total = (uint64_t) c.n_streams * c.n_blocks;
   if (i >= total)
      return;

   const uint32_t b = (uint32_t) (i % c.n_blocks);
   const float *bsum = c.bsum + (i - b);
   const float inv = 1.0f / NFCB200_BLOCK;

   const float mean = bsum[b] * inv;
   const float prev = (b ? bsum[b - 1] : bsum[0]) * inv;

   uint8_t f = c.flags[i] & SCR_TRIGGER;

   if (fabsf(mean - prev) > 0.025f * fmaxf(prev, 1e-6f))
      f |= SCR_TRIGGER;

   float avg = 0, wgt = 1.0f - c.meanW;
   for (uint32_t j = 1; j <= 8 && j <= b; j++)
   {
      avg += wgt * (bsum[b - j] * inv);
      wgt *= c.meanW;
   }

   const float avgEnd = c.meanW * avg + (1.0f - c.meanW) * mean;
   const float lo = fminf(fminf(avg, avgEnd), mean);
   const float hi = fmaxf(fmaxf(avg, avgEnd), mean);
   if (lo < 1.2f * c.high && hi > 0.8f * c.low)
      f |= SCR_TRIGGER | SCR_BAND;

   c.flags[i] = f;
}

// dilation: a block is active when a trigger lies within [b - POST, b + PRE], or at the stream start (nfc_chain.h)
__global__ void segment_activate_kernel(SegmentConfig c)
{
   const uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
   const uint64_t total = (uint64_t) c.n_streams * c.n_blocks;
   if (i >= total)
      return;

   const uint32_t b = (uint32_t) (i % c.n_blocks);
   const uint8_t *flags = c.flags + (i - b);

   // the stream start is always a segment -- unless stream 0 continues a capture from an injected carry
   // the stream start is always a segment -- unless stream 0 continues a capture from an injected carry: then its first
   // blocks are warm-up and their triggers (the screen's start-up transient) do not count (blocks_activate, nfc_chain.h)
   const bool cont = c.carryIn && i < c.n_blocks;
   bool act = b < NFCB200_START_BLOCKS && !cont;
   uint32_t lo = b > NFCB200_POST_BLOCKS ? b - NFCB200_POST_BLOCKS : 0;
   if (cont && lo < NFCB200_START_BLOCKS)
      lo = NFCB200_START_BLOCKS;
   const uint32_t hi = b + NFCB200_PRE_BLOCKS < c.n_blocks ? b + NFCB200_PRE_BLOCKS : c.n_blocks - 1;
   for (uint32_t k = lo; k <= hi && !act; k++)
      act = (flags[k] & SCR_TRIGGER) != 0;

   if (act)
      c.flags[i] |= SCR_ACTIVE; // other threads only read the trigger bit of this byte

   if (c.activeTotal)
   {
      const unsigned m = __ballot_sync(__activemask(), act);
      if (act && (threadIdx.x & 31) == (unsigned) (__ffs(m) - 1))
         atomicAdd(c.activeTotal, (uint32_t) __popc(m));
   }
}

// a segment starts at an active block with no active block among the previous GAP - 1 blocks (blocks_segments())
__global__ void segment_starts_kernel(SegmentConfig c)
{
   const uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
   const uint64_t total = (uint64_t) c.n_streams * c.n_blocks;
   if (i >= total)
      return;

   const uint32_t b = (uint32_t) (i % c.n_blocks);
   const uint32_t s = (uint32_t) (i / c.n_blocks);
   const uint8_t *flags = c.flags + (i - b);

   if (!(flags[b] & SCR_ACTIVE))
      return;

   const uint32_t lo = b >= NFCB200_GAP_BLOCKS - 1 ? b - (NFCB200_GAP_BLOCKS - 1) : 0;
   for (uint32_t k = lo; k < b; k++)
      if (flags[k] & SCR_ACTIVE)
         return;

   c.flags[i] |= SCR_START;
   atomicAdd(&c.counts[s], 1u);
   atomicAdd(c.segTotal, 1u);
}

// lanes per stream for the chosen group size
__global__ void segment_group_kernel(SegmentConfig c)
{
   uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
   if (s >= c.n_streams)
      return;
   const uint32_t n = c.counts[s];
   c.counts[s] = n ? (n - 1) / c.group + 1 : 0;
}

// one warp per stream: walk the start / active bits 32 blocks at a time and emit the lane records in time order
__global__ void segment_fill_kernel(SegmentConfig c, const __grid_constant__ Params dP)
{
   const uint32_t s = blockIdx.x;
   const uint32_t lane = threadIdx.x;
   if (s >= c.n_streams)
      return;

   const uint8_t *flags = c.flags + (size_t) s * c.n_blocks;
   const uint32_t off = c.offsets[s];
   const uint32_t nLanes = c.counts[s];
   const uint32_t nsamples = (uint32_t) c.n_samples;

   uint32_t laneIdx = 0;     // next lane record of this stream
   uint32_t inGroup = 0;     // segments already in the open lane
   uint32_t lastActive = 0;  // highest active block seen so far
   bool open = false;
   const uint32_t segOff = c.segOffsets[s];
   uint32_t segIdx = 0;      // next segment record of this stream

   // close segment record i at sample e and give it its feature range
   auto close_seg = [&](uint32_t i, uint32_t e) {
      SegRec &S = c.segs[segOff + i];
      S.end = e;
      S.featOff = atomicAdd(c.featTotal, (unsigned long long) (e - S.first));
   };

   for (uint32_t base = 0; base < c.n_blocks; base += 32)
   {
      const uint32_t b = base + lane;
      const uint8_t f = b < c.n_blocks ? flags[b] : 0;
      uint32_t startMask = __ballot_sync(0xffffffffu, (f & SCR_START) != 0);
      const uint32_t actMask = __ballot_sync(0xffffffffu, (f & SCR_ACTIVE) != 0);

      if (lane == 0)
      {
         while (startMask)
         {
            const uint32_t p = __ffs(startMask) - 1;
            startMask &= startMask - 1;

            const uint32_t lower = actMask & ((1u << p) - 1u);
            if (lower)
               lastActive = base + 31 - __clz(lower);

            if (open)
            {
               uint32_t e = (lastActive + 1) * NFCB200_BLOCK;
               e = e > nsamples ? nsamples : e;
               c.lanes[off + laneIdx - 1].end = e;
               c.lanes[off + laneIdx - 1].end0 = e;
               close_seg(segIdx - 1, e);
            }

            uint32_t segFirst = lane_first_sample(flags, c.n_blocks, base + p, c.shortHalo != 0);
            if (segFirst == 0 && c.carryIn && s == 0)
               segFirst = 1; // a continued capture has no stream start: also its first lane is a cold-started one
            {
               SegRec &S = c.segs[segOff + segIdx];
               S.stream = s;
               S.begin = (base + p) * NFCB200_BLOCK;
               S.first = segFirst;
               S.end = S.begin;
               S.band = S.begin - segFirst > NFCB200_HALO_SHORT ? 1u : 0u;
               S.hasFeat = 0;
               segIdx++;
            }

            if (inGroup == 0 && laneIdx < nLanes)
            {
               LaneRec &l = c.lanes[off + laneIdx];
               l.stream = s;
               l.begin = (base + p) * NFCB200_BLOCK;
               l.end = l.begin;
               l.end0 = l.begin;
               l.first = segFirst;
               l.seg0 = segOff + segIdx - 1;
               l.stop = 0;
               l.lockedMask = 0;
               l.gen = 0;
               l.dirty = 1;
               l.dead = 0;
               l.nframes = 0;
               laneIdx++;
            }

            open = true;
            if (++inGroup >= c.group)
               inGroup = 0;
         }

         if (actMask)
            lastActive = base + 31 - __clz(actMask);
      }
   }

   if (lane == 0)
   {
      if (open && laneIdx > 0)
      {
         uint32_t e = (lastActive + 1) * NFCB200_BLOCK;
         e = e > nsamples ? nsamples : e;
         c.lanes[off + laneIdx - 1].end = e;
         c.lanes[off + laneIdx - 1].end0 = e;
         close_seg(segIdx - 1, e);
      }

      Carry spec, pon;
      carry_speculate(spec, dP);
      carry_init(pon, dP);
      carry_canon(pon);
      if (c.carryIn && s == 0)
      {
         // the stream continues a capture: its first lane starts from the injected carry, the later ones speculate that
         // the session state it carries is still in force
         pon = *c.carryIn;
         spec = *c.carryIn;
      }

      for (uint32_t j = 0; j < nLanes; j++)
      {
         LaneRec &L = c.lanes[off + j];
         L.in = L.first == 0 ? pon : spec;
         c.queue[off + j] = off + j; // first round: every lane runs
      }
   }
}

// ---------------------------------------------------------------------------------------------------------------------
// thread lanes (the throughput path of large batches): one THREAD per lane, 32 lanes of a warp in lock step, history rings
// in global memory interleaved by lane (nfc_core.h Machine<32>).  Cold-started running sums: exact on 16-bit input, within
// 2e-6 on float input (DESIGN.md); the warp lanes below are the exact path.
// ---------------------------------------------------------------------------------------------------------------------
struct LaneConfig
{
   const void *samples;
   uint64_t n_samples;
   int sigtype;
   const uint8_t *flags;
   uint32_t n_blocks;
   LaneRec *lanes;
   uint32_t n_lanes;         // size of the lane table
   const uint32_t *queue;
   uint32_t queue_count;
   uint32_t *cursor;         // work-stealing cursor over the queue
   float *scratch;           // [n_warps][NFCB200_SCRATCH_FLOATS][32]
   uint8_t *sbuf;            // [n_warps * 32][512]
   FramePool pool;
   unsigned long long *work; // samples stepped (statistics)
   // stragglers: once the queue is empty, a lane that has run bail_margin samples past the length it was queued with gives
   // up and is decoded again by a warp lane (wlanes_kernel, 0.1-0.3 us per sample instead of 1.4-5): bail_margin 0 = never
   uint32_t bail_margin;
   uint32_t bail_always;     // test knob: give up past the margin whether the queue is empty or not
   uint32_t *overrun;        // [n_lanes] lanes that gave up
   uint32_t *overrun_count;
};

#define LANE_THREADS NFCB200_LANE_THREADS

#if defined(NFCB200_LANE_PROFILE)
// development build (make DEFS=-DNFCB200_LANE_PROFILE): where the thread lanes' steps and cycles go.  Per state class,
// [c] warp steps and [NFCB200_PROF_CLASSES + c] clock64() cycles of those warp steps; nfcb200.cu prints and clears them
// under NFCB200_TRACE.  The lanes of a warp step through one class at a time (one timed pass per class present), so a
// class's cycles are its own; a warp step therefore costs more than in the plain build, which interleaves the classes.
enum
{
   PROF_GATED,         // search mode before the detector gate (warm-up)
   PROF_SEARCH,        // search mode past the gate
   PROF_A_POLL,        // locked NFC-A, poll frame
   PROF_A_LISTEN0,     // locked NFC-A 106 kbps listen, before the start of frame (A_listen_start_ask)
   PROF_A_LISTEN1,     // locked NFC-A 106 kbps listen, symbols (A_listen_symbol_ask)
   PROF_LOCKED,        // every other locked state
   PROF_BOOK,          // lane_iterate examines retirement / skip-ahead at this step (and then steps)
   NFCB200_PROF_CLASSES
};
static __device__ unsigned long long nfcb200_lane_prof[2 * NFCB200_PROF_CLASSES];

// the class of the step a running lane takes next
__device__ __forceinline__ uint32_t lane_prof_class(const Front &F, const Lane &L, uint32_t pos, uint32_t n, bool inactive)
{
   if (pos >= n || ((pos & 31) == 0 && inactive))
      return PROF_BOOK;
   if (F.lock == LOCK_NONE)
      return F.k < F.gate ? PROF_GATED : PROF_SEARCH; // step_body gates on k - 1 after front_advance() incremented k
   if (F.lock != LOCK_A)
      return PROF_LOCKED;
   const FrameSt &fs = L.c.t[TECH_A].fs;
   if (fs.frameType == FT_Poll)
      return PROF_A_POLL;
   if (fs.frameType == FT_Listen && F.lockRate == 0)
      return fs.frameStart ? PROF_A_LISTEN1 : PROF_A_LISTEN0;
   return PROF_LOCKED;
}
#endif

// the ring taps of a step are staged in shared memory one step ahead (Machine TAPS = 2), four resident blocks per SM.
// BAIL: the straggler hand-over is compiled in (a separate instantiation: the extra state costs the plain kernel registers
// -- 219 -> 250 ms when it was not)
template <bool BAIL>
__global__ void __launch_bounds__(LANE_THREADS, 4) lanes_kernel(LaneConfig c, const __grid_constant__ Params dP)
{
   const uint32_t lane = threadIdx.x & 31;
   const uint32_t wg = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;

   float *rg = c.scratch + (size_t) wg * NFCB200_SCRATCH_FLOATS * 32 + lane;
   u8 *sb = c.sbuf + ((size_t) wg * 32 + lane) * 512;

   // the per-sample state of every lane (nfc_core.h Front) in shared memory, odd word stride: no bank conflicts
   constexpr u32 FRONT_STRIDE = (sizeof(Front) / 4) | 1u;
   __shared__ u32 hot[LANE_THREADS * FRONT_STRIDE];
   Front &F = *reinterpret_cast<Front *>(&hot[threadIdx.x * FRONT_STRIDE]);

   // the tap stages of every lane, [buffer][tap][thread]: each thread reads only the words its own requests wrote
   __shared__ float stage[2 * TAP_COUNT * LANE_THREADS];
   const bool stageable = taps_stageable(dP);

#if defined(NFCB200_LANE_PROFILE)
   // the warp's counters, written by its lane 0 and added to nfcb200_lane_prof when the warp is done
   __shared__ unsigned long long profAll[LANE_THREADS / 32][2 * NFCB200_PROF_CLASSES];
   unsigned long long *prof = profAll[threadIdx.x >> 5];
   if (lane == 0)
      for (uint32_t i = 0; i < 2 * NFCB200_PROF_CLASSES; i++)
         prof[i] = 0;
#endif

   for (;;)
   {
      uint32_t base = 0;
      if (lane == 0)
         base = atomicAdd(c.cursor, 32u);
      base = __shfl_sync(0xffffffffu, base, 0);

      if (base >= c.queue_count)
         break;

      const uint32_t qi = base + lane;
      const bool have = qi < c.queue_count;

      // correlation rings must read as zero until written (a fresh reference decoder); the sample rings are only read
      // after 1024 steps (detector gate) and the integration ring only after clear_for_listen(), so they need no wipe
      for (uint32_t i = NFCB200_OFF_CA; i < NFCB200_SCRATCH_FLOATS; i++)
         rg[(size_t) i * 32] = 0.0f;

      const uint32_t li = have ? c.queue[qi] : 0;
      LaneRec &R = c.lanes[li];

      Lane L;
      if (!have)
      {
         u32 *raw = (u32 *) &L.fe;
         for (u32 i = 0; i < sizeof(Front) / 4; i++)
            raw[i] = 0;
         for (u32 i = 0; i < sizeof(Carry) / 4; i++)
            ((u32 *) &L.c)[i] = 0;
      }
      DeviceSink sink;
      sink.pool = c.pool;
      sink.lane = li;
      sink.gen = have ? R.gen + 1 : 0;
      sink.seq = 0;

      if (have)
         lane_begin(L, dP, R.in, R.first, R.begin - R.first);

      Machine<32, DeviceSink, 2, false> M(dP, L, F, rg, sb, sink);
      M.attach_stage(&stage[threadIdx.x], stageable);
      M.reload_front();

      const uint64_t streamBase = have ? (uint64_t) R.stream * c.n_samples : 0;
      const uint8_t *flags = c.flags + (have ? (size_t) R.stream * c.n_blocks : 0);
      uint32_t end = have ? R.end : 0;
      const uint32_t n = (uint32_t) c.n_samples;
      LaneSucc succ;
      succ.init(have ? c.lanes : nullptr, li, c.n_lanes);

      uint32_t pos = have ? R.first : 0;
      uint32_t stepped = 0;
      bool running = have;
      bool bailed = false;
      const uint32_t patience = BAIL ? end - pos + c.bail_margin : 0xFFFFFFFFu;

      // the raw sample of the next step is requested one step ahead: every lane walks its own stream, so a warp touches 32
      // different lines and some lane misses the cache on almost every step
      float2 pend = make_float2(0.0f, 0.0f);
      uint32_t pendPos = 0xFFFFFFFFu;
      auto load = [&](uint32_t p) {
         const float2 raw = p == pendPos ? pend : load_raw(c.samples, c.sigtype, streamBase + p);
         if (p + 1 < n)
         {
            pend = load_raw(c.samples, c.sigtype, streamBase + p + 1);
            pendPos = p + 1;
         }
         return mag_from_raw(c.sigtype, raw);
      };
      auto active = [&](uint32_t p) { return (flags[p >> 8] & SCR_ACTIVE) != 0; };
      auto zero = [&]() {
         for (uint32_t i = NFCB200_OFF_CA; i < NFCB200_SCRATCH_FLOATS; i++)
            rg[(size_t) i * 32] = 0.0f;
      };

      // warp-synchronous stepping: kw is the same in all lanes, so is every ring slot label (k + kbase == kw + 1)
      for (uint32_t kw = 0; __any_sync(0xffffffffu, running); kw++)
      {
#if defined(NFCB200_LANE_PROFILE)
         const uint32_t cls = running ? lane_prof_class(F, L, pos, n, pos < n && !active(pos)) : NFCB200_PROF_CLASSES;
         for (uint32_t pc = 0; pc < NFCB200_PROF_CLASSES; pc++)
         {
            const uint32_t in = __ballot_sync(0xffffffffu, cls == pc);
            if (!in)
               continue;
            const long long t0 = clock64();
            if (cls == pc)
#else
         if (running)
#endif
         {
            running = lane_iterate(M, L, dP, pos, end, n, kw, stepped, load, active, zero, succ);

            // a straggler holds the whole launch: everything else is done (the queue is empty) and this lane is far past
            // the length it was queued with
            if constexpr (BAIL)
            {
               if (running && (kw & 1023u) == 1023u && stepped > patience && (c.bail_always || *((volatile uint32_t *) c.cursor) >= c.queue_count))
               {
                  running = false;
                  bailed = true;
               }
            }
         }
#if defined(NFCB200_LANE_PROFILE)
            __syncwarp();
            const long long t1 = clock64();
            if (lane == 0)
            {
               prof[pc]++;
               prof[NFCB200_PROF_CLASSES + pc] += (unsigned long long) (t1 - t0);
            }
         }
#endif
      }

      if (BAIL && bailed)
      {
         // the frames of this run are superseded by the generation of the warp lane's run; the record keeps the carry it
         // started from and stays dirty
         R.gen = sink.gen;
         R.dirty = 1;
         R.nframes = 0;
         c.overrun[atomicAdd(c.overrun_count, 1u)] = li;
         atomicAdd(c.work, (unsigned long long) stepped);
      }
      else if (have)
      {
         // `end` grew over the successors the run took over; the committed region (R.end) is only moved by the chain walk,
         // which derives the same swallow decisions from R.stop (a run never retires before the end it grew to)
         lane_record(R, L, pos, sink.gen, sink.seq, R.end);
         atomicAdd(c.work, (unsigned long long) stepped);
      }
   }

#if defined(NFCB200_LANE_PROFILE)
   if (lane == 0)
      for (uint32_t i = 0; i < 2 * NFCB200_PROF_CLASSES; i++)
         atomicAdd(&nfcb200_lane_prof[i], prof[i]);
#endif

   // the last step's requests for a step that never came
   asm volatile("cp.async.wait_all;" ::: "memory");
}

// ---------------------------------------------------------------------------------------------------------------------
// front pass: one THREAD per segment, registers only (nfc_wlane.h front_pass) -> feature pool
// ---------------------------------------------------------------------------------------------------------------------
struct FrontConfig
{
   const void *samples;
   uint64_t n_samples;
   int sigtype;
   SegRec *segs;
   uint32_t n_segs;
   float4 *pool;
};

#define FRONT_THREADS 64

template <int SIG>
__global__ void __launch_bounds__(FRONT_THREADS) front_kernel(FrontConfig c, const __grid_constant__ Params dP)
{
   const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
   if (i >= c.n_segs)
      return;

   SegRec S = c.segs[i];
   const uint64_t streamBase = (uint64_t) S.stream * c.n_samples;
   float4 *dst = c.pool + S.featOff;

   front_pass(
      dP, S.first, S.end, [&](uint32_t p) { return load_sample(c.samples, SIG, streamBase + p); },
      [&](uint32_t k, float w, float env, float dev, float avg) { __stcs(dst + k, make_float4(w, env, dev, avg)); }, S);

   SegRec &O = c.segs[i];
   O.tEnv = S.tEnv;
   O.tAvg = S.tAvg;
   O.tDev = S.tDev;
   O.tF1 = S.tF1;
   O.tPulse = S.tPulse;
   O.hasFeat = 1;
}

// ---------------------------------------------------------------------------------------------------------------------
// warp lanes: one WARP per lane, rings + lane state in shared memory (nfc_wlane.h WLane)
// ---------------------------------------------------------------------------------------------------------------------
struct WLaneConfig
{
   const void *samples;
   uint64_t n_samples;
   int sigtype;
   const uint8_t *flags;
   const float *bsum;
   uint32_t n_blocks;
   LaneRec *lanes;
   const uint32_t *queue;
   uint32_t queue_count;
   uint32_t *cursor;         // work-stealing cursor over the queue
   const SegRec *segs;
   uint32_t n_segs;
   const float4 *pool;
   FramePool frames;
   unsigned long long *work; // samples consumed (statistics)
   unsigned long long *phase; // [16] cycles and samples per phase (development counters)
   int use_tma;
};

#define WALK_TILE 512u     /* samples per staged tile                                     */
#define WALK_STAGES 3u     /* tiles in flight: the W / D / M sample rings are idle during a walk and hold them */
#define WALK_STAGE_BYTES (NFCB200_RING * 4u)

struct DevWarp
{
   static __device__ __forceinline__ u32 lane() { return threadIdx.x & 31; }
   static __device__ __forceinline__ u32 width() { return 32; }
   static __device__ __forceinline__ void sync() { __syncwarp(); }
   static __device__ __forceinline__ u32 min_u32(u32 v) { return __reduce_min_sync(0xffffffffu, v); }
   static __device__ __forceinline__ u32 max_u32(u32 v) { return __reduce_max_sync(0xffffffffu, v); }
   static __device__ __forceinline__ u32 add_u32(u32 v) { return __reduce_add_sync(0xffffffffu, v); }
   static __device__ __forceinline__ u32 or_u32(u32 v) { return __reduce_or_sync(0xffffffffu, v); }
   static __device__ __forceinline__ unsigned long long clock() { return clock64(); }
   static __device__ __forceinline__ float add_f32(float v)
   {
#pragma unroll
      for (int d = 16; d > 0; d >>= 1)
         v += __shfl_xor_sync(0xffffffffu, v, d);
      return v;
   }

   // running sums of the cnt (<= 32) samples after the current step: the reference's recurrence (add, then subtract: two
   // roundings per sample, NfcA.cpp:246-247), one detector per thread on six threads
   template <class WL>
   static __device__ __forceinline__ void sum_chains(WL &wl, u32 cnt)
   {
      wl.sum_chains_seq(cnt);
   }

   /*
    * The idle stretch [pos, target) with the sums alone.  The raw samples are staged by the TMA engine (cp.async.bulk 1-D
    * under an mbarrier, three tiles of 512 samples in flight per warp -- the sample rings for w / deviation / envelope are
    * not needed until the lane re-enters the features and serve as the staging buffers), converted to the exact magnitude
    * into the x ring, and six threads advance the six sums over the tile with the reference's own recurrence.
    */
   template <class WL>
   static __device__ __noinline__ void walk(WL &wl, u32 pos, u32 target)
   {
      const auto &src = wl.src;
      const u32 bs = sig_bytes(src.sigtype);

      if (!src.use_tma || (pos & 31) || (target & 31) || target <= pos)
      {
         wl.walk_generic(pos, target);
         return;
      }

      const u32 lane = threadIdx.x & 31;
      const u32 kbase = wl.F.kbase;
      u32 k = wl.F.k;
      u32 phase = wl.sh.barPhase;

      // thread d < 6 owns the running sum of detector d for the whole walk
      const SumChain mine = sum_chain(wl.P, lane < 6 ? lane : 0);
      const bool chain = lane < 6 && (wl.P.enabled & mine.tech) != 0;
      float sum = chain ? wl.F.fi[mine.fi] : 0.0f;

      unsigned char *staging = reinterpret_cast<unsigned char *>(wl.rg + NFCB200_OFF_W);
      uint64_t *bar = reinterpret_cast<uint64_t *>(wl.sh.bar);
      const unsigned char *gsrc = (const unsigned char *) src.samples + src.streamBase * bs;
      const float *X = wl.rg + NFCB200_OFF_X;
      const u32 total = target - pos;
      const u32 ntiles = (total + WALK_TILE - 1) / WALK_TILE;

      auto issue = [&](u32 i) {
         const u32 st = i % WALK_STAGES;
         const u32 p = pos + i * WALK_TILE;
         const u32 cnt = target - p < WALK_TILE ? target - p : WALK_TILE;
         mbar_expect_tx(&bar[st], cnt * bs);
         tma_load_1d(staging + st * WALK_STAGE_BYTES, gsrc + (uint64_t) p * bs, cnt * bs, &bar[st]);
      };

      // earlier ring fills went through the generic proxy: order them before the bulk copies into the same memory
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncwarp();

      if (lane == 0)
         for (u32 i = 0; i < WALK_STAGES && i < ntiles; i++)
            issue(i);

      for (u32 i = 0; i < ntiles; i++)
      {
         const u32 st = i % WALK_STAGES;
         const u32 p = pos + i * WALK_TILE;
         const u32 cnt = target - p < WALK_TILE ? target - p : WALK_TILE;
         const unsigned char *raw = staging + st * WALK_STAGE_BYTES;

         mbar_wait(&bar[st], (phase >> st) & 1u);
         phase ^= 1u << st;

         // exact magnitudes of the tile into the x ring (all threads)
         for (u32 g = lane; g < cnt; g += 32)
            wl.rg[NFCB200_OFF_X + ((k + 1 + g + kbase) & (NFCB200_RING - 1))] = sample_from_raw(raw, src.sigtype, g);
         __syncwarp();

         // the staging buffer is free again
         if (lane == 0 && i + WALK_STAGES < ntiles)
            issue(i + WALK_STAGES);

         // the six sums over the tile: s += x[t - sdd]; s -= x[t - sdd - p2] (cnt is a multiple of 32)
         if (chain)
         {
            u32 ia = (k + 1 + kbase - mine.sdd) & (NFCB200_RING - 1);
            u32 ib = (k + 1 + kbase - mine.sdd - mine.p2) & (NFCB200_RING - 1);
            for (u32 g = 0; g < cnt; g += 8)
            {
               float a[8], b[8];
#pragma unroll
               for (u32 q = 0; q < 8; q++)
               {
                  a[q] = X[(ia + q) & (NFCB200_RING - 1)];
                  b[q] = X[(ib + q) & (NFCB200_RING - 1)];
               }
#pragma unroll
               for (u32 q = 0; q < 8; q++)
               {
                  sum += a[q];
                  sum -= b[q];
               }
               ia = (ia + 8) & (NFCB200_RING - 1);
               ib = (ib + 8) & (NFCB200_RING - 1);
            }
         }

         k += cnt;
         __syncwarp();
      }

      __syncwarp();

      if (chain)
         wl.F.fi[mine.fi] = sum;
      if (lane == 0)
      {
         wl.advance(total);
         wl.sh.barPhase = phase;
      }
      __syncwarp();
   }
};

struct DevSrc
{
   const void *samples;
   int sigtype;
   uint64_t streamBase;
   const float4 *pool;
   const uint8_t *flags; // this stream's block flags
   const float *bsum;    // this stream's block sums
   const SegRec *segs;
   uint32_t nsegs;
   int use_tma;          // stream pitch and base are 16-byte aligned: bulk copies allowed

   __device__ __forceinline__ float x(u32 pos) const { return load_sample(samples, sigtype, streamBase + pos); }
   __device__ __forceinline__ Feat feat(unsigned long long i) const
   {
      const float4 v = __ldcs(pool + i);
      Feat f;
      f.w = v.x;
      f.env = v.y;
      f.dev = v.z;
      f.avg = v.w;
      return f;
   }
   __device__ __forceinline__ bool active(u32 pos) const { return (flags[pos >> 8] & SCR_ACTIVE) != 0; }
   __device__ __forceinline__ float bmean(u32 b) const { return bsum[b] * (1.0f / NFCB200_BLOCK); }
   __device__ __forceinline__ const SegRec &seg(u32 i) const { return segs[i]; }
   __device__ __forceinline__ u32 nseg() const { return nsegs; }
   __device__ __forceinline__ bool exact_int() const { return sigtype == SIG_MAG_S16; }
};

// shared memory of one warp lane: sample / integration / correlation rings, the lane state, the stream byte buffer, scratch
struct WLaneSmem
{
   float rg[NFCB200_SCRATCH_FLOATS];
   Lane L;
   WShared sh;
   u8 sb[512];
};

__global__ void __launch_bounds__(32) wlanes_kernel(WLaneConfig c, const __grid_constant__ Params dP)
{
   extern __shared__ __align__(16) unsigned char wl_smem[];
   WLaneSmem &sm = *reinterpret_cast<WLaneSmem *>(wl_smem);
   const u32 lane = threadIdx.x;

   if (lane == 0)
   {
      for (u32 i = 0; i < WALK_STAGES; i++)
         mbar_init(reinterpret_cast<uint64_t *>(&sm.sh.bar[i]), 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
      sm.sh.barPhase = 0;
      for (u32 i = 0; i < 8; i++)
         sm.sh.cyc[i] = sm.sh.cnt[i] = 0;
   }
   __syncwarp();

   for (;;)
   {
      u32 qi = 0;
      if (lane == 0)
         qi = atomicAdd(c.cursor, 1u);
      qi = __shfl_sync(0xffffffffu, qi, 0);
      if (qi >= c.queue_count)
         break;

      const u32 li = c.queue[qi];
      LaneRec &R = c.lanes[li];

      // correlation rings must read as zero until written (a fresh reference decoder); the sample rings are only read after
      // the detector gate, the integration ring only after clear_for_listen()
      for (u32 i = NFCB200_OFF_CA + lane; i < NFCB200_SCRATCH_FLOATS; i += 32)
         sm.rg[i] = 0.0f;
      __syncwarp();

      DeviceSink sink;
      sink.pool = c.frames;
      sink.lane = li;
      sink.gen = R.gen + 1;
      sink.seq = 0;

      DevSrc src;
      src.samples = c.samples;
      src.sigtype = c.sigtype;
      src.streamBase = (uint64_t) R.stream * c.n_samples;
      src.pool = c.pool;
      src.flags = c.flags + (size_t) R.stream * c.n_blocks;
      src.bsum = c.bsum + (size_t) R.stream * c.n_blocks;
      src.segs = c.segs;
      src.nsegs = c.n_segs;
      src.use_tma = c.use_tma;

      WLane<DevWarp, DeviceSink, DevSrc> WL(dP, sm.L, sm.rg, sm.sb, sink, sm.sh, src);
      WL.run(R, R.seg0, (u32) c.n_samples);

      if (lane == 0)
      {
         lane_record(R, sm.L, sm.sh.pos, sink.gen, sink.seq, R.end);
         atomicAdd(c.work, (unsigned long long) sm.sh.stepped);
      }
      __syncwarp();
   }

   if (lane < 16)
      atomicAdd(c.phase + lane, lane < 8 ? sm.sh.cyc[lane] : sm.sh.cnt[lane - 8]);
}

// ---------------------------------------------------------------------------------------------------------------------
// carry chain
// ---------------------------------------------------------------------------------------------------------------------
struct ChainConfig
{
   const Carry *carryIn; // carry in front of the first lane of stream 0, or null (power-on)
   LaneRec *lanes;
   const uint32_t *offsets;
   const uint32_t *counts;
   uint32_t n_streams;
   uint32_t *queue;
   uint32_t *queue_count;
};

/*
 * chain_walk() (nfc_chain.h), one WARP per stream: the sequential part is the loop over the lanes of the stream, but everything done
 * per lane is word-parallel -- 246 carry words compared (word_observed_equal) and composed (compose_word) -- and the lane
 * records are read with coalesced loads instead of one thread chasing 2 kB per lane.  The true carry lives in shared
 * memory.  Control flow is uniform across the warp (every thread evaluates the same scalar fields); lane 0 writes the
 * scalar results.  Must stay equivalent to chain_walk() (nfc_chain.h), which the CPU tests exercise.
 */
#define CHAIN_WARPS 4
#define CARRY_WORDS (sizeof(Carry) / 4)

__device__ __forceinline__ void carry_word_group(u32 w, int &g, u32 &wi)
{
   const u32 mod = NFCB200_MOD_WORDS, tech = sizeof(TechSt) / 4;
   if (w < 3 * mod) { g = 0; wi = w; }
   else if (w < 5 * mod) { g = 1; wi = w - 3 * mod; }
   else if (w < 7 * mod) { g = 2; wi = w - 5 * mod; }
   else if (w < 8 * mod) { g = 3; wi = w - 7 * mod; }
   else if (w < 8 * mod + 4 * tech) { g = 4 + (int) ((w - 8 * mod) / tech); wi = (w - 8 * mod) % tech; }
   else { g = 8; wi = w - 8 * mod - 4 * tech; }
}

__global__ void __launch_bounds__(CHAIN_WARPS * 32) chain_warp_kernel(ChainConfig c, const __grid_constant__ Params dP)
{
   static_assert(sizeof(Carry) == (8 * sizeof(Mod) + 4 * sizeof(TechSt) + 12), "carry groups must tile the Carry");

   __shared__ u32 carry[CHAIN_WARPS][2][CARRY_WORDS];

   const u32 lane = threadIdx.x & 31;
   const u32 wib = threadIdx.x >> 5;
   const u32 s = blockIdx.x * CHAIN_WARPS + wib;
   if (s >= c.n_streams)
      return;

   const u32 off = c.offsets[s];
   const u32 n = c.counts[s];
   LaneRec *lanes = c.lanes + off;

   u32 *cur = carry[wib][0];
   u32 *next = carry[wib][1];

   {
      Carry pon;
      carry_init(pon, dP);
      carry_canon(pon);
      const u32 *raw = (c.carryIn && s == 0) ? (const u32 *) c.carryIn : (const u32 *) &pon;
      for (u32 w = lane; w < CARRY_WORDS; w += 32)
         cur[w] = raw[w];
   }
   __syncwarp();

   u32 ndirty = 0;
   int prev = -1;

   for (u32 j = 0; j < n; j++)
   {
      LaneRec &L = lanes[j];

      if (L.dead)
         continue;

      if (prev >= 0)
      {
         LaneRec &Q = lanes[prev];
         const u32 qStop = Q.stop, qEnd = Q.end, qGen = Q.gen, qDirty = Q.dirty;
         const u32 reach = qStop > qEnd ? qStop : qEnd;

         if (qGen > 0 && (!qDirty || qStop < qEnd) && reach > L.first)
         {
            const u32 lEnd = L.end;
            const u32 newEnd = qEnd < lEnd ? lEnd : qEnd;
            const bool wake = qStop < newEnd && !qDirty;
            __syncwarp();
            if (lane == 0)
            {
               L.dead = 1;
               L.dirty = 0;
               Q.end = newEnd;
               if (wake)
                  Q.dirty = 1;
            }
            if (wake)
               ndirty++;
            __syncwarp();
            continue;
         }
      }

      const bool ran = L.gen > 0;
      const u32 touched = 0x10F | ((L.lockedMask & 0xF) << 4);
      const u32 wasDirty = L.dirty;
      LaneObs obs = lane_obs(L);
      obs.inert = carry_inert_mask(*reinterpret_cast<const Carry *>(cur));
      const u32 *in = (const u32 *) &L.in;
      const u32 *out = (const u32 *) &L.out;

      bool bad = false;
      for (u32 w = lane; w < CARRY_WORDS; w += 32)
      {
         int g;
         u32 wi;
         carry_word_group(w, g, wi);
         const u32 t = cur[w];
         u32 nx = t;
         if (ran && ((touched >> g) & 1))
         {
            const u32 a = in[w];
            if (!word_observed_equal(obs, g, wi, a, t))
               bad = true;
            nx = compose_word(obs, g, wi, t, out[w], a);
         }
         next[w] = nx;
      }

      const bool ok = ran && !__any_sync(0xffffffffu, bad);

      if (!ok)
      {
         if (ran)
         {
            u32 *inw = (u32 *) &L.in; // a lane that never ran keeps the carry it was created with
            for (u32 w = lane; w < CARRY_WORDS; w += 32)
               inw[w] = cur[w];
         }
         if (lane == 0)
            L.dirty = 1;
      }

      if (!ok || wasDirty)
         ndirty++;

      __syncwarp();

      u32 *tmp = cur;
      cur = next;
      next = tmp;
      prev = (int) j;
   }

   if (!ndirty)
      return;

   __syncwarp();
   for (u32 j = lane; j < n; j += 32)
   {
      LaneRec &L = lanes[j];
      if (L.dirty && !L.dead)
         c.queue[atomicAdd(c.queue_count, 1u)] = off + j;
   }
}

// length of every lane's own region + halo (the host orders the first-round queue by it: lanes of similar length share a
// warp, long lanes start first)
__global__ void lane_length_kernel(const LaneRec *lanes, uint32_t n, uint32_t *length)
{
   uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
   if (i < n)
      length[i] = lanes[i].end - lanes[i].first;
}

// development statistics (NFCB200_TRACE): how far the lanes really ran -- histogram of stop - first in 4 096-sample bins
// [0..63], the longest run as (length << 32 | lane) in [64..65] (one 64-bit word)
__global__ void lane_run_stat_kernel(const LaneRec *lanes, uint32_t n, unsigned long long *out)
{
   uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
   if (i >= n || lanes[i].dead || lanes[i].gen == 0)
      return;
   const uint32_t len = lanes[i].stop - lanes[i].first;
   const uint32_t bin = len / 4096 < 63 ? len / 4096 : 63;
   atomicAdd(&out[bin], 1ull);
   atomicMax(&out[64], ((unsigned long long) len << 32) | i);
}

// carry in front of the first lane of stream 0 that begins at or after `sample` (nfc_chain.h carry_before)
__global__ void carry_before_kernel(LaneRec *lanes, uint32_t n, const Carry *carryIn, uint32_t sample, Carry *out, uint32_t *laneBegin, const __grid_constant__ Params dP)
{
   if (threadIdx.x != 0 || blockIdx.x != 0)
      return;
   Carry c;
   u32 b;
   carry_before(lanes, n, dP, carryIn, sample, c, b);
   *out = c;
   *laneBegin = b;
}

// ---------------------------------------------------------------------------------------------------------------------
// frame gather on the device: the frames of the final generation of the live lanes, ordered (stream, time), packed
// ---------------------------------------------------------------------------------------------------------------------
// Lanes are globally ordered by (stream, time) and a run numbers its frames 0 .. nframes-1, so the position of a frame is
// a counting sort: offset[lane] + seq, offset = exclusive scan of the frame counts of the live lanes.

// one block: exclusive scan of the lanes' frame counts (dead lanes count 0) -> laneOff[0 .. n], live lane count
__global__ void __launch_bounds__(1024) frame_offsets_kernel(const LaneRec *lanes, uint32_t n, uint32_t *laneOff, unsigned long long *liveCount)
{
   __shared__ uint32_t warpSum[32];
   __shared__ uint32_t carry;
   const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
   uint32_t live = 0;

   if (tid == 0)
      carry = 0;
   __syncthreads();

   for (uint32_t base = 0; base < n; base += 1024)
   {
      const uint32_t i = base + tid;
      uint32_t v = 0;
      if (i < n && !lanes[i].dead)
      {
         v = lanes[i].nframes;
         live++;
      }
      uint32_t incl = v;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1)
      {
         const uint32_t o = __shfl_up_sync(0xffffffffu, incl, d);
         if ((int) lane >= d)
            incl += o;
      }
      if (lane == 31)
         warpSum[warp] = incl;
      __syncthreads();
      if (warp == 0)
      {
         uint32_t w = warpSum[lane];
#pragma unroll
         for (int d = 1; d < 32; d <<= 1)
         {
            const uint32_t o = __shfl_up_sync(0xffffffffu, w, d);
            if ((int) lane >= d)
               w += o;
         }
         warpSum[lane] = w; // inclusive over warps
      }
      __syncthreads();
      const uint32_t before = carry + (warp ? warpSum[warp - 1] : 0) + (incl - v);
      if (i < n)
         laneOff[i] = before;
      __syncthreads();
      if (tid == 1023)
         carry = before + v;
      __syncthreads();
   }

   if (tid == 0)
      laneOff[n] = carry;

   live = __reduce_add_sync(0xffffffffu, live);
   if (lane == 0 && live)
      atomicAdd(liveCount, (unsigned long long) live);
}

// scatter the kept records to their final position; `.lane` of a packed record holds the STREAM of the frame (offset by
// streamBase), extension chunks are re-packed behind extBase
__global__ void frame_compact_kernel(const FrameRec *pool, uint32_t nRecs, const LaneRec *lanes, uint32_t nLanes, const uint32_t *laneOff,
                                     const u8 *ext, uint32_t extChunks, uint32_t streamBase, FrameRec *out, u8 *extOut, uint32_t extCap, uint32_t *extCount)
{
   for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nRecs; i += gridDim.x * blockDim.x)
   {
      const FrameRec r = pool[i];
      if (r.lane >= nLanes)
         continue;
      const LaneRec &L = lanes[r.lane];
      if (L.dead || L.gen != r.gen || r.seq >= L.nframes)
         continue;

      FrameRec o = r;
      o.lane = streamBase + L.stream;
      o.ext = 0xFFFFFFFFu;

      if (r.len > 80)
      {
         const uint32_t rest = r.len - 80, chunks = (rest + 127) / 128;
         if (r.ext != 0xFFFFFFFFu && r.ext + chunks <= extChunks)
         {
            const uint32_t e = atomicAdd(extCount, chunks);
            if (e + chunks <= extCap)
            {
               const uint4 *src = reinterpret_cast<const uint4 *>(ext + (size_t) r.ext * 128);
               uint4 *dst = reinterpret_cast<uint4 *>(extOut + (size_t) e * 128);
               for (uint32_t k = 0; k < chunks * 8; k++)
                  dst[k] = src[k];
               o.ext = e;
            }
            else
               o.len = 80;
         }
         else
            o.len = 80; // extension chunk missing (pool exhausted, reported by the caller): truncated payload
      }

      out[laneOff[r.lane] + r.seq] = o;
   }
}

// ---------------------------------------------------------------------------------------------------------------------
// streaming: one sequential lane per handle, suspended / resumed across pushes, skipping idle blocks exactly like the
// batch lanes do (cold start HALO samples before the next active block from the exact carry it retired with)
// ---------------------------------------------------------------------------------------------------------------------
struct StreamState
{
   Lane L;
   Carry carry;     // exact canonical carry at `pos` while parked
   u32 running;     // 1: L is a live lane positioned at `pos`; 0: parked (dormant)
   u32 contig;      // parked only: L is still positioned exactly at `pos` (it can be resumed instead of cold started)
   u32 pos;         // absolute index of the next sample to consume
   u32 seq;
};

struct StreamConfig
{
   const void *samples;   // device buffer holding absolute samples [base, base + count)
   uint32_t base;
   uint32_t count;
   int sigtype;
   const uint8_t *flags;  // one byte per block, flags[0] is absolute block flagBase
   uint32_t flagBase;
   uint32_t flagCount;
   uint32_t limit;        // process samples < limit (absolute); limit <= base + count
   uint32_t final;        // end of stream: do not wait for more data
   StreamState *state;
   float *scratch;        // NFCB200_SCRATCH_FLOATS floats
   uint8_t *sbuf;         // 512 bytes
   FramePool pool;
};

__global__ void stream_kernel(StreamConfig c, const __grid_constant__ Params dP)
{
   if (threadIdx.x != 0 || blockIdx.x != 0)
      return;

   StreamState &S = *c.state;

   Lane L = S.L;

   DeviceSink sink;
   sink.pool = c.pool;
   sink.lane = 0;
   sink.gen = 1;
   sink.seq = S.seq;

   Machine<1, DeviceSink> M(dP, L, L.fe, c.scratch, c.sbuf, sink);

   u32 pos = S.pos;
   u32 running = S.running;
   u32 contig = S.contig;
   u32 noParkBefore = 0; // a resumed lane steps through the idle samples up to the next active block without re-parking

   auto active = [&](u32 p) -> bool {
      u32 b = p >> 8;
      if (b < c.flagBase || b - c.flagBase >= c.flagCount)
         return true; // blocks not screened yet count as active
      return (c.flags[b - c.flagBase] & SCR_ACTIVE) != 0;
   };

   while (pos < c.limit)
   {
      if (!running)
      {
         // parked: next active block at or after pos
         u32 b = pos >> 8;
         const u32 lastBlock = (c.limit - 1) >> 8;
         while (b <= lastBlock && !active(b << 8))
            b++;

         if (b > lastBlock)
         {
            // idle to the end of the known data.  Skip ahead, but never so far that a block turning active later
            // (the last block is still filling) could not get its full warm-up
            u32 hold = c.final ? c.limit : ((lastBlock << 8) > NFCB200_HALO ? (lastBlock << 8) - NFCB200_HALO : 0);
            if (hold > pos)
            {
               pos = hold;
               contig = 0;
            }
            break;
         }

         u32 begin = b << 8;
         if (begin < pos)
            begin = pos;

         if (begin >= pos + NFCB200_HALO || !contig)
         {
            // cold start HALO samples early from the exact carry (lane_begin restarts front end, rings, running sums)
            u32 first = begin >= pos + NFCB200_HALO ? begin - NFCB200_HALO : pos;
            for (u32 i = NFCB200_OFF_CA; i < NFCB200_SCRATCH_FLOATS; i++)
               c.scratch[i] = 0.0f;
            lane_begin(L, dP, S.carry, first, first ? NFCB200_HALO : 0);
            M.reload_front();
            pos = first;
         }
         // else: too close for a cold start and the parked machine is still positioned at pos: resume it

         noParkBefore = begin;
         running = 1;
         contig = 1;
      }

      while (pos < c.limit)
      {
         if (pos >= noParkBefore && !active(pos) && M.dormant())
         {
            S.carry = L.c;
            S.carry.edgeTime = L.fe.edgeTime;
            carry_canon(S.carry);
            running = 0;
            contig = 1;
            break;
         }

         M.step(load_sample(c.samples, c.sigtype, (uint64_t) (pos - c.base)));
         pos++;
      }
   }

   S.L = L;
   S.pos = pos;
   S.running = running;
   S.contig = contig;
   S.seq = sink.seq;
}

}

#endif
