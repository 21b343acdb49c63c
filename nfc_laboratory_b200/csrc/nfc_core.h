/*
 * nfc_core.h -- the exact per-sample decoder state machine ("lane"), compiled for the device by nvcc (csrc/nfc_decode.cu,
 * one lane per capture segment) and, for GPU-less CI only, by g++ inside tests/native/host_sim.cpp.
 *
 * This is NOT a port of the reference's nested `while (decoder->nextSample(buffer))` loops: the reference runs one
 * blocking loop per symbol decoder (NfcA.cpp:821, 948, 1104, 1230, 1343 ...).  Here the whole decoder is ONE flat
 * transition function `lane_step(x)` -- one sample in, at most one frame out -- so that 32 lanes of a warp (32 different
 * capture segments) advance in lock step, address their history rings with the same relative slot (coalesced, see
 * RG()), and can be suspended / resumed at any sample.  Every arithmetic expression keeps the reference's operation
 * order and float types (no FMA contraction: compile with -fmad=false / -ffp-contract=off) so that decisions are
 * bit-identical; each block cites the reference lines it restates.
 *
 * Ring addressing: the reference indexes its rings with the absolute clock (`clock & 1023`, `(1024 - sdd + clock) % p1`).
 * All accesses have the form (clock + const), so a per-lane rotation of slot labels is unobservable; lanes use the
 * LOCAL step counter k (same value in every lane of a warp) instead, which is what makes the accesses coalesce.
 */
#ifndef NFCB200_CORE_H
#define NFCB200_CORE_H

#include "nfc_params.h"

#if defined(__CUDACC__)
#define NFC_HD __host__ __device__ __forceinline__
#define NFC_HDN __host__ __device__ __noinline__
#else
#define NFC_HD inline
#define NFC_HDN inline
#endif

// per-sample value tap for the tests (tests/native/host_sim.cpp defines NFCB200_TRACE_VALUES and the sink); the product
// build compiles it away.  Channels follow the reference's signal debugger (NfcTech.h:32-37).
#if defined(NFCB200_TRACE_VALUES)
#define NFC_TRACE(ch, v) nfcb200_trace_value((ch), (v))
#else
#define NFC_TRACE(ch, v) ((void) 0)
#endif

namespace nfcb200 {

// ---------------------------------------------------------------------------------------------------------------------
// state
// ---------------------------------------------------------------------------------------------------------------------

// per-rate detector / symbol-decoder status (reference: NfcModulationStatus, NfcTech.h:221-259, minus the two rings)
struct Mod
{
   u32 searchModeState;
   u32 searchStartTime;
   u32 searchEndTime;
   u32 searchSyncTime;
   u32 searchPulseWidth;
   float searchValueThreshold;
   float searchPhaseThreshold;
   float searchLastPhase;
   float searchLastValue;
   float searchSyncValue;
   float searchCorrDValue;
   float searchCorr0Value;
   float searchCorr1Value;
   u32 symbolStartTime;
   u32 symbolEndTime;
   u32 symbolRiseTime;
   float filterIntegrate;
   float phaseIntegrate;
   float correlatedPeakValue;
   float detectorPeakValue;
   u32 correlatedPeakTime;
   u32 detectorPeakTime;
};

// NfcSymbolStatus (NfcTech.h:264-273); start/end/edge hold 32-bit values in the reference as well
struct Sym
{
   u32 pattern, value, start, end, edge, length;
};

// NfcStreamStatus (NfcTech.h:278-289) without the byte buffer (kept in lane scratch)
struct Bits
{
   u32 previous, pattern, bits, skip, data, flags, parity, bytes;
};

// NfcFrameStatus (NfcTech.h:294-315)
struct FrameSt
{
   u32 lastCommand, frameType, symbolRate, frameStart, frameEnd, guardEnd, waitingEnd;
   u32 frameGuardTime, frameWaitingTime, startUpGuardTime, requestGuardTime;
};

// NfcProtocolStatus (NfcA.cpp:74-91 and twins)
struct Proto
{
   u32 maxFrameSize, frameGuardTime, frameWaitingTime, startUpGuardTime, requestGuardTime;
};

struct TechSt
{
   FrameSt fs;
   Proto ps;
   u32 chained;
};

// bit of Lane::lcWritten for word k of Proto (maxFrameSize, frameGuardTime, frameWaitingTime, startUpGuardTime, requestGuardTime)
#define NFCB200_PSW(t, k) (1u << (8 + 5 * (t) + (k)))

// the part of the decoder that survives between capture segments ("carry"): everything except the front-end
// recurrences and the rings, which a lane re-derives over its warm-up halo (DESIGN.md, "segment speculation")
struct Carry
{
   Mod mA[3];
   Mod mB[2];
   Mod mF[2]; // rates 212, 424
   Mod mV;
   TechSt t[4];
   u32 carrierOn;  // carrierOnTime  (0 = unset)
   u32 carrierOff; // carrierOffTime (0 = unset)
   u32 edgeTime;   // carrierEdgeTime (NfcTech.cpp:77-92): the time of the last strong edge, however old, stamps the next carrier
                   // frame (NfcDecoder.cpp:477, 502).  The working copy is Front::edgeTime; this is its value at lane boundaries
};

// front end (NfcDecoderStatus scalars, NfcTech.h:317-393) plus the rest of the state a lane touches on EVERY sample.
// On the device this block lives in shared memory (31 words per lane, odd stride: no bank conflicts), everything else
// of a lane in thread-local memory: with 16 resident warps per SM the local state (1.4 kB per lane) does not fit the L1
// cache, and the per-sample fields were the bulk of its traffic.
struct Front
{
   u32 clk;         // signalClock
   u32 k;           // local step since the (re)start of the lane: warm-up gate, detector gate
   u32 kbase;       // k + kbase labels the ring slots: equal in all lanes of a warp -> coalesced ring traffic
   u32 pulseFilter;
   u32 closed;      // leaky count of samples with the envelope gate closed (lane retirement only, not in the reference)
   float env, avg, dev, f1;
   float edgePeak;
   u32 edgeTime;
   // correlation ring phases, advanced every sample (replaces the reference's three `%` per rate per sample)
   u32 cA[3], cF[2], cV1, cV0;
   // the detectors' running sums (NfcModulationStatus::filterIntegrate), indexed like the Mods of Carry: mA[0..2],
   // mB[0..1] (unused), mF[0..1], mV.  They never cross lanes: a lane restarts them with its rings (carry_canon)
   float fi[8];
   // bit i: Mod i has search state pending, i.e. the precondition of its detector's idle fast path is false
   u32 busy;
   u32 lock;      // LOCK_*
   u32 lockRate;  // rate index of the locked modulation
   u32 gate;      // local steps during which the detectors are off (reference: signalClock < BUFFER_SIZE)
   u32 warm;      // local steps during which carrier detection is suppressed (cold-started lanes)
   u32 edgeHold;  // local steps during which the carrier-edge tracker is off: the DC-removal filter of a cold-started front end
                  // rings for a few samples (w starts at x), which is not an edge of the signal
   u32 gateSum;   // local steps before which not even the detectors' running sums advance (<= gate).  Between gateSum and
                  // gate only the sums and their correlation rings run (sums_only()): a lane that skipped an idle stretch with
                  // its sums carried exactly (nfc_wlane.h) refills the rings this way before its detectors open
};

enum { LOCK_NONE = 0, LOCK_A = 1, LOCK_B = 2, LOCK_F = 3, LOCK_V = 4 };

struct Lane
{
   Front fe;
   Carry c;
   Sym sym;
   Bits st;
   u32 pulseBits; // NFC-V pulse code: 2 or 8 (decoder->pulse)
   u32 lockedMask; // techs that were locked at least once during this run (bit t), for the carry dependency check
   // finer dependency tracking of the run on its incoming carry (nfc_chain.h chain_walk):
   u32 lcWritten;  // bit t: frameStatus.lastCommand of tech t was assigned during this run; bit 8 + 5 t + k: word k of tech t's
                   // protocol status (NFCB200_PSW) was assigned -- only used to PREDICT the carry behind a run that must be
                   // repeated (nfc_chain.h compose_word): a run that assigns the value it happened to start from did assign it
   u32 lcLive;     // bit t: ... and was read by a listen frame before any assignment (the run depends on the carry value)
   u32 fZeroed;    // bit r: NFC-F rate r searchPulseWidth was reset during this run (restart / reset / listen clear)
   u32 fThrWritten;// bit r: NFC-F rate r searchValueThreshold was assigned during this run; bit 2 + r: searchLastValue; bit 4 + r: searchLastPhase
   u32 fThrRead;   // bit r: ... and was compared before any assignment, against fThrSync[r]; bits 2 + r / 4 + r: the incoming
                   // searchLastValue / searchLastPhase was read before the run assigned it (NfcF.cpp:300, 344, 349)
   u32 edgeWritten;// the carrier edge time was assigned during this run (an edge, or the reset after a carrier frame)
   u32 edgeLive;   // ... and a carrier frame read it before any assignment (the run depends on the carried value)
   u32 fInc0[2];   // `searchPulseWidth++ < 94` tests executed before the first reset (NfcF.cpp:307)
   float fThrSync[2];
};

// one decoded frame (payload stays in the lane's byte buffer until the sink copies it)
struct FrameOut
{
   u32 tech, type, flags, phase, rate, start, end, len;
};

// ---------------------------------------------------------------------------------------------------------------------
// CRC (reference: lab-data Crc.cpp:96-112 -- table driven there, bitwise here, same polynomial and bit order)
// ---------------------------------------------------------------------------------------------------------------------
NFC_HD unsigned short crc_ccitt16(const u8 *data, u32 from, u32 to, unsigned short init, bool refin)
{
   unsigned short crc = init;

   if (to == from)
      return (unsigned short) ~init;

   if (refin)
   {
      for (u32 i = from; i < to; i++)
      {
         crc ^= data[i];
         for (int b = 0; b < 8; b++)
            crc = (crc & 1) ? (unsigned short) ((crc >> 1) ^ 0x8408) : (unsigned short) (crc >> 1);
      }
   }
   else
   {
      for (u32 i = from; i < to; i++)
      {
         crc ^= (unsigned short) (data[i] << 8);
         for (int b = 0; b < 8; b++)
            crc = (crc & 0x8000) ? (unsigned short) ((crc << 1) ^ 0x1021) : (unsigned short) (crc << 1);
      }
   }

   return crc;
}

// NfcA.cpp:1994-2005
NFC_HD bool odd_parity_ok(u32 value, u32 parity)
{
   for (u32 i = 0; i < 8; i++)
      if (value & (1u << i))
         parity ^= 1;
   return parity != 0;
}

// NfcTech.cpp:39-42: abs(x - env) / env < 0.05f.  The IEEE division is only executed when the quotient is within 2 % of the
// threshold; outside that band the comparison is decided by a / env <= 0.049 (1 + ulp) < 0.05 resp. >= 0.051 (1 - ulp) > 0.05.
// The shortcut needs a positive envelope: a negative one (mono input with negative samples) makes the reference's quotient
// negative, i.e. "open", and env == 0 gives inf / NaN, which compare false there as well as here.
NFC_HD bool gate_open(float adiff, float env)
{
   if (env > 0.0f)
   {
      if (adiff < 0.049f * env)
         return true;
      if (adiff > 0.051f * env)
         return false;
   }
   return (adiff / env) < 0.05f;
}

// ---------------------------------------------------------------------------------------------------------------------
// lane machine.  STRIDE = 1 on the host, 32 on the device (scratch words of the 32 lanes of a warp are interleaved).
// SINK must provide: void frame(const FrameOut &f, const u8 *payload)
// ---------------------------------------------------------------------------------------------------------------------
// TAPS selects how the search-mode detectors fetch their ring taps (device latency hiding, no semantics):
//   0  where the reference reads them (one dependent ring access after the other)
//   2  staged one step ahead (Machine::stage_advance): the taps step k + 1 reads are requested during step k into a
//      per-lane stage -- shared memory filled by cp.async on the device, a plain copy on the host -- and the taps of
//      delay 1 are forwarded from the write that produces them; locked lanes other than NFC-A poll frames and NFC-A
//      106 kbps (ASK) listen frames get prefetch hints for their next step
// Word index of a tap inside one stage buffer.  The locked NFC-A poll decoder uses the words of its own rate; the locked
// NFC-A ASK listen decoder (rate 0, sdd == 0) reuses them for I[t-p2] of the integration ring (TAP_XA1) and C[fp2].
enum : u32
{
   TAP_XA0 = 0,   // NFC-A x[t-sdd] per rate (rate 0 has sdd == 0: the current sample, never staged)
   TAP_XA1 = 3,   // NFC-A x[t-sdd-p2]
   TAP_CA2 = 6,   // NFC-A C[fp2]
   TAP_WB = 9,    // NFC-B w[t-sdd] per rate (rate 0: the current edge value, never staged)
   TAP_XF1 = 11,  // NFC-F 212 / 424 x[t-p2]
   TAP_CF2 = 13,  // NFC-F C[fp2]
   TAP_XV0 = 15,  // NFC-V x[t-sdd]
   TAP_XV1 = 16,  // NFC-V x[t-sdd-p2]
   TAP_CV2 = 17,  // NFC-V C[fp2]
   TAP_FWD = 18,  // forwarded C[fp3] (slot c - 1, written by the previous step): NFC-A rates 0..2, then NFC-F 212 / 424
   TAP_COUNT = 23
};

// threads per block of the kernel that stages taps (nfc_decode.cuh lanes_kernel): the word stride of its stage
#define NFCB200_LANE_THREADS 128

// A tap is requested one step before it is read, before that step writes its own ring slots, so every requested tap
// must be at least two steps old when it is read.  True when that holds at the periods of P; otherwise nothing is staged.
NFC_HD bool taps_stageable(const Params &P)
{
   bool ok = true;
   for (int r = 0; r < 3; r++)
   {
      const RateParams &b = P.A[r];
      ok = ok && (b.sdd == 0 || b.sdd >= 2) && b.sdd + b.p2 >= 2 && b.p1 >= b.p2 + 2; // C[fp2] is p1 - p2 steps old
   }
   // the ASK listen decoder (rate 0: sdd == 0) reads w of the current step and writes I[t] each step: I[t-p2] is p2 steps old
   ok = ok && P.A[0].sdd == 0 && P.A[0].p2 >= 2;
   for (int r = 0; r < 2; r++)
      ok = ok && (P.B[r].sdd == 0 || P.B[r].sdd >= 2);
   for (int r = 1; r <= 2; r++)
   {
      const RateParams &b = P.F[r];
      ok = ok && b.sdd + b.p2 >= 2 && b.p1 >= b.p2 + 2;
   }
   return ok && P.V.sdd >= 2 && P.V.p1 >= P.V.p2 + 2;
}

#if defined(NFCB200_CHECK_TAPS)
// development check: every staged tap that is used is compared with a direct ring read (nfcb200.cu reports the counts);
// nfcb200_taps_kind counts the used taps by the kind of the stage they came from (Machine::stgState bits 0-2)
#if defined(__CUDACC__)
static __device__ unsigned long long nfcb200_taps_used, nfcb200_taps_differ, nfcb200_taps_kind[8];
#else
static unsigned long long nfcb200_taps_used, nfcb200_taps_differ, nfcb200_taps_kind[8];
#endif
#endif

// CG: ring accesses bypass the L1 cache (ld/st.global.cg).  A ring line is written once and read a few times hundreds
// of steps later -- no L1 reuse -- while the lanes' local state and sample lines live in the same L1.
template <int STRIDE, class SINK, int TAPS = 0, bool CG = false>
struct Machine
{
   // one ring word: converts to float (load) and takes a float (store)
   struct RingRef
   {
      float *p;

      NFC_HD operator float() const
      {
#if defined(__CUDA_ARCH__)
         if (CG)
            return __ldcg(p);
#endif
         return *p;
      }

      NFC_HD void operator=(float v) const
      {
#if defined(__CUDA_ARCH__)
         if (CG)
         {
            __stcg(p, v);
            return;
         }
#endif
         *p = v;
      }
   };

   const Params &P;
   Lane &L;
   Front &F;  // the per-sample state: L.fe itself, or its working copy in shared memory (device lanes)
   float *rg; // lane scratch (already offset by the lane index on the device)
   u8 *sb;    // 512-byte stream buffer
   SINK &sink;
   // TAPS == 2: two stage buffers, this step's (F.k & 1) and the next step's; word (buf, tap) at
   // stage_base()[(buf * TAP_COUNT + tap) * STG_STRIDE].  The device passes the lane's column of a shared-memory array
   // ([buf][tap][thread]: no bank conflicts); the host build keeps its own.
   static constexpr u32 STG_STRIDE = STRIDE == 1 ? 1 : NFCB200_LANE_THREADS;
   float *stg;
   float ownStage[TAPS == 2 && STRIDE == 1 ? 2 * TAP_COUNT : 1];
   // STG_ON | kind of this step's stage (bits 0-2) | kind of the next step's (3-5) | forwarded taps present in this
   // step's (8-12) | in the next step's (16-20).  Kind: 0 nothing staged, KIND_SEARCH, KIND_POLL + NFC-A rate,
   // KIND_LISTEN_ASK + NFC-A rate (only rate 0, 106 kbps, listens with ASK).
   u32 stgState;
   static constexpr u32 STG_ON = 1u << 31, KIND_SEARCH = 1, KIND_POLL = 2, KIND_LISTEN_ASK = 5;
   float curX, curW;  // sample and edge value of the current step (ring slot of delay 0)
   bool slow;         // a detector left its idle fast path during this step: F.busy must be rebuilt
   // feature-fed front end (nfc_wlane.h): the recurrences of nextSample were evaluated by the front pass, the sample rings
   // are already filled for this step; only the scalars the detectors read are taken over
   bool featMode;
   float featAvg;

   NFC_HD Machine(const Params &p, Lane &l, Front &f, float *r, u8 *s, SINK &k)
      : P(p), L(l), F(f), rg(r), sb(s), sink(k), stg(nullptr), stgState(0), curX(0), curW(0), slow(false), featMode(false),
        featAvg(0)
   {
      if constexpr (TAPS == 2 && STRIDE == 1)
         stgState = taps_stageable(P) ? STG_ON : 0;
   }

   // TAPS == 2 on the device: the lane's stage (column threadIdx.x of a [2][TAP_COUNT][NFCB200_LANE_THREADS] array in
   // shared memory); `stageable` = taps_stageable(P), evaluated once per launch
   NFC_HD void attach_stage(float *s, bool stageable)
   {
      stg = s;
      stgState = stageable ? STG_ON : 0;
   }

   // running sum of a Mod (index = position of the Mod inside Carry: mA, mB, mF, mV are contiguous)
   NFC_HD float &FI(const Mod &m)
   {
      return F.fi[(u32) (&m - &L.c.mA[0])];
   }

   // (re)load the working copy of the per-sample state after lane_begin() rewrote L.fe, and rebuild the busy mask
   NFC_HD void reload_front()
   {
      if (&F != &L.fe)
         F = L.fe;
      refresh_busy();
      slow = false;
      stage_reset(); // new ring slot labels (k, kbase), rings wiped by the caller
   }

   // write the working copy back (suspended lanes: streaming entry point)
   NFC_HD void store_front()
   {
      if (&F != &L.fe)
         L.fe = F;
   }

   NFC_HD void refresh_busy()
   {
      u32 b = 0;
      for (int r = 0; r < 3; r++)
      {
         const Mod &m = L.c.mA[r];
         if (m.symbolStartTime | m.searchStartTime | m.searchEndTime | m.correlatedPeakTime)
            b |= 1u << r;
      }
      for (int r = 0; r < 2; r++)
      {
         const Mod &m = L.c.mB[r];
         if (m.symbolStartTime | m.searchEndTime | m.detectorPeakTime)
            b |= 8u << r;
         const Mod &f = L.c.mF[r];
         if (f.symbolStartTime | f.symbolEndTime | f.searchStartTime | f.searchEndTime | f.searchSyncTime | f.correlatedPeakTime)
            b |= 32u << r;
      }
      {
         const Mod &m = L.c.mV;
         if (m.searchStartTime | m.searchEndTime | m.correlatedPeakTime)
            b |= 128u;
      }
      F.busy = b;
   }

#define RG(off, i) (RingRef {&rg[((off) + (i)) * STRIDE]})
#define SMP(off, delay) RG(off, (F.k + F.kbase - (delay)) & (NFCB200_RING - 1))

   NFC_HD void zero_mod(Mod &m)
   {
      m.searchModeState = 0;
      m.searchStartTime = 0;
      m.searchEndTime = 0;
      m.searchSyncTime = 0;
      m.searchPulseWidth = 0;
      m.searchValueThreshold = 0;
      m.searchPhaseThreshold = 0;
      m.searchLastPhase = 0;
      m.searchLastValue = 0;
      m.searchSyncValue = 0;
      m.searchCorrDValue = 0;
      m.searchCorr0Value = 0;
      m.searchCorr1Value = 0;
      m.symbolStartTime = 0;
      m.symbolEndTime = 0;
      m.symbolRiseTime = 0;
      FI(m) = 0;
      m.phaseIntegrate = 0;
      m.correlatedPeakValue = 0;
      m.detectorPeakValue = 0;
      m.correlatedPeakTime = 0;
      m.detectorPeakTime = 0;
   }

   NFC_HD void zero_ring(u32 off, u32 len)
   {
      for (u32 i = 0; i < len; i++)
         RG(off, i) = 0;
      stage_drop();
   }

   NFC_HD void clear_bits()
   {
      L.st.previous = L.st.pattern = L.st.bits = L.st.skip = L.st.data = L.st.flags = L.st.parity = L.st.bytes = 0;
   }

   NFC_HD void clear_sym()
   {
      L.sym.pattern = L.sym.value = L.sym.start = L.sym.end = L.sym.edge = L.sym.length = 0;
   }

   NFC_HD void put_byte(u32 value)
   {
      // the reference writes streamStatus.buffer[512] unchecked (maxFrameSize may reach 4096, NfcA.cpp:1716); cap here
      if (L.st.bytes < 512)
         sb[L.st.bytes] = (u8) value;
      L.st.bytes++;
   }

   NFC_HD Mod &locked_mod()
   {
      switch (F.lock)
      {
         case LOCK_A:
            return L.c.mA[F.lockRate];
         case LOCK_B:
            return L.c.mB[F.lockRate];
         case LOCK_F:
            return L.c.mF[F.lockRate - 1];
         default:
            return L.c.mV;
      }
   }

   NFC_HD const RateParams &locked_rate() const
   {
      switch (F.lock)
      {
         case LOCK_A:
            return P.A[F.lockRate];
         case LOCK_B:
            return P.B[F.lockRate];
         case LOCK_F:
            return P.F[F.lockRate];
         default:
            return P.V;
      }
   }

   // the "clear modulation status for receiving card response" block shared by all techs (NfcA.cpp:491-511,
   // NfcB.cpp:515-535, NfcF.cpp:483-503, NfcV.cpp:509-529): field-wise clear + memset of both rings
   NFC_HD void clear_for_listen(Mod &m, u32 corrOff, u32 corrLen)
   {
      m.symbolStartTime = 0;
      m.symbolEndTime = 0;
      FI(m) = 0;
      m.phaseIntegrate = 0;
      m.searchModeState = 0;
      m.searchSyncTime = 0;
      m.searchStartTime = 0;
      m.searchEndTime = 0;
      m.searchPulseWidth = 0;
      m.searchLastValue = 0;
      m.searchLastPhase = 0;
      m.searchValueThreshold = 0;
      m.searchPhaseThreshold = 0;
      m.correlatedPeakValue = 0;
      zero_ring(NFCB200_OFF_I, NFCB200_RING);
      if (corrLen)
         zero_ring(corrOff, corrLen);
   }

   NFC_HD void emit(u32 tech, u32 type, u32 flags, u32 phase, u32 rate, u32 start, u32 end, const u8 *payload, u32 len)
   {
      FrameOut f;
      f.tech = tech;
      f.type = type;
      f.flags = flags;
      f.phase = phase;
      f.rate = rate;
      f.start = start;
      f.end = end;
      f.len = len > 512 ? 512 : len;
      sink.frame(f, payload);
   }

   // ------------------------------------------------------------------------------------------------------------------
   // front end: NfcDecoderStatus::nextSample, NfcTech.cpp:28-105
   // ------------------------------------------------------------------------------------------------------------------
   // clock and ring phases of the new sample (first half of nextSample: everything that does not need the value)
   NFC_HD void front_advance()
   {
      Front &f = F;

      ++f.clk;
      ++f.k;
      ++f.pulseFilter;

      // correlation ring phases (signalIndex % period), kept incrementally
      for (int r = 0; r < 3; r++)
         if (++f.cA[r] == P.A[r].p1)
            f.cA[r] = 0;
      for (int r = 0; r < 2; r++)
         if (++f.cF[r] == P.F[r + 1].p1)
            f.cF[r] = 0;
      if (++f.cV1 == P.V.p1)
         f.cV1 = 0;
      if (++f.cV0 == P.V.p0)
         f.cV0 = 0;
   }

   NFC_HD void front(float x)
   {
      Front &f = F;

      // NfcTech.cpp:39-42: signalDiff = abs(x - env) / env; gate = signalDiff < 0.05f.  The IEEE division is only
      // executed when the quotient is within 2 % of the threshold; outside that band the comparison is decided by
      // a / env <= 0.049 (1 + ulp) < 0.05 resp. >= 0.051 (1 - ulp) > 0.05 (inf / NaN at env == 0 compare false, as there)
      const float adiff = fabsf(x - f.env);
      const bool open = gate_open(adiff, f.env);

      // retirement bookkeeping: while the gate stays closed the envelope is stale and thresholds derived from it
      // differ from what the screening pass assumes, so such a lane is never dormant
      if (open)
         f.closed = f.closed ? f.closed - 1 : 0;
      else if (f.closed < 4096)
         f.closed++;

      if (open || f.pulseFilter > (u32) (P.etu * 10))
      {
         f.pulseFilter = 0;
         f.env = f.env * P.envW0 + x * P.envW1;
      }
      else if (f.k - 1 < (u32) P.etu) // reference: signalClock < elementaryTimeUnit (k - 1 == clock on a fresh stream)
      {
         f.env = x;
      }

      float n0 = x + f.f1 * P.iirA; // :56
      float w = n0 - f.f1;          // :59
      f.f1 = n0;                    // :62

      f.dev = f.dev * P.mdevW0 + fabsf(w) * P.mdevW1; // :65
      f.avg = f.avg * P.meanW0 + x * P.meanW1;        // :68

      // the ring keeps the envelope instead of modulateDepth (:74): the depth is only read on detector triggers and
      // in listen mode, and depth_at() evaluates the reference expression from the stored x and envelope when it is
      SMP(NFCB200_OFF_X, 0) = x;
      SMP(NFCB200_OFF_W, 0) = w;
      curX = x;
      curW = w;
      NFC_TRACE(0, x);     // NfcTech.cpp:98-101
      NFC_TRACE(1, w);
      NFC_TRACE(2, f.dev);
      NFC_TRACE(3, f.avg);
      SMP(NFCB200_OFF_D, 0) = f.dev;
      SMP(NFCB200_OFF_M, 0) = f.env;

      edge_track(w); // :77-92
   }

   // the carrier-edge tracker of nextSample (NfcTech.cpp:77-92) on the edge value of the current step
   NFC_HD void edge_track(float w)
   {
      Front &f = F;
      float rect = fabsf(w);

      if (f.k <= f.edgeHold)
         return;

      if (rect > P.highThr)
      {
         if (rect > f.edgePeak)
         {
            f.edgePeak = rect;
            f.edgeTime = f.clk;
            L.edgeWritten = 1;
         }
      }
      else if (rect < P.lowThr)
      {
         f.edgePeak = 0;
      }
   }

   // feature mode: x / w / dev / envelope of this step already sit in the sample rings (slot of delay 0)
   NFC_HD void front_feat()
   {
      Front &f = F;
      curX = SMP(NFCB200_OFF_X, 0);
      curW = SMP(NFCB200_OFF_W, 0);
      f.env = SMP(NFCB200_OFF_M, 0);
      f.avg = featAvg;
      NFC_TRACE(0, curX);
      NFC_TRACE(1, curW);
      NFC_TRACE(2, (float) SMP(NFCB200_OFF_D, 0));
      NFC_TRACE(3, f.avg);
      edge_track(curW);
   }

   // the detectors' running sums and correlation rings of one search-mode sample without any detector logic: what every
   // detectModulation does on a sample on which nothing can trigger (NfcA.cpp:246-250, NfcF.cpp:240-244, NfcV.cpp:258-270)
   NFC_HD void sums_only()
   {
      if (P.enabled & EN_A)
         for (int r = 0; r < 3; r++)
         {
            const RateParams &b = P.A[r];
            Mod &m = L.c.mA[r];
            FI(m) += SMP(NFCB200_OFF_X, b.sdd);
            FI(m) -= SMP(NFCB200_OFF_X, b.sdd + b.p2);
            put_corr(r, b.corr, F.cA[r], FI(m));
         }
      if (P.enabled & EN_F)
         for (int r = 1; r <= 2; r++)
         {
            const RateParams &b = P.F[r];
            Mod &m = L.c.mF[r - 1];
            FI(m) += SMP(NFCB200_OFF_X, b.sdd);
            FI(m) -= SMP(NFCB200_OFF_X, b.sdd + b.p2);
            put_corr(3 + r - 1, b.corr, F.cF[r - 1], FI(m));
         }
      if (P.enabled & EN_V)
      {
         const RateParams &b = P.V;
         Mod &m = L.c.mV;
         FI(m) += SMP(NFCB200_OFF_X, b.sdd);
         FI(m) -= SMP(NFCB200_OFF_X, b.sdd + b.p2);
         RG(b.corr, F.cV1) = FI(m);
      }
   }

   // sample[..].modulateDepth of `delay` samples ago: (env - clamp(x, 0, env)) / env, NfcTech.cpp:74
   NFC_HD float depth_at(u32 delay)
   {
      float x = SMP(NFCB200_OFF_X, delay);
      float env = SMP(NFCB200_OFF_M, delay);
      float clamped = x < 0.0f ? 0.0f : (env < x ? env : x);
      return (env - clamped) / env;
   }

   // NfcDecoder::Impl::detectCarrier, NfcDecoder.cpp:472-523
   NFC_HD void detect_carrier()
   {
      Front &f = F;

      if (f.avg > P.highThr)
      {
         if (!L.c.carrierOn)
         {
            if (!L.edgeWritten)
               L.edgeLive = 1;
            L.edgeWritten = 1;
            L.c.carrierOn = f.edgeTime ? f.edgeTime : f.clk;
            emit(TT_Any, FT_CarrierOn, 0, PH_Carrier, 0, L.c.carrierOn, L.c.carrierOn, sb, 0);
            L.c.carrierOff = 0;
            f.edgeTime = 0;
         }
      }
      else if (f.avg < P.lowThr)
      {
         if (!L.c.carrierOff)
         {
            if (!L.edgeWritten)
               L.edgeLive = 1;
            L.edgeWritten = 1;
            L.c.carrierOff = f.edgeTime ? f.edgeTime : f.clk;
            emit(TT_Any, FT_CarrierOff, 0, PH_Carrier, 0, L.c.carrierOff, L.c.carrierOff, sb, 0);
            L.c.carrierOn = 0;
            f.edgeTime = 0;
         }
      }
   }

   // S0 / S1 of the half-symbol correlator over a ring of period p1 (NfcA.cpp:241-255): C is written at slot c
   NFC_HD void corr_points(u32 c, u32 p1, u32 p2, u32 &fp2, u32 &fp3) const
   {
      fp2 = c + p2;
      if (fp2 >= p1)
         fp2 -= p1; // (signalIndex + p2) % p1, valid because p2 < p1
      fp3 = c ? c - 1 : p1 - 1; // (signalIndex + p1 - 1) % p1
   }

   // ------------------------------------------------------------------------------------------------------------------
   // NFC-A
   // ------------------------------------------------------------------------------------------------------------------

   // NfcA::Impl::resetModulation, NfcA.cpp:1451-1475
   NFC_HD void A_reset()
   {
      for (int r = 0; r < 3; r++)
      {
         zero_mod(L.c.mA[r]);
         zero_ring(P.A[r].corr, P.A[r].p1);
      }
      // integrationData of all rates: one shared ring, all-zero whenever a listen phase starts (see DESIGN.md)
      zero_ring(NFCB200_OFF_I, NFCB200_RING);
      clear_bits();
      clear_sym();
      L.c.t[TECH_A].fs.frameType = 0;
      L.c.t[TECH_A].fs.frameStart = 0;
      L.c.t[TECH_A].fs.frameEnd = 0;
      F.lock = LOCK_NONE;
   }

   // NfcA::Impl::detectModulation, NfcA.cpp:217-411 (the clock / envelope gates are applied by the caller)
   NFC_HD bool A_detect()
   {
      const float env = F.env;
      const u32 clk = F.clk;
      const float minimumCorrelationValue = env * P.thr[TECH_A].corr;
      const float minDeep = P.thr[TECH_A].modMin;

      for (int rate = 0; rate < 3; rate++)
      {
         const RateParams &b = P.A[rate];
         Mod &m = L.c.mA[rate];

         u32 fp1 = F.cA[rate], fp2, fp3;
         corr_points(fp1, b.p1, b.p2, fp2, fp3);

         // :246-250
         const bool hoisted = staged_for(KIND_SEARCH);
         FI(m) += (hoisted && b.sdd == 0) ? curX : tap(hoisted, TAP_XA0 + rate, SMP(NFCB200_OFF_X, b.sdd));
         FI(m) -= tap(hoisted, TAP_XA1 + rate, SMP(NFCB200_OFF_X, b.sdd + b.p2));
         put_corr(rate, b.corr, fp1, FI(m));

         // :253-255
         const float c2 = tap(hoisted, TAP_CA2 + rate, RG(b.corr, fp2));
         const float c3 = fwd_tap(hoisted, rate, RG(b.corr, fp3));
         float s0 = FI(m) - c2;
         float s1 = c2 - c3;

         NFC_TRACE(4, FI(m) / (float) b.p2); // NfcA.cpp:259-261 (the highest rate writes last)
         NFC_TRACE(5, (s0 - s1) / (float) b.p2);

         // idle fast path (not in the reference): with no search state pending, the rest of this iteration only acts when
         // correlatedSD < -minimumCorrelationValue (:291).  (s0 - s1) / p2 < -T needs s0 - s1 < -T p2 (1 - ulp): anything
         // above half of that cannot trigger, so the IEEE division and the state tests are skipped
         if (!(F.busy & (1u << rate)) && (s0 - s1) > -0.5f * minimumCorrelationValue * (float) b.p2)
            continue;

         slow = true;

         float sd = (s0 - s1) / (float) b.p2;

         // :268-279 recover status from previous partial search
         if (m.correlatedPeakTime && clk > m.correlatedPeakTime + b.p1)
         {
            m.symbolStartTime = 0;
            m.symbolEndTime = 0;
            m.searchStartTime = 0;
            m.searchEndTime = 0;
            m.searchSyncTime = 0;
            m.detectorPeakTime = 0;
            m.detectorPeakValue = 0;
            m.correlatedPeakTime = 0;
            m.correlatedPeakValue = 0;
         }

         if (clk < m.searchStartTime) // :282
            continue;

         if (!m.symbolStartTime) // :285-306
         {
            float deep = depth_at(b.sdd + b.p8);

            if (sd < -minimumCorrelationValue)
            {
               if (sd < m.correlatedPeakValue)
               {
                  m.correlatedPeakValue = sd;
                  m.correlatedPeakTime = clk;
                  m.searchEndTime = clk + b.p4;
               }

               if (deep > m.detectorPeakValue)
               {
                  m.detectorPeakValue = deep;
                  m.detectorPeakTime = clk;
               }
            }
         }
         else // :307-318
         {
            if (sd > minimumCorrelationValue)
            {
               if (sd > m.correlatedPeakValue)
               {
                  m.correlatedPeakValue = sd;
                  m.correlatedPeakTime = clk;
               }
            }
         }

         if (clk != m.searchEndTime) // :321
            continue;

         if (!m.symbolStartTime) // :324-350
         {
            if (m.detectorPeakValue < minDeep)
            {
               m.symbolStartTime = 0;
               m.symbolEndTime = 0;
               m.searchSyncTime = 0;
               m.searchStartTime = 0;
               m.searchEndTime = 0;
               m.searchPulseWidth = 0;
               m.correlatedPeakTime = 0;
               m.correlatedPeakValue = 0;
               m.detectorPeakTime = 0;
               m.detectorPeakValue = 0;
               continue;
            }

            m.searchSyncTime = m.correlatedPeakTime + b.p2;
            m.searchStartTime = m.searchSyncTime - b.p8;
            m.searchEndTime = m.searchSyncTime + b.p8;
            m.symbolStartTime = m.correlatedPeakTime - b.p2;
            m.correlatedPeakTime = 0;
            m.correlatedPeakValue = 0;
            continue;
         }

         // :353-378
         m.symbolEndTime = m.correlatedPeakTime;
         m.searchPulseWidth = m.symbolEndTime - m.symbolStartTime;

         u32 minimumPulseWidth = b.p1 - b.p4; // compared unsigned in the reference (unsigned < int)
         u32 maximumPulseWidth = b.p1 + b.p4;

         if (m.correlatedPeakTime == 0 || m.detectorPeakValue < minDeep || m.searchPulseWidth < minimumPulseWidth || m.searchPulseWidth > maximumPulseWidth)
         {
            m.symbolStartTime = 0;
            m.symbolEndTime = 0;
            m.searchSyncTime = 0;
            m.searchStartTime = 0;
            m.searchEndTime = 0;
            m.searchPulseWidth = 0;
            m.correlatedPeakTime = 0;
            m.correlatedPeakValue = 0;
            m.detectorPeakTime = 0;
            m.detectorPeakValue = 0;
            continue;
         }

         // :381-407 lock
         m.searchSyncTime = m.symbolEndTime + b.p1;
         m.searchStartTime = m.searchSyncTime - b.p8;
         m.searchEndTime = m.searchSyncTime + b.p8;
         m.searchValueThreshold = m.correlatedPeakValue / 2;
         m.searchCorr0Value = 0;
         m.searchCorr1Value = 0;
         m.correlatedPeakTime = 0;
         m.correlatedPeakValue = 0;

         FrameSt &fs = L.c.t[TECH_A].fs;
         fs.frameType = FT_Poll;
         fs.symbolRate = b.sps;
         fs.frameStart = m.symbolStartTime - b.sdd;
         fs.frameEnd = 0;

         L.sym.value = 0;
         L.sym.start = m.symbolStartTime - b.sdd;
         L.sym.end = m.symbolEndTime - b.sdd;
         L.sym.length = L.sym.end - L.sym.start;
         L.sym.pattern = 4; // PatternZ

         F.lock = LOCK_A;
         F.lockRate = rate;
         return true;
      }

      return false;
   }

   enum { A_Invalid = 0, A_No = 1, A_X = 2, A_Y = 3, A_Z = 4, A_D = 5, A_E = 6, A_F = 7, A_M = 8, A_N = 9, A_S = 10, A_O = 11 };

   // NfcA::Impl::checkCrc, NfcA.cpp:1978-1989
   NFC_HD bool A_crc_ok(u32 size) const
   {
      if (size < 2)
         return true;
      if (size > 512)
         return false; // past the 512-byte buffer (the reference's CRC reads beyond its buffer[512]): a CRC error
      unsigned short crc = crc_ccitt16(sb, 0, size - 2, 0x6363, true);
      unsigned short res = (unsigned short) ((sb[size - 2] & 0xff) | ((sb[size - 1] & 0xff) << 8));
      return res == crc;
   }

   // frame byte access: the reference reads RawFrame storage unchecked (Buffer.h:656-668); bytes beyond the frame
   // length are recycled pool memory there, zero here
   NFC_HD u32 fb(u32 i, u32 len) const
   {
      return i < len && i < 512 ? sb[i] : 0;
   }

   NFC_HD void A_default_protocol(Proto &ps)
   {
      ps.maxFrameSize = 256; L.lcWritten |= NFCB200_PSW(TECH_A, 0);
      ps.startUpGuardTime = P.A_sfgt; L.lcWritten |= NFCB200_PSW(TECH_A, 3);
      ps.frameGuardTime = P.A_fgt; L.lcWritten |= NFCB200_PSW(TECH_A, 1);
      ps.frameWaitingTime = P.A_fwt; L.lcWritten |= NFCB200_PSW(TECH_A, 2);
      ps.requestGuardTime = P.A_rgt; L.lcWritten |= NFCB200_PSW(TECH_A, 4);
   }

   // NfcA::Impl::process and the processXXX chain, NfcA.cpp:1480-1973
   NFC_HD void A_process(u32 type, u32 len, u32 &flags, u32 &phase)
   {
      if (type != FT_Poll && !((L.lcWritten >> TECH_A) & 1))
         L.lcLive |= 1u << TECH_A; // a listen frame classified with the lastCommand this lane started from

      TechSt &t = L.c.t[TECH_A];
      FrameSt &fs = t.fs;
      Proto &ps = t.ps;
      const bool poll = type == FT_Poll;
      const u32 b0 = fb(0, len);

      if (poll)
      {
         fs.startUpGuardTime = ps.startUpGuardTime;
         fs.frameWaitingTime = ps.frameWaitingTime;
         fs.frameGuardTime = ps.frameGuardTime;
         fs.requestGuardTime = ps.requestGuardTime;
      }
      else
      {
         fs.frameGuardTime = ps.frameGuardTime;
      }

      bool done = false;

      // processREQA :1592-1631
      if (poll)
      {
         if ((b0 == 0x26 || b0 == 0x52) && len == 1)
         {
            phase = PH_Selection;
            fs.lastCommand = b0;
            L.lcWritten |= 1u << TECH_A;
            A_default_protocol(ps);
            fs.frameGuardTime = P.A_fgt;
            fs.frameWaitingTime = P.A_fwtAtqa;
            t.chained = 0;
            done = true;
         }
      }
      else if (fs.lastCommand == 0x26 || fs.lastCommand == 0x52)
      {
         phase = PH_Selection;
         done = true;
      }

      // processHLTA :1636-1665
      if (!done && poll && b0 == 0x50 && len == 4 && !(flags & FL_Crc))
      {
         phase = PH_Selection;
         flags |= !A_crc_ok(len) ? FL_Crc : 0;
         fs.lastCommand = b0;
            L.lcWritten |= 1u << TECH_A;
         A_default_protocol(ps);
         t.chained = 0;
         A_reset();
         done = true;
      }

      if (!done)
      {
         if (!(t.chained & FL_Encrypted))
         {
            do
            {
               // processSELn :1670-1699
               if (poll)
               {
                  if (b0 == 0x93 || b0 == 0x95 || b0 == 0x97)
                  {
                     phase = PH_Selection;
                     fs.lastCommand = b0;
            L.lcWritten |= 1u << TECH_A;
                     fs.frameGuardTime = P.A_fgt;
                     fs.frameWaitingTime = P.A_fwtAtqa;
                     break;
                  }
               }
               else if (fs.lastCommand == 0x93 || fs.lastCommand == 0x95 || fs.lastCommand == 0x97)
               {
                  phase = PH_Selection;
                  break;
               }

               // processRATS :1704-1790
               if (poll)
               {
                  if (b0 == 0xE0)
                  {
                     int fsdi = (fb(1, len) >> 4) & 0x0F;
                     fs.lastCommand = b0;
            L.lcWritten |= 1u << TECH_A;
                     ps.maxFrameSize = (u32) nfc_fds_table((int) fsdi); L.lcWritten |= NFCB200_PSW(TECH_A, 0);
                     fs.frameWaitingTime = P.fwtActivation;
                     phase = PH_Selection;
                     flags |= !A_crc_ok(len) ? FL_Crc : 0;
                     break;
                  }
               }
               else if (fs.lastCommand == 0xE0)
               {
                  u32 offset = 0;
                  u32 tl = fb(offset++, len);

                  if (tl > 0)
                  {
                     u32 t0 = fb(offset++, len);

                     if (t0 & 0x10)
                        offset++;

                     if (t0 & 0x20)
                     {
                        u32 tb = fb(offset++, len);
                        u32 sfgi = tb & 0x0f;
                        u32 fwi = (tb >> 4) & 0x0f;
                        if (sfgi == 15)
                           sfgi = 0;
                        if (fwi == 15)
                           fwi = 4;
                        ps.startUpGuardTime = (u32) (int) (P.stu * nfc_xgt_table((int) sfgi)); L.lcWritten |= NFCB200_PSW(TECH_A, 3);
                        ps.frameWaitingTime = (u32) (int) (P.stu * nfc_xgt_table((int) fwi)); L.lcWritten |= NFCB200_PSW(TECH_A, 2);
                     }
                     else
                     {
                        ps.startUpGuardTime = P.A_sfgt; L.lcWritten |= NFCB200_PSW(TECH_A, 3);
                        ps.frameWaitingTime = P.A_fwt; L.lcWritten |= NFCB200_PSW(TECH_A, 2);
                     }
                  }

                  phase = PH_Selection;
                  flags |= !A_crc_ok(len) ? FL_Crc : 0;
                  break;
               }

               // processPPSr :1795-1822
               if (poll)
               {
                  if ((b0 & 0xF0) == 0xD0)
                  {
                     fs.lastCommand = b0 & 0xF0;
            L.lcWritten |= 1u << TECH_A;
                     phase = PH_Selection;
                     flags |= !A_crc_ok(len) ? FL_Crc : 0;
                     break;
                  }
               }
               else if (fs.lastCommand == 0xD0)
               {
                  phase = PH_Selection;
                  flags |= !A_crc_ok(len) ? FL_Crc : 0;
                  break;
               }

               // processAUTH :1827-1868
               if (poll)
               {
                  if (b0 == 0x60 || b0 == 0x61)
                  {
                     fs.lastCommand = b0;
            L.lcWritten |= 1u << TECH_A;
                     phase = PH_Application;
                     flags |= !A_crc_ok(len) ? FL_Crc : 0;
                     break;
                  }
               }
               else if (fs.lastCommand == 0x60 || fs.lastCommand == 0x61)
               {
                  t.chained = FL_Encrypted;
                  phase = PH_Application;
                  break;
               }

               // processIBlock :1873-1900
               if (poll)
               {
                  if ((b0 & 0xE2) == 0x02 && len > 4)
                  {
                     fs.lastCommand = b0 & 0xE2;
            L.lcWritten |= 1u << TECH_A;
                     phase = PH_Application;
                     flags |= !A_crc_ok(len) ? FL_Crc : 0;
                     break;
                  }
               }
               else if (fs.lastCommand == 0x02)
               {
                  phase = PH_Application;
                  flags |= !A_crc_ok(len) ? FL_Crc : 0;
                  break;
               }

               // processRBlock :1905-1932
               if (poll)
               {
                  if ((b0 & 0xE6) == 0xA2 && len == 3)
                  {
                     fs.lastCommand = b0 & 0xE6;
            L.lcWritten |= 1u << TECH_A;
                     phase = PH_Application;
                     flags |= !A_crc_ok(len) ? FL_Crc : 0;
                     break;
                  }
               }
               else if (fs.lastCommand == 0xA2)
               {
                  phase = PH_Application;
                  flags |= !A_crc_ok(len) ? FL_Crc : 0;
                  break;
               }

               // processSBlock :1937-1964
               if (poll)
               {
                  if ((b0 & 0xC7) == 0xC0 && len == 4)
                  {
                     fs.lastCommand = b0 & 0xC7;
            L.lcWritten |= 1u << TECH_A;
                     phase = PH_Application;
                     flags |= !A_crc_ok(len) ? FL_Crc : 0;
                     break;
                  }
               }
               else if (fs.lastCommand == 0xC0)
               {
                  phase = PH_Application;
                  flags |= !A_crc_ok(len) ? FL_Crc : 0;
                  break;
               }

               // processOther :1969-1973
               phase = PH_Application;
               flags |= !A_crc_ok(len) ? FL_Crc : 0;
            }
            while (false);
         }
         else
         {
            flags &= ~(u32) FL_Parity; // :1536
            phase = PH_Application;
         }
      }

      flags |= t.chained; // :1545

      if (poll) // :1548-1577
      {
         if (F.lock == LOCK_A)
         {
            u32 sdd = P.A[F.lockRate].sdd;
            fs.guardEnd = fs.frameEnd + fs.frameGuardTime + sdd;
            fs.waitingEnd = fs.frameEnd + fs.frameWaitingTime + sdd;
            fs.frameType = FT_Listen;
         }
      }
      else
      {
         if (F.lock == LOCK_A)
            fs.guardEnd = fs.frameEnd + fs.frameGuardTime + P.A[F.lockRate].sdd;
         fs.frameType = 0;
         fs.lastCommand = 0;
         L.lcWritten |= 1u << TECH_A;
      }

      fs.frameStart = 0;
      fs.frameEnd = 0;
   }

   // one sample of decodePollFrameSymbolAsk, NfcA.cpp:812-934.  Returns a pattern or A_Invalid (no symbol yet).
   NFC_HD int A_poll_symbol()
   {
      const RateParams &b = P.A[F.lockRate];
      Mod &m = L.c.mA[F.lockRate];
      const u32 clk = F.clk;

      u32 fp1 = F.cA[F.lockRate], fp2, fp3;
      corr_points(fp1, b.p1, b.p2, fp2, fp3);

      const u32 rate = F.lockRate;
      const bool hoisted = staged_for(KIND_POLL + rate);
      FI(m) += (hoisted && b.sdd == 0) ? curX : tap(hoisted, TAP_XA0 + rate, SMP(NFCB200_OFF_X, b.sdd));
      FI(m) -= tap(hoisted, TAP_XA1 + rate, SMP(NFCB200_OFF_X, b.sdd + b.p2));
      put_corr(rate, b.corr, fp1, FI(m));

      const float c2 = tap(hoisted, TAP_CA2 + rate, RG(b.corr, fp2));
      const float c3 = fwd_tap(hoisted, rate, RG(b.corr, fp3));
      float s0 = FI(m) - c2;
      float s1 = c2 - c3;

      NFC_TRACE(4, FI(m) / (float) b.p2); // NfcA.cpp:845-846
      NFC_TRACE(5, s0 / (float) b.p4);

      if (clk < m.searchStartTime) // the quotient below is only read past this point
         return A_Invalid;

      float sd = fabsf(s0 - s1) / (float) b.p2;

      if (sd > m.correlatedPeakValue && sd > m.searchValueThreshold) // :858
      {
         m.correlatedPeakValue = sd;
         m.correlatedPeakTime = clk;
      }

      if (clk == m.searchSyncTime) // :865
      {
         m.searchCorrDValue = sd;
         m.searchCorr0Value = s0;
         m.searchCorr1Value = s1;
      }

      if (clk != m.searchEndTime)
         return A_Invalid;

      return A_poll_symbol_tail();
   }

   // end of the search window of decodePollFrameSymbolAsk (NfcA.cpp:875-932): classify the symbol, open the next window
   NFC_HD int A_poll_symbol_tail()
   {
      const RateParams &b = P.A[F.lockRate];
      Mod &m = L.c.mA[F.lockRate];

      if (m.searchCorrDValue < m.searchValueThreshold) // :877 Pattern-Y
      {
         m.symbolStartTime = m.symbolEndTime;
         m.symbolEndTime = m.searchSyncTime;
         m.symbolRiseTime = m.symbolStartTime;
         L.sym.value = 1;
         L.sym.pattern = A_Y;
      }
      else if (m.searchCorr0Value > m.searchCorr1Value) // :890 Pattern-Z
      {
         m.symbolStartTime = m.symbolEndTime;
         m.symbolEndTime = m.correlatedPeakTime;
         m.symbolRiseTime = m.correlatedPeakTime - b.p2;
         L.sym.value = 0;
         L.sym.pattern = A_Z;
      }
      else // Pattern-X
      {
         m.symbolStartTime = m.symbolEndTime;
         m.symbolEndTime = m.correlatedPeakTime;
         m.symbolRiseTime = m.correlatedPeakTime;
         L.sym.value = 1;
         L.sym.pattern = A_X;
      }

      m.searchSyncTime = m.symbolEndTime + b.p1; // :916-923
      m.searchStartTime = m.searchSyncTime - b.p8;
      m.searchEndTime = m.searchSyncTime + b.p8;
      m.searchCorrDValue = 0;
      m.searchCorr0Value = 0;
      m.searchCorr1Value = 0;
      m.correlatedPeakTime = 0;
      m.correlatedPeakValue = 0;

      L.sym.start = m.symbolStartTime - b.sdd;
      L.sym.end = m.symbolEndTime - b.sdd;
      L.sym.edge = m.symbolRiseTime - b.sdd;
      L.sym.length = L.sym.end - L.sym.start;

      return (int) L.sym.pattern;
   }

   // one sample of decodePollFrame, NfcA.cpp:432-563
   NFC_HD void A_poll_step()
   {
      int pattern = A_poll_symbol();

      if (pattern <= A_No)
         return;

      A_poll_after(pattern);
   }

   // decodePollFrame once a symbol is complete (NfcA.cpp:438-560)
   NFC_HD void A_poll_after(int pattern)
   {
      TechSt &t = L.c.t[TECH_A];
      Bits &st = L.st;
      bool frameEnd = false, truncateError = false;

      st.pattern = (u32) pattern;

      if (st.pattern == A_Y && (st.previous == A_Y || st.previous == A_Z))
         frameEnd = true;
      else if (st.bytes == t.ps.maxFrameSize)
         truncateError = true;

      if (frameEnd || truncateError)
      {
         if (st.bytes > 0 || st.bits == 7)
         {
            if (st.bits >= 7)
               put_byte(st.data);

            u32 flags = 0, phase = 0;

            if (st.flags & FL_Parity)
               flags |= FL_Parity;
            if (truncateError)
               flags |= FL_Truncated;
            if (st.bytes == 1 && st.bits == 7)
               flags |= FL_Short;

            u32 len = st.bytes, rate = t.fs.symbolRate, start = t.fs.frameStart, end = t.fs.frameEnd;

            A_process(FT_Poll, len, flags, phase);

            emit(TT_A, FT_Poll, flags, phase, rate, start, end, sb, len);

            clear_bits();

            if (F.lock == LOCK_A) // :491-511
               clear_for_listen(L.c.mA[F.lockRate], P.A[F.lockRate].corr, P.A[F.lockRate].p1);

            return;
         }

         A_reset();
         return;
      }

      if (L.sym.edge) // :525
         t.fs.frameEnd = L.sym.edge;

      if (st.previous)
      {
         u32 value = (st.previous == A_X);

         if (st.bits < 8)
         {
            st.data = st.data | (value << st.bits++);
         }
         else if (st.bytes < t.ps.maxFrameSize)
         {
            put_byte(st.data);
            st.flags |= !odd_parity_ok(st.data, value) ? FL_Parity : 0;
            st.data = st.bits = 0;
         }
         else
         {
            A_reset();
            return;
         }
      }

      st.previous = st.pattern;
   }

   // NfcA::Impl::resetFrameSearch, NfcA.cpp:1426-1446
   NFC_HD void A_reset_frame_search()
   {
      if (F.lock == LOCK_A)
      {
         Mod &m = L.c.mA[F.lockRate];
         m.symbolStartTime = 0;
         m.symbolEndTime = 0;
         m.symbolRiseTime = 0;
         m.searchSyncTime = 0;
         m.searchStartTime = 0;
         m.searchEndTime = 0;
         m.searchPulseWidth = 0;
         m.correlatedPeakTime = 0;
         m.correlatedPeakValue = 0;
         m.detectorPeakTime = 0;
         m.detectorPeakValue = 0;
      }
      L.c.t[TECH_A].fs.frameStart = 0;
   }

   // common part of the ASK listen integrator (w^2 * 10 over half a symbol), NfcA.cpp:955-973 / 1110-1130
   NFC_HD void A_listen_ask_integrate(const RateParams &b, Mod &m, float &s0, float &s1)
   {
      u32 fp1 = F.cA[F.lockRate], fp2, fp3;
      corr_points(fp1, b.p1, b.p2, fp2, fp3);

      const u32 rate = F.lockRate;
      const bool hoisted = staged_for(KIND_LISTEN_ASK + rate);
      float data = hoisted ? curW : (float) SMP(NFCB200_OFF_W, b.sdd); // staged only at rate 0, where sdd == 0
      float v = data * data * 10;

      SMP(NFCB200_OFF_I, b.sdd) = v;

      FI(m) += v;
      FI(m) -= tap(hoisted, TAP_XA1 + rate, SMP(NFCB200_OFF_I, b.sdd + b.p2));

      put_corr(rate, b.corr, fp1, FI(m));

      const float c2 = tap(hoisted, TAP_CA2 + rate, RG(b.corr, fp2));
      const float c3 = fwd_tap(hoisted, rate, RG(b.corr, fp3));
      s0 = FI(m) - c2;
      s1 = c2 - c3;
   }

   // one sample of decodeListenFrameStartAsk, NfcA.cpp:939-1090
   NFC_HD int A_listen_start_ask()
   {
      const RateParams &b = P.A[F.lockRate];
      Mod &m = L.c.mA[F.lockRate];
      FrameSt &fs = L.c.t[TECH_A].fs;
      const u32 clk = F.clk;

      float s0, s1;
      A_listen_ask_integrate(b, m, s0, s1);

      float deep = depth_at(0); // futureIndex

      if (clk < fs.guardEnd)
         return A_Invalid;

      if (clk == fs.guardEnd)
         m.searchValueThreshold = SMP(NFCB200_OFF_D, b.sdd) * (float) b.p8;

      if (clk > fs.waitingEnd)
         return A_No;

      if (deep > P.thr[TECH_A].modMin)
         return A_No;

      if (!m.symbolStartTime)
      {
         if (s0 > m.searchValueThreshold && s0 > m.correlatedPeakValue)
         {
            m.correlatedPeakValue = s0;
            m.correlatedPeakTime = clk;
            m.searchEndTime = clk + b.p4;
         }
      }
      else
      {
         if (s0 < -m.searchValueThreshold && s0 < m.correlatedPeakValue)
         {
            m.correlatedPeakValue = s0;
            m.correlatedPeakTime = clk;
         }
      }

      if (clk != m.searchEndTime)
         return A_Invalid;

      if (!m.symbolStartTime) // :1032-1040
      {
         m.searchSyncTime = m.correlatedPeakTime + b.p2;
         m.searchEndTime = m.searchEndTime + b.p2;
         m.symbolStartTime = m.correlatedPeakTime - b.p2;
         m.correlatedPeakTime = 0;
         m.correlatedPeakValue = 0;
         return A_Invalid;
      }

      m.symbolEndTime = m.correlatedPeakTime;
      m.searchPulseWidth = m.symbolEndTime - m.symbolStartTime;

      u32 minimumPulseWidth = b.p1 - b.p8;
      u32 maximumPulseWidth = b.p1 + b.p8;

      if (m.correlatedPeakTime == 0 || m.searchPulseWidth < minimumPulseWidth || m.searchPulseWidth > maximumPulseWidth)
      {
         m.symbolStartTime = 0;
         m.symbolEndTime = 0;
         m.searchSyncTime = 0;
         m.searchStartTime = 0;
         m.searchEndTime = 0;
         m.searchPulseWidth = 0;
         m.correlatedPeakTime = 0;
         m.correlatedPeakValue = 0;
         m.detectorPeakTime = 0;
         m.detectorPeakValue = 0;
         return A_Invalid;
      }

      m.searchSyncTime = m.symbolEndTime + b.p1;
      m.searchStartTime = m.searchSyncTime - b.p8;
      m.searchEndTime = m.searchSyncTime + b.p8;
      m.searchValueThreshold = fabsf(m.correlatedPeakValue * 0.25f);
      m.searchCorr0Value = 0;
      m.searchCorr1Value = 0;
      m.correlatedPeakTime = 0;
      m.correlatedPeakValue = 0;

      L.sym.value = 1;
      L.sym.start = m.symbolStartTime - b.sdd;
      L.sym.end = m.symbolEndTime - b.sdd;
      L.sym.length = L.sym.end - L.sym.start;
      L.sym.pattern = A_D;

      return A_D;
   }

   // one sample of decodeListenFrameSymbolAsk, NfcA.cpp:1095-1214
   NFC_HD int A_listen_symbol_ask()
   {
      const RateParams &b = P.A[F.lockRate];
      Mod &m = L.c.mA[F.lockRate];
      const u32 clk = F.clk;

      float s0, s1;
      A_listen_ask_integrate(b, m, s0, s1);
      float sd = fabsf(s0 - s1);

      if (clk < m.searchStartTime)
         return A_Invalid;

      if (sd > m.correlatedPeakValue)
      {
         m.correlatedPeakValue = sd;
         m.correlatedPeakTime = clk;
      }

      if (clk == m.searchSyncTime)
      {
         m.searchCorrDValue = sd;
         m.searchCorr0Value = s0;
         m.searchCorr1Value = s1;
      }

      if (clk != m.searchEndTime)
         return A_Invalid;

      return A_listen_symbol_ask_tail();
   }

   // end of the search window of decodeListenFrameSymbolAsk (NfcA.cpp:1150-1212)
   NFC_HD int A_listen_symbol_ask_tail()
   {
      const RateParams &b = P.A[F.lockRate];
      Mod &m = L.c.mA[F.lockRate];

      if (m.searchCorrDValue > m.searchValueThreshold)
      {
         m.symbolStartTime = m.symbolEndTime;
         m.symbolEndTime = m.correlatedPeakTime;
         m.searchValueThreshold = m.correlatedPeakValue * 0.25f;

         if (m.searchCorr0Value > m.searchCorr1Value)
         {
            m.symbolRiseTime = m.searchSyncTime;
            L.sym.value = 0;
            L.sym.pattern = A_E;
         }
         else
         {
            m.symbolRiseTime = m.searchSyncTime - b.p2;
            L.sym.value = 1;
            L.sym.pattern = A_D;
         }
      }
      else
      {
         m.symbolStartTime = m.symbolEndTime;
         m.symbolEndTime = m.searchSyncTime;
         m.symbolRiseTime = 0;
         L.sym.pattern = A_F;
      }

      m.searchSyncTime = m.symbolEndTime + b.p1;
      m.searchStartTime = m.searchSyncTime - b.p8;
      m.searchEndTime = m.searchSyncTime + b.p8;
      m.correlatedPeakTime = 0;
      m.correlatedPeakValue = 0;

      L.sym.start = m.symbolStartTime - b.sdd;
      L.sym.end = m.symbolEndTime - b.sdd;
      L.sym.edge = m.symbolRiseTime - b.sdd;
      L.sym.length = L.sym.end - L.sym.start;

      return (int) L.sym.pattern;
   }

   // one sample of decodeListenFrameStartBpsk, NfcA.cpp:1220-1329
   NFC_HD int A_listen_start_bpsk()
   {
      const RateParams &b = P.A[F.lockRate];
      Mod &m = L.c.mA[F.lockRate];
      FrameSt &fs = L.c.t[TECH_A].fs;
      const u32 clk = F.clk;

      float data = SMP(NFCB200_OFF_W, b.sdd);
      float delay1 = SMP(NFCB200_OFF_W, b.sdd + b.p1);
      float deep = depth_at(0);

      float v = data * delay1 * 10;
      SMP(NFCB200_OFF_I, b.sdd) = v;

      if (clk < fs.guardEnd)
         return A_Invalid;

      if (clk == fs.guardEnd)
         m.searchValueThreshold = SMP(NFCB200_OFF_D, b.sdd);

      if (clk > fs.waitingEnd)
         return A_No;

      if (deep > P.thr[TECH_A].modMin)
         return A_No;

      m.phaseIntegrate += v;
      m.phaseIntegrate -= SMP(NFCB200_OFF_I, b.sdd + b.p4);

      if (m.phaseIntegrate > m.searchValueThreshold) // :1277
      {
         if (!m.symbolStartTime)
            m.symbolStartTime = clk;

         m.searchEndTime = clk + b.p2;
      }

      if (!m.symbolEndTime && (m.phaseIntegrate < 0 || clk == m.searchEndTime)) // :1286
      {
         int preambleSyncLength = (int) (clk - m.symbolStartTime);

         if (preambleSyncLength < P.etu * 3 || preambleSyncLength > P.etu * 4)
         {
            m.symbolStartTime = 0;
            m.symbolEndTime = 0;
            m.searchEndTime = 0;
            return A_Invalid;
         }

         m.symbolEndTime = m.searchEndTime + b.p2;
      }

      if (clk != m.searchEndTime)
         return A_Invalid;

      m.searchSyncTime = m.symbolEndTime + b.p2; // :1311-1316
      m.searchLastPhase = m.phaseIntegrate;
      m.searchPhaseThreshold = fabsf(m.phaseIntegrate * 0.25f);
      m.detectorPeakTime = 0;

      L.sym.value = 0;
      L.sym.start = m.symbolStartTime - b.p1 - b.sdd;
      L.sym.end = m.symbolEndTime - b.p1 - b.sdd;
      L.sym.length = L.sym.end - L.sym.start;
      L.sym.pattern = A_S;

      return A_S;
   }

   // shared BPSK symbol step of NFC-A (NfcA.cpp:1334-1421) and NFC-B (NfcB.cpp:954-1040): identical apart from the
   // pattern codes.  Returns 0 none, 1 end-of-frame (PatternO), 2 symbol
   NFC_HD int bpsk_symbol(const RateParams &b, Mod &m, bool &toggled)
   {
      const u32 clk = F.clk;

      float data = SMP(NFCB200_OFF_W, b.sdd);
      float delay1 = SMP(NFCB200_OFF_W, b.sdd + b.p1);

      float v = data * delay1 * 10;
      SMP(NFCB200_OFF_I, b.sdd) = v;

      m.phaseIntegrate += v;
      m.phaseIntegrate -= SMP(NFCB200_OFF_I, b.sdd + b.p4);

      if (!m.detectorPeakTime)
      {
         if ((m.phaseIntegrate > 0 && m.searchLastPhase < 0) || (m.phaseIntegrate < 0 && m.searchLastPhase > 0))
         {
            m.detectorPeakTime = clk;
            m.searchSyncTime = clk + b.p2;
            m.searchLastPhase = m.phaseIntegrate;
         }
      }

      if (clk != m.searchSyncTime)
         return 0;

      if (fabsf(m.phaseIntegrate) < fabsf(m.searchPhaseThreshold))
         return 1;

      m.symbolStartTime = m.symbolEndTime;
      m.symbolEndTime = m.searchSyncTime + b.p2;
      m.searchSyncTime = m.searchSyncTime + b.p1;
      m.searchLastPhase = m.phaseIntegrate;
      m.detectorPeakTime = 0;

      toggled = false;

      if (m.phaseIntegrate < -m.searchPhaseThreshold)
         toggled = true;
      else
         m.searchPhaseThreshold = m.phaseIntegrate * 0.25f;

      return 2;
   }

   NFC_HD void A_emit_listen(u32 flags)
   {
      TechSt &t = L.c.t[TECH_A];
      u32 phase = 0;
      u32 len = L.st.bytes, rate = P.A[F.lockRate].sps, start = t.fs.frameStart, end = t.fs.frameEnd;
      A_process(FT_Listen, len, flags, phase);
      emit(TT_A, FT_Listen, flags, phase, rate, start, end, sb, len);
      A_reset();
   }

   // one sample of decodeListenFrame, NfcA.cpp:568-807
   NFC_HD void A_listen_step()
   {
      FrameSt &fs = L.c.t[TECH_A].fs;

      if (F.lockRate == 0) // 106k ASK / Manchester
      {
         if (!fs.frameStart)
         {
            int pattern = A_listen_start_ask();

            if (pattern == A_D)
               fs.frameStart = L.sym.start;
            else if (pattern == A_No)
               A_reset();

            return;
         }

         int pattern = A_listen_symbol_ask();

         if (pattern <= A_No)
            return;

         A_listen_ask_after(pattern);
         return;
      }

      A_listen_step_bpsk();
   }

   // decodeListenFrame (106 kbps) once a symbol is complete, NfcA.cpp:598-690
   NFC_HD void A_listen_ask_after(int pattern)
   {
      TechSt &t = L.c.t[TECH_A];
      FrameSt &fs = t.fs;
      Bits &st = L.st;
      bool frameEnd = false, truncateError = false;

      {
         if (pattern == A_F)
            frameEnd = true;
         else if (st.bytes == t.ps.maxFrameSize)
            truncateError = true;

         if (frameEnd || truncateError)
         {
            if (st.bytes > 0 || st.bits == 4)
            {
               if (st.bits == 4)
                  put_byte(st.data);

               u32 flags = 0;
               if (st.flags & FL_Parity)
                  flags |= FL_Parity;
               if (truncateError)
                  flags |= FL_Truncated;
               if (st.bytes == 1 && st.bits == 4)
                  flags |= FL_Short;

               A_emit_listen(flags);
               return;
            }

            A_reset_frame_search(); // :653
            return;
         }

         if (L.sym.edge)
            fs.frameEnd = L.sym.edge;

         if (st.bits < 8)
         {
            st.data |= (L.sym.value << st.bits++);
         }
         else if (st.bytes < t.ps.maxFrameSize)
         {
            put_byte(st.data);
            st.flags |= !odd_parity_ok(st.data, L.sym.value) ? FL_Parity : 0;
            st.data = st.bits = 0;
         }
         else
         {
            A_reset();
         }

         return;
      }
   }

   // 212k / 424k BPSK listen frames, NfcA.cpp:693-807
   NFC_HD void A_listen_step_bpsk()
   {
      TechSt &t = L.c.t[TECH_A];
      FrameSt &fs = t.fs;
      Bits &st = L.st;
      bool frameEnd = false, truncateError = false;

      if (!fs.frameStart)
      {
         int pattern = A_listen_start_bpsk();

         if (pattern == A_S)
            fs.frameStart = L.sym.start;
         else if (pattern == A_No)
            A_reset();

         return;
      }

      const RateParams &b = P.A[F.lockRate];
      Mod &m = L.c.mA[F.lockRate];
      bool toggled = false;
      int r = bpsk_symbol(b, m, toggled);

      if (r == 0)
         return;

      int pattern;

      if (r == 1)
      {
         pattern = A_O;
      }
      else
      {
         if (toggled)
         {
            L.sym.value = !L.sym.value;
            L.sym.pattern = (L.sym.pattern == A_M) ? A_N : A_M;
         }

         L.sym.start = m.symbolStartTime - b.p1 - b.sdd;
         L.sym.end = m.symbolEndTime - b.p1 - b.sdd;
         L.sym.length = L.sym.end - L.sym.start;
         pattern = (int) L.sym.pattern;

         if (pattern <= A_No) // `while ((pattern = ...) > NoPattern)`
            return;
      }

      if (pattern == A_O)
         frameEnd = true;
      else if (st.bytes == t.ps.maxFrameSize)
         truncateError = true;

      if (frameEnd || truncateError)
      {
         if (st.bits == 9)
         {
            put_byte(st.data);
            st.flags |= odd_parity_ok(st.data, st.parity) ? FL_Parity : 0; // last byte: inverted parity, :734
         }

         if (st.bytes > 0)
         {
            fs.frameEnd = L.sym.end;

            u32 flags = 0;
            if (st.flags & FL_Parity)
               flags |= FL_Parity;
            if (truncateError)
               flags |= FL_Truncated;

            A_emit_listen(flags);
            return;
         }

         A_reset();
         return;
      }

      if (st.bits < 8)
      {
         st.data |= (L.sym.value << st.bits);
      }
      else if (st.bits < 9)
      {
         st.parity = L.sym.value;
      }
      else
      {
         put_byte(st.data);
         st.flags |= !odd_parity_ok(st.data, st.parity) ? FL_Parity : 0;
         st.data = L.sym.value;
         st.bits = 0;
      }

      st.bits++;
   }

   // ------------------------------------------------------------------------------------------------------------------
   // NFC-B
   // ------------------------------------------------------------------------------------------------------------------
   enum { B_Invalid = 0, B_No = 1, B_L = 2, B_H = 3, B_S = 4, B_M = 5, B_N = 6, B_O = 7 };

   // NfcB::Impl::resetModulation, NfcB.cpp:1045-1069
   NFC_HD void B_reset()
   {
      zero_mod(L.c.mB[0]);
      zero_mod(L.c.mB[1]);
      zero_ring(NFCB200_OFF_I, NFCB200_RING);
      clear_bits();
      clear_sym();
      L.c.t[TECH_B].fs.frameType = 0;
      L.c.t[TECH_B].fs.frameStart = 0;
      L.c.t[TECH_B].fs.frameEnd = 0;
      F.lock = LOCK_NONE;
   }

   NFC_HD static void B_clear_search(Mod &m, bool sync)
   {
      m.symbolStartTime = 0;
      m.symbolEndTime = 0;
      m.searchStartTime = 0;
      m.searchEndTime = 0;
      if (sync)
         m.searchSyncTime = 0;
      m.detectorPeakTime = 0;
      m.detectorPeakValue = 0;
   }

   // NfcB::Impl::detectModulation, NfcB.cpp:238-432
   NFC_HD bool B_detect()
   {
      const u32 clk = F.clk;
      const float env = F.env;

      for (int rate = 0; rate <= 1; rate++)
      {
         const RateParams &b = P.B[rate];
         Mod &m = L.c.mB[rate];

         const bool hoisted = staged_for(KIND_SEARCH);
         float edge = (hoisted && b.sdd == 0) ? curW : tap(hoisted, TAP_WB + rate, SMP(NFCB200_OFF_W, b.sdd));

         // idle fast path (not in the reference): with no SOF search pending the iteration only acts on a falling edge
         // below -envelope * minimumModulationDeep (:283); the per-sample rewrite of searchValueThreshold (:280) is dead
         if (!(F.busy & (8u << rate)) && !(edge < -(env * P.thr[TECH_B].modMin)))
            continue;

         slow = true;

         float deep = depth_at(b.sdd);

         // :265-274
         if (deep > P.thr[TECH_B].modMax || (m.detectorPeakTime && clk > m.detectorPeakTime + b.p1))
            B_clear_search(m, true);

         if (!m.symbolStartTime) // :277-305
         {
            m.searchValueThreshold = env * P.thr[TECH_B].modMin;

            if (edge < -m.searchValueThreshold && edge < m.detectorPeakValue)
            {
               m.detectorPeakValue = edge;
               m.detectorPeakTime = clk;
               m.searchEndTime = clk + b.p4;
            }

            if (clk != m.searchEndTime)
               continue;

            m.symbolStartTime = m.detectorPeakTime - b.p8;
            m.searchStartTime = m.symbolStartTime + (10 * b.p1) - b.p2;
            m.searchEndTime = m.symbolStartTime + (11 * b.p1) + b.p2;
            m.searchValueThreshold = fabsf(m.detectorPeakValue * 0.5f);
            m.detectorPeakValue = 0;
            m.detectorPeakTime = 0;
            continue;
         }

         if (!m.symbolEndTime) // :308-361
         {
            if (clk < m.searchStartTime)
            {
               if (edge > m.searchValueThreshold)
               {
                  m.symbolStartTime = 0;
                  m.symbolEndTime = 0;
                  m.searchStartTime = 0;
                  m.searchEndTime = 0;
                  m.detectorPeakTime = 0;
                  m.detectorPeakValue = 0;
               }
               continue;
            }

            if (edge > m.searchValueThreshold && edge > m.detectorPeakValue)
            {
               m.detectorPeakValue = edge;
               m.detectorPeakTime = clk;
               m.searchEndTime = clk + b.p4;
            }

            if (clk != m.searchEndTime)
               continue;

            if (!m.detectorPeakTime)
            {
               m.symbolStartTime = 0;
               m.symbolEndTime = 0;
               m.searchStartTime = 0;
               m.searchEndTime = 0;
               m.detectorPeakValue = 0;
               continue;
            }

            m.symbolEndTime = m.detectorPeakTime;
            m.searchStartTime = m.detectorPeakTime + (2 * b.p1) - b.p2;
            m.searchEndTime = m.detectorPeakTime + (3 * b.p1) + b.p2;
            m.searchValueThreshold = fabsf(m.detectorPeakValue) / 2;
            m.detectorPeakValue = 0;
            m.detectorPeakTime = 0;
            continue;
         }

         if (clk < m.searchStartTime) // :364-377
         {
            if (edge < -m.searchValueThreshold)
            {
               m.symbolStartTime = 0;
               m.symbolEndTime = 0;
               m.searchStartTime = 0;
               m.searchEndTime = 0;
               m.detectorPeakTime = 0;
               m.detectorPeakValue = 0;
            }
            continue;
         }

         if (edge < -m.searchValueThreshold && m.detectorPeakValue > edge) // :380
         {
            m.detectorPeakValue = edge;
            m.detectorPeakTime = clk;
            m.searchEndTime = clk + b.p4;
         }

         if (clk != m.searchEndTime)
            continue;

         if (!m.detectorPeakTime) // :392-402 (note: `break`, the 212k detector is skipped for this sample)
         {
            m.symbolStartTime = 0;
            m.symbolEndTime = 0;
            m.searchStartTime = 0;
            m.searchEndTime = 0;
            m.detectorPeakTime = 0;
            m.detectorPeakValue = 0;
            break;
         }

         m.symbolEndTime = m.detectorPeakTime; // :408-428
         m.searchSyncTime = m.symbolEndTime + b.p2;
         m.searchStartTime = 0;
         m.searchEndTime = 0;
         m.searchValueThreshold = fabsf(m.detectorPeakValue * 0.5f);
         m.detectorPeakTime = 0;
         m.detectorPeakValue = 0;

         FrameSt &fs = L.c.t[TECH_B].fs;
         fs.frameType = FT_Poll;
         fs.symbolRate = b.sps;
         fs.frameStart = m.symbolStartTime - b.sdd;
         fs.frameEnd = 0;

         F.lock = LOCK_B;
         F.lockRate = rate;
         return true;
      }

      return false;
   }

   // NfcB::Impl::checkCrc, NfcB.cpp:1272-1283
   NFC_HD bool B_crc_ok(u32 size) const
   {
      if (size < 3)
         return false;
      if (size > 512)
         return false; // past the 512-byte buffer (the reference's CRC reads beyond its buffer[512]): a CRC error
      unsigned short crc = (unsigned short) ~crc_ccitt16(sb, 0, size - 2, 0xFFFF, true);
      unsigned short res = (unsigned short) ((sb[size - 2] & 0xff) | ((sb[size - 1] & 0xff) << 8));
      return res == crc;
   }

   // NfcB::Impl::process, NfcB.cpp:1074-1267
   NFC_HD void B_process(u32 type, u32 len, u32 &flags, u32 &phase)
   {
      if (type != FT_Poll && !((L.lcWritten >> TECH_B) & 1))
         L.lcLive |= 1u << TECH_B; // a listen frame classified with the lastCommand this lane started from

      TechSt &t = L.c.t[TECH_B];
      FrameSt &fs = t.fs;
      Proto &ps = t.ps;
      const bool poll = type == FT_Poll;
      const u32 b0 = fb(0, len);

      if (poll)
      {
         fs.startUpGuardTime = ps.startUpGuardTime;
         fs.frameWaitingTime = ps.frameWaitingTime;
         fs.frameGuardTime = ps.frameGuardTime;
         fs.requestGuardTime = ps.requestGuardTime;
      }
      else
      {
         fs.frameGuardTime = ps.frameGuardTime;
      }

      do
      {
         // processREQB :1153-1206
         if (poll)
         {
            if (b0 == 0x05 && len == 5)
            {
               fs.lastCommand = b0;
            L.lcWritten |= 1u << TECH_B;
               ps.maxFrameSize = 256; L.lcWritten |= NFCB200_PSW(TECH_B, 0);
               ps.startUpGuardTime = P.B_sfgt; L.lcWritten |= NFCB200_PSW(TECH_B, 3);
               ps.frameGuardTime = P.B_fgt; L.lcWritten |= NFCB200_PSW(TECH_B, 1);
               ps.frameWaitingTime = P.B_fwt; L.lcWritten |= NFCB200_PSW(TECH_B, 2);
               ps.requestGuardTime = P.B_rgt; L.lcWritten |= NFCB200_PSW(TECH_B, 4);
               fs.frameGuardTime = P.B_tr0min;
               fs.frameWaitingTime = P.B_fwtAtqb;
               t.chained = 0;
               phase = PH_Selection;
               flags |= !B_crc_ok(len) ? FL_Crc : 0;
               break;
            }
         }
         else if (fs.lastCommand == 0x05)
         {
            int fdsi = (fb(10, len) >> 4) & 0x0f;
            int fwi = (fb(11, len) >> 4) & 0x0f;
            ps.maxFrameSize = (u32) nfc_fds_table((int) fdsi); L.lcWritten |= NFCB200_PSW(TECH_B, 0);
            ps.frameWaitingTime = (u32) (int) (P.stu * nfc_xgt_table((int) fwi)); L.lcWritten |= NFCB200_PSW(TECH_B, 2);
            phase = PH_Selection;
            flags |= !B_crc_ok(len) ? FL_Crc : 0;
            break;
         }

         // processATTRIB :1212-1258
         if (poll)
         {
            if (b0 == 0x1d && len > 10)
            {
               fs.lastCommand = b0;
            L.lcWritten |= 1u << TECH_B;
               u32 param1 = fb(5, len), param2 = fb(6, len);
               u32 tr0i = (param1 >> 6) & 0x3;
               u32 fdsi = param2 & 0xf;
               ps.maxFrameSize = (u32) nfc_fds_table((int) fdsi); L.lcWritten |= NFCB200_PSW(TECH_B, 0);
               if (!tr0i)
                  ps.frameGuardTime = P.B_fgt;
               else
                  ps.frameGuardTime = (u32) (int) (P.stu * (tr0i == 1 ? 48 * 16 : tr0i == 2 ? 16 * 16 : 0));
               L.lcWritten |= NFCB200_PSW(TECH_B, 1);
               fs.frameWaitingTime = P.fwtActivation;
               t.chained = 0;
               phase = PH_Selection;
               flags |= !B_crc_ok(len) ? FL_Crc : 0;
               break;
            }
         }
         else if (fs.lastCommand == 0x1d)
         {
            phase = PH_Selection;
            break;
         }

         // processOther :1263-1267
         phase = PH_Application;
         flags |= !B_crc_ok(len) ? FL_Crc : 0;
      }
      while (false);

      flags |= t.chained;

      if (poll)
      {
         if (F.lock == LOCK_B)
         {
            u32 sdd = P.B[F.lockRate].sdd;
            fs.guardEnd = fs.frameEnd + fs.frameGuardTime + sdd;
            fs.waitingEnd = fs.frameEnd + fs.frameWaitingTime + sdd;
            fs.frameType = FT_Listen;
         }
      }
      else
      {
         if (F.lock == LOCK_B)
            fs.guardEnd = fs.frameEnd + fs.frameGuardTime + P.B[F.lockRate].sdd;
         fs.frameType = 0;
         fs.lastCommand = 0;
         L.lcWritten |= 1u << TECH_B;
      }

      fs.frameStart = 0;
      fs.frameEnd = 0;
   }

   // one sample of decodePollFrameSymbolAsk, NfcB.cpp:684-762
   NFC_HD int B_poll_symbol()
   {
      const RateParams &b = P.B[F.lockRate];
      Mod &m = L.c.mB[F.lockRate];
      const u32 clk = F.clk;

      float edge = SMP(NFCB200_OFF_W, b.sdd);
      float deep = depth_at(b.sdd);

      if (clk > m.searchStartTime && clk < m.searchEndTime)
      {
         edge = fabsf(edge);

         if (edge > m.searchValueThreshold && m.detectorPeakValue < edge)
         {
            m.detectorPeakValue = edge;
            m.searchSyncTime = clk + b.p2;
         }
      }

      if (clk != m.searchSyncTime)
         return B_Invalid;

      m.symbolStartTime = m.symbolEndTime;
      m.symbolEndTime = m.searchSyncTime + b.p2;
      m.searchStartTime = m.searchSyncTime + b.p4;
      m.searchEndTime = m.searchStartTime + b.p2;
      m.searchSyncTime = m.searchSyncTime + b.p1;
      m.detectorPeakValue = 0;

      if (deep > P.thr[TECH_B].modMin)
      {
         L.sym.value = 0;
         L.sym.pattern = B_L;
      }
      else
      {
         L.sym.value = 1;
         L.sym.pattern = B_H;
      }

      L.sym.start = m.symbolStartTime - b.sdd;
      L.sym.end = m.symbolEndTime - b.sdd;
      L.sym.length = L.sym.end - L.sym.start;

      return (int) L.sym.pattern;
   }

   // one sample of decodePollFrame, NfcB.cpp:453-567
   NFC_HD void B_poll_step()
   {
      int pattern = B_poll_symbol();

      if (pattern <= B_No)
         return;

      TechSt &t = L.c.t[TECH_B];
      Bits &st = L.st;
      bool frameEnd = false, truncateError = false, streamError = false;

      if (st.bits == 9 && !st.data && pattern == B_L)
         frameEnd = true;
      else if (st.bits == 9 && pattern == B_L)
         streamError = true;
      else if (st.bits == 0 && pattern == B_H && st.skip == 6)
         streamError = true;
      else if (st.bytes == t.ps.maxFrameSize)
         truncateError = true;
      else if ((st.bits == 0 && pattern == B_H) && ++st.skip)
         return;

      if (frameEnd || streamError || truncateError)
      {
         if (st.bytes > 2)
         {
            t.fs.frameEnd = L.sym.end;

            u32 flags = 0, phase = 0;
            if (truncateError || streamError)
               flags |= FL_Truncated;

            u32 len = st.bytes, rate = P.B[F.lockRate].sps, start = t.fs.frameStart, end = t.fs.frameEnd;

            B_process(FT_Poll, len, flags, phase);
            emit(TT_B, FT_Poll, flags, phase, rate, start, end, sb, len);

            clear_bits();

            if (F.lock == LOCK_B)
               clear_for_listen(L.c.mB[F.lockRate], 0, 0);

            return;
         }

         B_reset();
         return;
      }

      if (st.bits < 9)
      {
         if (st.bits > 0)
            st.data |= (L.sym.value << (st.bits - 1));
         st.bits++;
      }
      else
      {
         put_byte(st.data);
         st.data = 0;
         st.bits = 0;
         st.skip = 0;
      }
   }

   // one sample of decodeListenFrameStartBpsk, NfcB.cpp:767-949
   NFC_HD int B_listen_start()
   {
      const RateParams &b = P.B[F.lockRate];
      Mod &m = L.c.mB[F.lockRate];
      FrameSt &fs = L.c.t[TECH_B].fs;
      const u32 clk = F.clk;

      float data = SMP(NFCB200_OFF_W, b.sdd);
      float delay1 = SMP(NFCB200_OFF_W, b.sdd + b.p1);
      float deep = depth_at(0);

      float v = data * delay1 * 10;
      SMP(NFCB200_OFF_I, b.sdd) = v;

      m.phaseIntegrate += v; // integrates always (:793-794)
      m.phaseIntegrate -= SMP(NFCB200_OFF_I, b.sdd + b.p4);

      if (clk < fs.guardEnd)
         return B_Invalid;

      if (clk == fs.guardEnd)
         m.searchValueThreshold = SMP(NFCB200_OFF_D, b.sdd);

      if (clk > fs.waitingEnd)
         return B_No;

      if (deep > P.thr[TECH_B].modMax)
         return B_No;

      if (clk < m.searchStartTime)
         return B_Invalid;

      if (m.phaseIntegrate > m.searchValueThreshold)
      {
         if (!m.symbolStartTime)
            m.symbolStartTime = clk;

         m.searchEndTime = clk + b.p2;
      }

      if (clk != m.searchEndTime && m.phaseIntegrate > 0)
         return B_Invalid;

      u32 length, lo, hi;

      switch (m.searchModeState)
      {
         case 0: // LISTEN_MODE_TR1
            length = clk - m.symbolStartTime;
            lo = P.B_tr1Min;
            hi = P.B_tr1Max;
            break;
         case 1: // LISTEN_MODE_SOS_S1
            length = clk - m.symbolEndTime;
            lo = P.B_s1Min;
            hi = P.B_s1Max;
            break;
         case 2: // LISTEN_MODE_SOS_S2
            length = clk - m.symbolEndTime;
            lo = P.B_s2Min;
            hi = P.B_s2Max;
            break;
         default:
            return B_Invalid; // the reference's switch has no default: falls out of the switch, loops
      }

      if (length < lo || length > hi) // int vs unsigned in the reference: compared unsigned
      {
         m.searchModeState = 0;
         m.searchStartTime = 0;
         m.searchEndTime = 0;
         m.symbolStartTime = 0;
         m.symbolEndTime = 0;
         return B_Invalid;
      }

      m.symbolEndTime = clk;

      if (m.searchModeState < 2)
      {
         m.searchModeState++;
         m.searchStartTime = clk + b.p1 + b.p4;
         m.searchEndTime = 0;
         return B_Invalid;
      }

      m.searchSyncTime = clk + b.p2; // :927-943
      m.searchLastPhase = m.phaseIntegrate;
      m.searchPhaseThreshold = fabsf(m.detectorPeakValue * 0.25f);
      m.searchStartTime = 0;
      m.searchEndTime = 0;
      m.detectorPeakValue = 0;

      L.sym.value = 1;
      L.sym.start = m.symbolStartTime - b.p1 - b.sdd;
      L.sym.end = m.symbolEndTime - b.p1 - b.sdd;
      L.sym.length = L.sym.end - L.sym.start;
      L.sym.pattern = B_S;

      return B_S;
   }

   // one sample of decodeListenFrame, NfcB.cpp:572-679
   NFC_HD void B_listen_step()
   {
      TechSt &t = L.c.t[TECH_B];
      FrameSt &fs = t.fs;
      Bits &st = L.st;

      if (!fs.frameStart)
      {
         int pattern = B_listen_start();

         if (pattern == B_S)
            fs.frameStart = L.sym.start;
         else if (pattern == B_No)
            B_reset();

         return;
      }

      const RateParams &b = P.B[F.lockRate];
      Mod &m = L.c.mB[F.lockRate];
      bool toggled = false;
      int r = bpsk_symbol(b, m, toggled);

      if (r == 0)
         return;

      int pattern;

      if (r == 1)
      {
         pattern = B_O;
      }
      else
      {
         if (toggled)
         {
            L.sym.value = !L.sym.value;
            L.sym.pattern = (L.sym.pattern == B_M) ? B_N : B_M;
         }

         L.sym.start = m.symbolStartTime - b.p1 - b.sdd;
         L.sym.end = m.symbolEndTime - b.p1 - b.sdd;
         L.sym.length = L.sym.end - L.sym.start;
         pattern = (int) L.sym.pattern;

         if (pattern <= B_No)
            return;
      }

      bool frameEnd = false, truncateError = false, streamError = false;

      if (st.bits == 9 && !st.data && pattern == B_M)
         frameEnd = true;
      else if ((st.bits == 0 && pattern == B_N) || (st.bits == 9 && pattern == B_M))
         streamError = true;
      else if (st.bytes == t.ps.maxFrameSize)
         truncateError = true;

      if (frameEnd || streamError || truncateError)
      {
         if (st.bytes > 0)
         {
            fs.frameEnd = L.sym.end + P.B_eofComp;

            u32 flags = 0, phase = 0;
            if (truncateError || streamError)
               flags |= FL_Truncated;

            u32 len = st.bytes, rate = b.sps, start = fs.frameStart, end = fs.frameEnd;

            B_process(FT_Listen, len, flags, phase);
            emit(TT_B, FT_Listen, flags, phase, rate, start, end, sb, len);
         }

         B_reset();
         return;
      }

      if (st.bits < 9)
      {
         if (st.bits > 0)
            st.data |= (L.sym.value << (st.bits - 1));
         st.bits++;
      }
      else
      {
         put_byte(st.data);
         st.data = 0;
         st.bits = 0;
      }
   }

   // ------------------------------------------------------------------------------------------------------------------
   // NFC-F
   // ------------------------------------------------------------------------------------------------------------------
   enum { F_Invalid = 0, F_No = 1, F_L = 2, F_H = 3, F_S = 4, F_E = 5 };

   // NfcF::Impl::resetModulation, NfcF.cpp:1047-1071
   NFC_HD void F_reset()
   {
      L.fZeroed |= 3;
      L.fThrWritten |= 0x3F; // threshold, searchLastValue, searchLastPhase of both rates
      for (int r = 0; r < 2; r++)
      {
         zero_mod(L.c.mF[r]);
         zero_ring(P.F[r + 1].corr, P.F[r + 1].p1);
      }
      clear_bits();
      clear_sym();
      L.c.t[TECH_F].fs.frameType = 0;
      L.c.t[TECH_F].fs.frameStart = 0;
      L.c.t[TECH_F].fs.frameEnd = 0;
      F.lock = LOCK_NONE;
   }

   NFC_HD void F_note_zeroed(const Mod &m)
   {
      u32 bit = (&m == &L.c.mF[1]) ? 2u : 1u;
      L.fZeroed |= bit;
      L.fThrWritten |= bit;
   }

   NFC_HD static void F_restart_search(Mod &m)
   {
      m.symbolStartTime = 0;
      m.symbolEndTime = 0;
      m.searchSyncTime = 0;
      m.searchSyncValue = 0;
      m.searchStartTime = 0;
      m.searchEndTime = 0;
      m.searchPulseWidth = 0;
      m.searchValueThreshold = 0;
      m.correlatedPeakValue = 0;
      m.correlatedPeakTime = 0;
   }

   // the preamble tracker shared by detectModulation (NfcF.cpp:273-404) and decodeListenFrameStartAsk (:810-932).
   // `ge` selects the listen variant's `>=` threshold test (:814).  Returns true when the preamble->sync transition
   // was accepted (symbol timings are left in m).
   NFC_HD bool F_track_preamble(const RateParams &b, Mod &m, float s0, float sd, float minimumCorrelationValue, bool ge)
   {
      const u32 clk = F.clk;

      if (clk < m.searchStartTime)
         return false;

      if (ge ? (sd >= minimumCorrelationValue) : (sd > minimumCorrelationValue))
      {
         if (sd > m.correlatedPeakValue)
         {
            m.correlatedPeakValue = sd;
            m.correlatedPeakTime = clk;

            if (!m.searchSyncTime)
            {
               m.searchSyncValue = sd;
               m.searchCorr0Value = s0;
               m.searchEndTime = clk + b.p8;
            }
         }
      }

      if (clk == m.searchSyncTime)
      {
         m.searchSyncValue = sd;
         m.searchLastValue = s0;
         L.fThrWritten |= (&m == &L.c.mF[1]) ? 8u : 4u;
      }

      if (clk != m.searchEndTime)
         return false;

      // dependency bookkeeping (not in the reference): which incoming values did this run actually observe
      const u32 fr = (&m == &L.c.mF[1]) ? 1u : 0u;
      if (!((L.fZeroed >> fr) & 1))
         L.fInc0[fr]++;
      if (!((L.fThrWritten >> fr) & 1) && !((L.fThrRead >> fr) & 1))
      {
         L.fThrRead |= 1u << fr;
         L.fThrSync[fr] = m.searchSyncValue;
      }

      if (m.searchPulseWidth++ < 94)
      {
         if (m.correlatedPeakTime == 0 || m.searchSyncValue < m.searchValueThreshold)
         {
            F_restart_search(m);
            F_note_zeroed(m);
            return false;
         }
      }

      if (m.searchSyncValue > m.searchValueThreshold)
      {
         L.fThrWritten |= 1u << fr;
         if (!m.symbolStartTime)
            m.symbolStartTime = m.correlatedPeakTime - b.p2;

         m.symbolEndTime = m.correlatedPeakTime;
         m.searchSyncTime = m.symbolEndTime + b.p2;
         m.searchStartTime = m.searchSyncTime - b.p8;
         m.searchEndTime = m.searchSyncTime + b.p8;
         m.searchValueThreshold = m.correlatedPeakValue / 2;
         if (!((L.fThrWritten >> (2 + fr)) & 1))
            L.fThrRead |= 4u << fr; // the searchLastValue this run started from is used
         L.fThrWritten |= 16u << fr;
         m.searchLastPhase = m.searchLastValue;
         m.correlatedPeakTime = 0;
         m.correlatedPeakValue = 0;
         return false;
      }

      if (!((L.fThrWritten >> (4 + fr)) & 1))
         L.fThrRead |= 16u << fr; // no threshold pass in this run yet: the searchLastPhase it started from decides

      if ((m.searchLastPhase < 0 && m.searchCorr0Value < 0) || (m.searchLastPhase > 0 && m.searchCorr0Value > 0))
         m.symbolStartTime -= b.p2;

      int preambleLength = (int) (m.symbolEndTime - m.symbolStartTime);
      int preambleMinLength = (int) (b.pre1 - b.p4);
      int preambleMaxLength = (int) (b.pre1 + b.p4);

      if (preambleLength < preambleMinLength || preambleLength > preambleMaxLength)
      {
         F_restart_search(m);
         F_note_zeroed(m);
         return false;
      }

      m.searchModeState = m.searchLastPhase > 0 ? 0 : 1; // OBSERVED : REVERSED
      m.searchSyncTime = m.searchSyncTime + b.p2;
      m.searchStartTime = m.searchSyncTime - b.p4;
      m.searchEndTime = m.searchSyncTime + b.p4;
      m.correlatedPeakTime = 0;
      m.correlatedPeakValue = 0;
      return true;
   }

   NFC_HD void F_correlate(const RateParams &b, Mod &m, u32 fp1, float &s0, float &s1, float &sd)
   {
      u32 fp2, fp3;
      corr_points(fp1, b.p1, b.p2, fp2, fp3);
      put_corr(3 + (u32) (&b - &P.F[1]), b.corr, fp1, FI(m));
      s0 = FI(m) - RG(b.corr, fp2);
      s1 = RG(b.corr, fp2) - RG(b.corr, fp3);
      sd = fabsf(s0 - s1) / (float) b.p2;
   }

   // NfcF::Impl::detectModulation, NfcF.cpp:206-408
   NFC_HD bool F_detect()
   {
      const u32 clk = F.clk;
      const float minimumCorrelationValue = F.env * P.thr[TECH_F].corr;

      for (int rate = 1; rate <= 2; rate++)
      {
         const RateParams &b = P.F[rate];
         Mod &m = L.c.mF[rate - 1];

         const bool hoisted = staged_for(KIND_SEARCH);
         FI(m) += (hoisted && b.sdd == 0) ? curX : SMP(NFCB200_OFF_X, b.sdd);
         FI(m) -= tap(hoisted, TAP_XF1 + rate - 1, SMP(NFCB200_OFF_X, b.sdd + b.p2));

         // idle fast path (not in the reference): with no search window pending (the residual pulse counter / threshold
         // only matter at a window end) the iteration only acts when correlatedSD > minimumCorrelationValue (:277); the
         // "recover" block (:260-271) rewrites zeros.  |s0 - s1| below half of T p2 cannot reach the threshold.
         if (!(F.busy & (16u << rate)))
         {
            u32 fq2, fq3;
            const u32 fq1 = F.cF[rate - 1];
            corr_points(fq1, b.p1, b.p2, fq2, fq3);
            put_corr(3 + rate - 1, b.corr, fq1, FI(m));
            const float c2 = tap(hoisted, TAP_CF2 + rate - 1, RG(b.corr, fq2));
            const float c3 = fwd_tap(hoisted, 3 + rate - 1, RG(b.corr, fq3));
            float q0 = FI(m) - c2;
            float q1 = c2 - c3;
            if (fabsf(q0 - q1) < 0.5f * minimumCorrelationValue * (float) b.p2)
               continue;
         }

         slow = true;

         float deep = depth_at(b.sdd);

         float s0, s1, sd;
         F_correlate(b, m, F.cF[rate - 1], s0, s1, sd);

         // :260-271
         if (deep > P.thr[TECH_F].modMax || (m.correlatedPeakTime && clk > m.correlatedPeakTime + b.p1))
         {
            m.symbolStartTime = 0;
            m.symbolEndTime = 0;
            m.searchStartTime = 0;
            m.searchEndTime = 0;
            m.searchSyncTime = 0;
            m.detectorPeakTime = 0;
            m.detectorPeakValue = 0;
            m.correlatedPeakTime = 0;
            m.correlatedPeakValue = 0;
         }

         if (!F_track_preamble(b, m, s0, sd, minimumCorrelationValue, false))
            continue;

         L.sym.start = m.symbolStartTime; // :390-402
         L.sym.end = m.symbolEndTime;
         L.sym.length = L.sym.end - L.sym.start;
         L.sym.pattern = F_S;

         FrameSt &fs = L.c.t[TECH_F].fs;
         fs.frameType = FT_Poll;
         fs.symbolRate = b.sps;
         fs.frameStart = L.sym.start;
         fs.frameEnd = 0;

         F.lock = LOCK_F;
         F.lockRate = rate;
         return true;
      }

      return false;
   }

   // NfcF::Impl::checkCrc, NfcF.cpp:1215-1226 (payload only: the two sync bytes were stripped)
   NFC_HD bool F_crc_ok(const u8 *d, u32 size) const
   {
      if (size < 2)
         return false;
      unsigned short crc = crc_ccitt16(d, 0, size - 2, 0x0000, false);
      unsigned short res = (unsigned short) (((d[size - 2] & 0xff) << 8) | (d[size - 1] & 0xff));
      return res == crc;
   }

   // NfcF::Impl::process, NfcF.cpp:1076-1210.  d = payload after the sync bytes
   NFC_HD void F_process(u32 type, const u8 *d, u32 len, u32 &flags, u32 &phase)
   {
      if (type != FT_Poll && !((L.lcWritten >> TECH_F) & 1))
         L.lcLive |= 1u << TECH_F; // a listen frame classified with the lastCommand this lane started from

      TechSt &t = L.c.t[TECH_F];
      FrameSt &fs = t.fs;
      Proto &ps = t.ps;
      const bool poll = type == FT_Poll;

      if (poll)
      {
         fs.startUpGuardTime = ps.startUpGuardTime;
         fs.frameWaitingTime = ps.frameWaitingTime;
         fs.frameGuardTime = ps.frameGuardTime;
         fs.requestGuardTime = ps.requestGuardTime;
      }
      else
      {
         fs.frameGuardTime = ps.frameGuardTime;
      }

      bool done = false;

      // processREQC :1152-1201
      if (poll)
      {
         u32 b1 = 1 < len ? d[1] : 0;

         if (b1 == 0x00)
         {
            fs.lastCommand = b1;
            L.lcWritten |= 1u << TECH_F;
            int tsn = (int) (5 < len ? d[5] : 0);
            ps.maxFrameSize = 256; L.lcWritten |= NFCB200_PSW(TECH_F, 0);
            ps.startUpGuardTime = P.F_sfgt; L.lcWritten |= NFCB200_PSW(TECH_F, 3);
            ps.frameGuardTime = P.F_fgt; L.lcWritten |= NFCB200_PSW(TECH_F, 1);
            ps.frameWaitingTime = P.F_fwt; L.lcWritten |= NFCB200_PSW(TECH_F, 2);
            ps.requestGuardTime = P.F_rgt; L.lcWritten |= NFCB200_PSW(TECH_F, 4);
            fs.frameGuardTime = (u32) (P.stu * 1024);
            fs.frameWaitingTime = (u32) (P.stu * (512 * 64 + (tsn + 1) * (256 * 64)));
            t.chained = 0;
            phase = PH_Selection;
            flags |= !F_crc_ok(d, len) ? FL_Crc : 0;
            done = true;
         }
      }
      else if (fs.lastCommand == 0x00)
      {
         phase = PH_Selection;
         flags |= !F_crc_ok(d, len) ? FL_Crc : 0;
         done = true;
      }

      if (!done) // processOther
      {
         phase = PH_Application;
         flags |= !F_crc_ok(d, len) ? FL_Crc : 0;
      }

      flags |= t.chained;

      if (poll)
      {
         if (F.lock == LOCK_F)
         {
            u32 sdd = P.F[F.lockRate].sdd;
            fs.guardEnd = fs.frameEnd + fs.frameGuardTime + sdd;
            fs.waitingEnd = fs.frameEnd + fs.frameWaitingTime + sdd;
            fs.frameType = FT_Listen;
         }
      }
      else
      {
         if (F.lock == LOCK_F)
            fs.guardEnd = fs.frameEnd + fs.frameGuardTime + P.F[F.lockRate].sdd;
         fs.frameType = 0;
         fs.lastCommand = 0;
         L.lcWritten |= 1u << TECH_F;
      }

      fs.frameStart = 0;
      fs.frameEnd = 0;
   }

   // one sample of decodePollFrameSymbolAsk / decodeListenFrameSymbolAsk, NfcF.cpp:641-744, 941-1042 (identical bodies)
   NFC_HD int F_symbol()
   {
      const RateParams &b = P.F[F.lockRate];
      Mod &m = L.c.mF[F.lockRate - 1];
      const u32 clk = F.clk;

      FI(m) += SMP(NFCB200_OFF_X, b.sdd);
      FI(m) -= SMP(NFCB200_OFF_X, b.sdd + b.p2);

      float s0, s1, sd;
      F_correlate(b, m, F.cF[F.lockRate - 1], s0, s1, sd);

      if (clk < m.searchStartTime)
         return F_Invalid;

      if (sd > m.searchValueThreshold && sd > m.correlatedPeakValue)
      {
         m.correlatedPeakValue = sd;
         m.correlatedPeakTime = clk;
      }

      if (clk == m.searchSyncTime)
      {
         m.searchCorr0Value = s0;
         m.searchCorr1Value = s1;
      }

      if (clk != m.searchEndTime)
         return F_Invalid;

      if (!m.correlatedPeakTime)
         return F_E;

      m.symbolStartTime = m.symbolEndTime;
      m.symbolEndTime = m.correlatedPeakTime;
      m.searchSyncTime = m.symbolEndTime + b.p1;
      m.searchStartTime = m.searchSyncTime - b.p4;
      m.searchEndTime = m.searchSyncTime + b.p4;
      m.searchValueThreshold = m.correlatedPeakValue / 2;
      m.correlatedPeakTime = 0;
      m.correlatedPeakValue = 0;

      L.sym.start = m.symbolStartTime - b.sdd;
      L.sym.end = m.symbolEndTime - b.sdd;
      L.sym.length = L.sym.end - L.sym.start;

      if ((m.searchModeState == 0 && m.searchCorr0Value > m.searchCorr1Value) || (m.searchModeState == 1 && m.searchCorr0Value < m.searchCorr1Value))
      {
         L.sym.value = 0;
         L.sym.pattern = F_L;
      }
      else
      {
         L.sym.value = 1;
         L.sym.pattern = F_H;
      }

      return (int) L.sym.pattern;
   }

   // frame assembly shared by decodePollFrame (NfcF.cpp:428-529) and decodeListenFrame (:534-636)
   NFC_HD void F_frame_step(int pattern, u32 type)
   {
      TechSt &t = L.c.t[TECH_F];
      Bits &st = L.st;
      bool frameEnd = false, truncateError = false;

      if (pattern == F_E)
         frameEnd = true;
      else if (st.bytes == t.ps.maxFrameSize)
         truncateError = true;

      if (frameEnd || truncateError)
      {
         if (st.bytes > 2)
         {
            t.fs.frameEnd = L.sym.end;

            u32 flags = 0, phase = 0;
            if (truncateError)
               flags |= FL_Truncated;
            if (sb[0] != 0xB2 || sb[1] != 0x4D)
               flags |= FL_Sync;

            u32 total = st.bytes > 512 ? 512 : st.bytes;
            u32 len = total - 2, rate = P.F[F.lockRate].sps, start = t.fs.frameStart, end = t.fs.frameEnd;

            F_process(type, sb + 2, len, flags, phase);
            emit(TT_F, type, flags, phase, rate, start, end, sb + 2, len);

            if (type == FT_Poll)
            {
               clear_bits();

               if (F.lock == LOCK_F)
               {
                  clear_for_listen(L.c.mF[F.lockRate - 1], P.F[F.lockRate].corr, P.F[F.lockRate].p1);
                  F_note_zeroed(L.c.mF[F.lockRate - 1]);
                  L.fThrWritten |= 0x14u << (F.lockRate - 1); // searchLastValue / searchLastPhase cleared as well
               }

               return;
            }
         }

         F_reset();
         return;
      }

      st.data = (st.data << 1) | L.sym.value;

      if (++st.bits == 8)
      {
         put_byte(st.data);
         st.data = 0;
         st.bits = 0;
      }
   }

   // one sample of decodeListenFrameStartAsk, NfcF.cpp:749-936
   NFC_HD int F_listen_start()
   {
      const RateParams &b = P.F[F.lockRate];
      Mod &m = L.c.mF[F.lockRate - 1];
      FrameSt &fs = L.c.t[TECH_F].fs;
      const u32 clk = F.clk;

      FI(m) += SMP(NFCB200_OFF_X, b.sdd);
      FI(m) -= SMP(NFCB200_OFF_X, b.sdd + b.p2);

      if (clk < (fs.guardEnd - b.p1))
         return F_Invalid;

      float s0, s1, sd;
      F_correlate(b, m, F.cF[F.lockRate - 1], s0, s1, sd);

      if (clk < fs.guardEnd)
         return F_Invalid;

      if (clk == fs.guardEnd)
         m.searchValueThreshold = SMP(NFCB200_OFF_D, b.sdd) * 10;

      if (clk > fs.waitingEnd)
         return F_No;

      // note: the threshold passed for the `>=` test is searchValueThreshold itself (:814)
      if (!F_track_preamble(b, m, s0, sd, m.searchValueThreshold, true))
         return F_Invalid;

      L.sym.start = m.symbolStartTime - b.sdd;
      L.sym.end = m.symbolEndTime - b.sdd;
      L.sym.length = L.sym.end - L.sym.start;
      L.sym.pattern = F_S;
      return F_S;
   }

   NFC_HD void F_poll_step()
   {
      int pattern = F_symbol();
      if (pattern > F_No)
         F_frame_step(pattern, FT_Poll);
   }

   NFC_HD void F_listen_step()
   {
      FrameSt &fs = L.c.t[TECH_F].fs;

      if (!fs.frameStart)
      {
         int pattern = F_listen_start();

         if (pattern == F_S)
            fs.frameStart = L.sym.start;
         else if (pattern == F_No)
            F_reset();

         return;
      }

      int pattern = F_symbol();
      if (pattern > F_No)
         F_frame_step(pattern, FT_Listen);
   }

   // ------------------------------------------------------------------------------------------------------------------
   // NFC-V
   // ------------------------------------------------------------------------------------------------------------------
   enum { V_Invalid = 0, V_No = 1, V_0 = 2, V_1 = 3, V_2 = 4, V_8 = 5, V_S = 6, V_E = 7 };

   // NfcV::Impl::resetModulation, NfcV.cpp:1079-1103
   NFC_HD void V_reset()
   {
      clear_bits();
      clear_sym();
      zero_mod(L.c.mV);
      zero_ring(P.V.corr, P.V.p0 > P.V.p1 ? P.V.p0 : P.V.p1);
      zero_ring(NFCB200_OFF_I, NFCB200_RING);
      L.c.t[TECH_V].fs.frameType = 0;
      L.c.t[TECH_V].fs.frameStart = 0;
      L.c.t[TECH_V].fs.frameEnd = 0;
      L.pulseBits = 0;
      F.lock = LOCK_NONE;
   }

   NFC_HD static void V_clear_search(Mod &m)
   {
      m.symbolStartTime = 0;
      m.symbolEndTime = 0;
      m.searchStartTime = 0;
      m.searchEndTime = 0;
      m.correlatedPeakTime = 0;
      m.correlatedPeakValue = 0;
      m.detectorPeakTime = 0;
      m.detectorPeakValue = 0;
   }

   // half-symbol pulse correlator of detectModulation / decodePollFrameSymbolPpm (NfcV.cpp:258-274, 688-703)
   NFC_HD float V_pulse_corr(Mod &m, float &signalData)
   {
      const RateParams &b = P.V;
      u32 fp1 = F.cV1;
      u32 fp2 = fp1 + b.p2;
      if (fp2 >= b.p1)
         fp2 -= b.p1;

      const bool hoisted = staged_for(KIND_SEARCH) && F.lock == LOCK_NONE;

      signalData = tap(hoisted, TAP_XV0, SMP(NFCB200_OFF_X, b.sdd));

      FI(m) += signalData;
      FI(m) -= tap(hoisted, TAP_XV1, SMP(NFCB200_OFF_X, b.sdd + b.p2));

      RG(b.corr, fp1) = FI(m);

      return (tap(hoisted, TAP_CV2, RG(b.corr, fp2)) - FI(m)) / (float) b.p2;
   }

   // NfcV::Impl::detectModulation, NfcV.cpp:236-435
   NFC_HD bool V_detect()
   {
      const RateParams &b = P.V;
      Mod &m = L.c.mV;
      const u32 clk = F.clk;
      const float minimumCorrelationValue = F.env * P.thr[TECH_V].corr;

      float signalData;
      float s0 = V_pulse_corr(m, signalData);

      // idle fast path (not in the reference): nothing pending and the pulse correlation far below the trigger (:305)
      if (!(F.busy & 128u) && !(s0 > minimumCorrelationValue))
         return false;

      slow = true;

      float deep = depth_at(b.sdd + b.p8);

      if (m.correlatedPeakTime && clk > m.correlatedPeakTime + b.p0) // :287-298
      {
         m.symbolStartTime = 0;
         m.symbolEndTime = 0;
         m.searchStartTime = 0;
         m.searchEndTime = 0;
         m.searchSyncTime = 0;
         m.detectorPeakTime = 0;
         m.detectorPeakValue = 0;
         m.correlatedPeakTime = 0;
         m.correlatedPeakValue = 0;
      }

      if (clk < m.searchStartTime)
         return false;

      if (s0 > minimumCorrelationValue)
      {
         if (s0 > m.correlatedPeakValue)
         {
            m.correlatedPeakValue = s0;
            m.correlatedPeakTime = clk;
            m.searchEndTime = clk + b.p4;
         }

         if (deep > m.detectorPeakValue)
         {
            m.detectorPeakValue = deep;
            m.detectorPeakTime = clk;
         }
      }

      if (clk != m.searchEndTime)
         return false;

      if (signalData < minimumCorrelationValue || m.correlatedPeakTime == 0 || m.detectorPeakValue < P.thr[TECH_V].modMin)
      {
         V_clear_search(m);
         return false;
      }

      if (!m.symbolStartTime) // :345-359
      {
         m.symbolStartTime = m.correlatedPeakTime - b.p2;
         m.searchStartTime = m.symbolStartTime + (2 * b.p1);
         m.searchEndTime = m.symbolStartTime + (4 * b.p1);
         m.correlatedPeakTime = 0;
         m.correlatedPeakValue = 0;
         m.detectorPeakTime = 0;
         m.detectorPeakValue = 0;
         return false;
      }

      FrameSt &fs = L.c.t[TECH_V].fs;

      if (m.correlatedPeakTime > (m.symbolStartTime + 3 * b.p1 - b.p8) && m.correlatedPeakTime < (m.symbolStartTime + 3 * b.p1 + b.p8))
      {
         m.symbolEndTime = m.correlatedPeakTime + b.p1;
         m.searchSyncTime = m.symbolEndTime;
         m.searchStartTime = m.searchSyncTime;
         m.searchEndTime = m.searchSyncTime + P.V_len2;
         fs.symbolRate = b.sps / 2;
         L.pulseBits = 2;
      }
      else if (m.correlatedPeakTime > (m.symbolStartTime + 4 * b.p1 - b.p8) && m.correlatedPeakTime < (m.symbolStartTime + 4 * b.p1 + b.p8))
      {
         m.symbolEndTime = m.correlatedPeakTime;
         m.searchSyncTime = m.symbolEndTime;
         m.searchStartTime = m.searchSyncTime;
         m.searchEndTime = m.searchSyncTime + P.V_len8;
         fs.symbolRate = b.sps / 32;
         L.pulseBits = 8;
      }
      else
      {
         V_clear_search(m);
         return false;
      }

      fs.frameType = FT_Poll;
      fs.frameStart = m.symbolStartTime - b.sdd;
      fs.frameEnd = 0;

      m.correlatedPeakTime = 0;
      m.correlatedPeakValue = 0;
      m.searchValueThreshold = minimumCorrelationValue;

      F.lock = LOCK_V;
      F.lockRate = 0;
      return true;
   }

   // NfcV::Impl::checkCrc, NfcV.cpp:1194-1205
   NFC_HD bool V_crc_ok(u32 size) const
   {
      if (size < 3)
         return false;
      if (size > 512)
         return false; // past the 512-byte buffer (the reference's CRC reads beyond its buffer[512]): a CRC error
      unsigned short crc = (unsigned short) ~crc_ccitt16(sb, 0, size - 2, 0xFFFF, true);
      unsigned short res = (unsigned short) ((sb[size - 2] & 0xff) | ((sb[size - 1] & 0xff) << 8));
      return res == crc;
   }

   // NfcV::Impl::process, NfcV.cpp:1108-1189
   NFC_HD void V_process(u32 type, u32 len, u32 &flags, u32 &phase)
   {
      if (type != FT_Poll && !((L.lcWritten >> TECH_V) & 1))
         L.lcLive |= 1u << TECH_V; // a listen frame classified with the lastCommand this lane started from

      TechSt &t = L.c.t[TECH_V];
      FrameSt &fs = t.fs;
      const bool poll = type == FT_Poll;

      if (poll)
      {
         fs.frameGuardTime = t.ps.frameGuardTime;
         fs.frameWaitingTime = t.ps.frameWaitingTime;
      }
      else
      {
         fs.frameGuardTime = t.ps.frameGuardTime;
      }

      phase = PH_Application;
      flags |= !V_crc_ok(len) ? FL_Crc : 0;
      flags |= t.chained;

      if (poll)
      {
         if (F.lock == LOCK_V)
         {
            fs.guardEnd = fs.frameEnd + fs.frameGuardTime - P.V.sdd; // minus: NfcV.cpp:1147-1150
            fs.waitingEnd = fs.frameEnd + fs.frameWaitingTime - P.V.sdd;
            fs.frameType = FT_Listen;
         }
      }
      else
      {
         if (F.lock == LOCK_V)
            fs.guardEnd = fs.frameEnd + fs.frameGuardTime + P.V.sdd;
         fs.frameType = 0;
         fs.lastCommand = 0;
         L.lcWritten |= 1u << TECH_V;
      }

      fs.frameStart = 0;
      fs.frameEnd = 0;
   }

   // one sample of decodePollFrameSymbolPpm, NfcV.cpp:672-795
   NFC_HD int V_poll_symbol()
   {
      const RateParams &b = P.V;
      Mod &m = L.c.mV;
      const u32 clk = F.clk;

      float signalData;
      float s0 = V_pulse_corr(m, signalData);

      if (clk < m.searchStartTime)
         return V_Invalid;

      if (s0 > m.searchValueThreshold)
      {
         if (s0 > m.correlatedPeakValue)
         {
            m.correlatedPeakValue = s0;
            m.correlatedPeakTime = clk;
            m.searchEndTime = clk + b.p4;
         }
      }

      if (clk != m.searchEndTime)
         return V_Invalid;

      // EOF: pulse in the first half of the second slot (:734-751)
      if (m.correlatedPeakTime > (m.searchStartTime + 1 * b.p1 + b.p4) && m.correlatedPeakTime < (m.searchStartTime + 2 * b.p1 - b.p4))
      {
         m.symbolEndTime = m.correlatedPeakTime + b.p2;
         L.sym.value = 0;
         L.sym.start = m.symbolStartTime - b.sdd;
         L.sym.end = m.symbolEndTime - b.sdd;
         L.sym.length = L.sym.end - L.sym.start;
         L.sym.pattern = V_S;
         return V_S;
      }

      L.sym.value = 0;
      L.sym.start = m.symbolStartTime - b.sdd;
      L.sym.end = m.symbolEndTime - b.sdd;
      L.sym.length = L.sym.end - L.sym.start;
      L.sym.pattern = V_E;

      const u32 periods = 1u << L.pulseBits;
      const u32 length = L.pulseBits == 2 ? P.V_len2 : P.V_len8;

      // slot search (:761-789).  slot->end = round((i + 1) * stu * 256), NfcV.cpp:228-232
      for (u32 i = 0; i < periods; i++)
      {
         u32 slotEnd = (u32) (int) round((double) (i + 1) * P.stu * 256);

         if (m.correlatedPeakTime > (m.searchStartTime + slotEnd - b.p4) && m.correlatedPeakTime < (m.searchStartTime + slotEnd + b.p4))
         {
            m.symbolStartTime = m.correlatedPeakTime - slotEnd;
            m.symbolEndTime = m.symbolStartTime + length;
            m.searchSyncTime = m.symbolEndTime;
            m.searchStartTime = m.searchSyncTime;
            m.searchEndTime = m.searchSyncTime + length;
            m.correlatedPeakTime = 0;
            m.correlatedPeakValue = 0;

            L.sym.value = i;
            L.sym.start = m.symbolStartTime - b.sdd;
            L.sym.end = m.symbolEndTime - b.sdd;
            L.sym.length = L.sym.end - L.sym.start;
            L.sym.pattern = L.pulseBits == 2 ? V_2 : V_8;
            return (int) L.sym.pattern;
         }
      }

      return V_E;
   }

   // frame assembly of decodePollFrame (NfcV.cpp:450-556) / decodeListenFrame (:561-667)
   NFC_HD void V_frame_step(int pattern, u32 type)
   {
      TechSt &t = L.c.t[TECH_V];
      Bits &st = L.st;
      bool frameEnd = false, truncateError = false, streamError = false;

      if (pattern == V_S)
         frameEnd = true;
      else if (pattern == V_E)
         streamError = true;
      else if (st.bytes == t.ps.maxFrameSize)
         truncateError = true;

      if (frameEnd || streamError || truncateError)
      {
         if (st.bytes > 0)
         {
            if (st.bits == 8)
               put_byte(st.data);

            t.fs.frameEnd = L.sym.end;

            u32 flags = 0, phase = 0;
            if (truncateError || streamError)
               flags |= FL_Truncated;

            u32 len = st.bytes, rate = t.fs.symbolRate, start = t.fs.frameStart, end = t.fs.frameEnd;

            V_process(type, len, flags, phase);
            emit(TT_V, type, flags, phase, rate, start, end, sb, len);

            if (type == FT_Poll)
            {
               clear_bits();

               if (F.lock == LOCK_V)
                  clear_for_listen(L.c.mV, P.V.corr, P.V.p0 > P.V.p1 ? P.V.p0 : P.V.p1);

               return;
            }
         }

         V_reset();
         return;
      }

      if (st.bits == 8)
      {
         put_byte(st.data);
         st.data = 0;
         st.bits = 0;
      }

      st.data |= (L.sym.value << st.bits);
      st.bits += (type == FT_Poll) ? L.pulseBits : 1;
   }

   // full-symbol w^2 * 10 correlator of the NFC-V listen decoders (NfcV.cpp:817-835, 1000-1018)
   NFC_HD float V_listen_corr(Mod &m)
   {
      const RateParams &b = P.V;
      u32 fp1 = F.cV0;
      u32 fp2 = fp1 + b.p1;
      if (fp2 >= b.p0)
         fp2 -= b.p0;

      float data = SMP(NFCB200_OFF_W, b.sdd);
      float v = data * data * 10;
      SMP(NFCB200_OFF_I, b.sdd) = v;

      FI(m) += v;
      FI(m) -= SMP(NFCB200_OFF_I, b.sdd + b.p1);

      RG(b.corr, fp1) = FI(m);
      stage_drop(); // a slot of the ring's search-mode period (phase cV0, not cV1)

      return RG(b.corr, fp2) - FI(m);
   }

   // one sample of decodeListenFrameStartAsk, NfcV.cpp:800-980
   NFC_HD int V_listen_start()
   {
      const RateParams &b = P.V;
      Mod &m = L.c.mV;
      FrameSt &fs = L.c.t[TECH_V].fs;
      const u32 clk = F.clk;

      float s0 = V_listen_corr(m);
      float deep = depth_at(0);

      if (clk < fs.guardEnd)
         return V_Invalid;

      if (clk == fs.guardEnd)
         m.searchValueThreshold = SMP(NFCB200_OFF_D, b.sdd);

      if (clk > fs.waitingEnd)
         return V_No;

      if (deep > P.thr[TECH_V].modMax)
         return V_No;

      if (clk < m.searchStartTime)
         return V_Invalid;

      if (s0 < -m.searchValueThreshold && s0 < m.correlatedPeakValue)
      {
         m.correlatedPeakValue = s0;
         m.correlatedPeakTime = clk;
         m.searchEndTime = clk + b.p8;
      }

      if (s0 > m.searchValueThreshold && s0 > m.correlatedPeakValue)
      {
         m.correlatedPeakValue = s0;
         m.correlatedPeakTime = clk;
         m.searchEndTime = clk + b.p8;
      }

      if (clk != m.searchEndTime)
         return V_Invalid;

      if (m.searchModeState == 0) // LISTEN_MODE_PREAMBLE1
      {
         if (!m.symbolStartTime)
         {
            m.symbolStartTime = m.correlatedPeakTime - b.p1;
            m.searchStartTime = m.correlatedPeakTime + b.p0;
            m.searchEndTime = m.searchStartTime + b.p1;
            m.correlatedPeakValue = 0;
            m.correlatedPeakTime = 0;
            return V_Invalid;
         }

         m.symbolEndTime = m.correlatedPeakTime;

         u32 preambleS1Length = m.symbolEndTime - m.symbolStartTime - b.p1; // int vs unsigned: compared unsigned

         if (m.correlatedPeakTime == 0 || preambleS1Length < P.V_s1Min || preambleS1Length > P.V_s1Max)
         {
            m.searchModeState = 0;
            m.searchStartTime = 0;
            m.searchEndTime = 0;
            m.symbolStartTime = 0;
            m.symbolEndTime = 0;
            return V_Invalid;
         }

         m.searchModeState = 1;
         m.searchStartTime = m.correlatedPeakTime + b.p1 - b.p2;
         m.searchEndTime = m.searchStartTime + b.p1;
         m.correlatedPeakValue = 0;
         m.correlatedPeakTime = 0;
         return V_Invalid;
      }

      if (m.searchModeState == 1) // LISTEN_MODE_PREAMBLE2
      {
         u32 preambleS2Length = m.correlatedPeakTime - m.symbolEndTime;

         if (m.correlatedPeakTime == 0 || preambleS2Length < P.V_s2Min || preambleS2Length > P.V_s2Max)
         {
            m.searchModeState = 0;
            m.searchStartTime = 0;
            m.searchEndTime = 0;
            m.symbolStartTime = 0;
            m.symbolEndTime = 0;
            return V_Invalid;
         }

         m.symbolEndTime = m.correlatedPeakTime;
         m.searchSyncTime = m.symbolEndTime + b.p0;
         m.searchStartTime = m.searchSyncTime - b.p4;
         m.searchEndTime = m.searchSyncTime + b.p4;
         m.searchValueThreshold = (float) (m.correlatedPeakValue * 0.25);
         m.searchCorr0Value = 0;
         m.searchCorr1Value = 0;
         m.correlatedPeakTime = 0;
         m.correlatedPeakValue = 0;

         L.sym.value = 0;
         L.sym.start = m.symbolStartTime - b.sdd;
         L.sym.end = m.symbolEndTime - b.sdd;
         L.sym.length = L.sym.end - L.sym.start;
         L.sym.pattern = V_S;
         return V_S;
      }

      return V_Invalid;
   }

   // one sample of decodeListenFrameSymbolAsk, NfcV.cpp:985-1074
   NFC_HD int V_listen_symbol()
   {
      const RateParams &b = P.V;
      Mod &m = L.c.mV;
      const u32 clk = F.clk;

      float s0 = V_listen_corr(m);
      float sd = fabsf(s0);

      if (clk < m.searchStartTime)
         return V_Invalid;

      if (sd > m.searchValueThreshold && sd > m.correlatedPeakValue)
      {
         m.searchCorr0Value = s0;
         m.searchCorr1Value = -s0;
         m.correlatedPeakValue = sd;
         m.symbolEndTime = clk;
      }

      if (clk != m.searchEndTime)
         return V_Invalid;

      if (m.correlatedPeakValue < m.searchValueThreshold)
         return V_S;

      m.symbolStartTime = m.symbolEndTime;
      m.symbolEndTime = m.symbolStartTime + b.p0;
      m.searchSyncTime = m.symbolEndTime;
      m.searchStartTime = m.searchSyncTime - b.p4;
      m.searchEndTime = m.searchSyncTime + b.p4;
      m.searchValueThreshold = (float) (m.correlatedPeakValue * 0.25);
      m.correlatedPeakTime = 0;
      m.correlatedPeakValue = 0;

      L.sym.value = m.searchCorr0Value > m.searchCorr1Value ? 0 : 1;
      L.sym.start = m.symbolStartTime - b.sdd;
      L.sym.end = m.symbolEndTime - b.sdd;
      L.sym.length = L.sym.end - L.sym.start;
      L.sym.pattern = L.sym.value ? V_1 : V_0;

      return (int) L.sym.pattern;
   }

   NFC_HD void V_poll_step()
   {
      int pattern = V_poll_symbol();
      if (pattern > V_No)
         V_frame_step(pattern, FT_Poll);
   }

   NFC_HD void V_listen_step()
   {
      FrameSt &fs = L.c.t[TECH_V].fs;

      if (!fs.frameStart)
      {
         int pattern = V_listen_start();

         if (pattern == V_S)
            fs.frameStart = L.sym.start;
         else if (pattern == V_No)
            V_reset();

         return;
      }

      int pattern = V_listen_symbol();
      if (pattern > V_No)
         V_frame_step(pattern, FT_Listen);
   }

   // ------------------------------------------------------------------------------------------------------------------
   // latency hiding for the ring taps (device; no semantics).  A lone ring access costs an L2 / HBM round trip: the lane
   // scratch of all resident warps (852 kB per warp) is far larger than the caches, and every tap is its own 128-byte
   // line (32 lanes x 4 bytes), written hundreds of steps before it is read.  A warp step lasts far longer than one round
   // trip, and every tap of search mode and of the NFC-A poll and ASK listen decoders is at least two steps old when it
   // is read, except slot c - 1 of a correlation ring, which the previous step wrote.  So TAPS == 2 requests the taps of
   // step k + 1 at the start of step k (cp.async into the stage in shared memory: no registers held while in flight) and
   // forwards the slot c - 1 values from the writes of step k (put_corr).  The tap set is chosen from the state at step
   // k; step k + 1 uses its stage only when that choice matches what it runs, and reads the rings directly otherwise.
   // A stage is dropped by every ring write other than the per-step slot writes (zero_ring -- the wipes of the
   // correlation and integration rings when a listen phase starts or a decoder resets --, V_listen_corr) and by a restart
   // of the lane (reload_front), so the values used never depend on the prediction (NFCB200_CHECK_TAPS).  A step that
   // switches from the poll to the listen decoder wipes the rings, and its stage was chosen for the poll decoder anyway.
   // ------------------------------------------------------------------------------------------------------------------
   NFC_HD float *stage_base()
   {
      if constexpr (STRIDE == 1)
         return ownStage;
      return stg;
   }

   NFC_HD float &stage_word(u32 buf, u32 tap)
   {
      return stage_base()[(buf * TAP_COUNT + tap) * STG_STRIDE];
   }

   // both stages invalid; the requests still in flight land before anything new is requested
   NFC_HD void stage_reset()
   {
      if constexpr (TAPS == 2)
      {
#if defined(__CUDA_ARCH__)
         asm volatile("cp.async.wait_all;" ::: "memory");
#endif
         stgState &= STG_ON;
      }
   }

   // the next step's stage invalid (a ring write it may have read ahead of)
   NFC_HD void stage_drop()
   {
      if constexpr (TAPS == 2)
         stgState &= ~(0x1F0038u);
   }

   // this step's stage holds the tap set `kind`
   NFC_HD bool staged_for(u32 kind) const
   {
      return TAPS == 2 && (stgState & 7u) == kind;
   }

   // a tap: from this step's stage when `use`, else from the ring
   NFC_HD float tap(bool use, u32 t, RingRef direct)
   {
      if constexpr (TAPS == 2)
      {
         if (use)
         {
            const float v = stage_word(F.k & 1, t);
#if defined(NFCB200_CHECK_TAPS)
            union
            {
               float f;
               u32 u;
            } a, e;
            a.f = v;
            e.f = direct;
            const bool same = a.u == e.u;
#if defined(__CUDA_ARCH__)
            atomicAdd(&nfcb200_taps_used, 1ull);
            atomicAdd(&nfcb200_taps_kind[stgState & 7u], 1ull);
            if (!same)
               atomicAdd(&nfcb200_taps_differ, 1ull);
#elif !defined(__CUDACC__)
            nfcb200_taps_used++;
            nfcb200_taps_kind[stgState & 7u]++;
            nfcb200_taps_differ += same ? 0 : 1;
#endif
#endif
            return v;
         }
      }
      return direct;
   }

   // slot c - 1 of correlation ring `fwd` (TAP_FWD order): forwarded by the previous step when it wrote it
   NFC_HD float fwd_tap(bool use, u32 fwd, RingRef direct)
   {
      return tap(use && ((stgState >> (8 + fwd)) & 1u), TAP_FWD + fwd, direct);
   }

   // the per-step write of correlation ring `fwd` (slot c of this step), also forwarded into the next step's stage
   NFC_HD void put_corr(u32 fwd, u32 off, u32 slot, float v)
   {
      RG(off, slot) = v;
      if constexpr (TAPS == 2)
      {
         stage_word((F.k + 1) & 1, TAP_FWD + fwd) = v;
         stgState |= 1u << (16 + fwd);
      }
   }

   // request ring word (off, index) into word `t` of stage buffer `buf`
   NFC_HD void stage_fetch(u32 buf, u32 t, u32 off, u32 index)
   {
      float *dst = &stage_word(buf, t);
      const float *src = &rg[(off + index) * STRIDE];
#if defined(__CUDA_ARCH__)
      asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((u32) __cvta_generic_to_shared(dst)), "l"(src) : "memory");
#else
      *dst = *src;
#endif
   }

   // the taps the search-mode detectors read at the next step (ring phases and slot labels one step on)
   NFC_HD void stage_search(u32 buf)
   {
      for (int r = 0; r < 3; r++)
      {
         const RateParams &b = P.A[r];
         const u32 c = wrap(F.cA[r] + 1, b.p1);
         if (b.sdd)
            stage_fetch(buf, TAP_XA0 + r, NFCB200_OFF_X, slot_at(b.sdd, 1));
         stage_fetch(buf, TAP_XA1 + r, NFCB200_OFF_X, slot_at(b.sdd + b.p2, 1));
         stage_fetch(buf, TAP_CA2 + r, b.corr, wrap(c + b.p2, b.p1));
      }
      for (int r = 0; r < 2; r++)
         if (P.B[r].sdd)
            stage_fetch(buf, TAP_WB + r, NFCB200_OFF_W, slot_at(P.B[r].sdd, 1));
      for (int r = 1; r <= 2; r++)
      {
         const RateParams &b = P.F[r];
         const u32 c = wrap(F.cF[r - 1] + 1, b.p1);
         stage_fetch(buf, TAP_XF1 + r - 1, NFCB200_OFF_X, slot_at(b.sdd + b.p2, 1));
         stage_fetch(buf, TAP_CF2 + r - 1, b.corr, wrap(c + b.p2, b.p1));
      }
      const u32 c = wrap(F.cV1 + 1, P.V.p1);
      stage_fetch(buf, TAP_XV0, NFCB200_OFF_X, slot_at(P.V.sdd, 1));
      stage_fetch(buf, TAP_XV1, NFCB200_OFF_X, slot_at(P.V.sdd + P.V.p2, 1));
      stage_fetch(buf, TAP_CV2, P.V.corr, wrap(c + P.V.p2, P.V.p1));
   }

   // the taps of a locked NFC-A decoder of rate r at the next step: x[t-sdd] when sdd != 0, ring `off` at delay sdd + p2
   // and C[fp2].  A_poll_symbol() reads the sample ring (off = X); A_listen_ask_integrate() reads the integration ring
   // (off = I) and the edge value of the current step (rate 0, sdd == 0).
   NFC_HD void stage_a(u32 buf, u32 r, u32 off)
   {
      const RateParams &b = P.A[r];
      const u32 c = wrap(F.cA[r] + 1, b.p1);
      if (b.sdd)
         stage_fetch(buf, TAP_XA0 + r, NFCB200_OFF_X, slot_at(b.sdd, 1));
      stage_fetch(buf, TAP_XA1 + r, off, slot_at(b.sdd + b.p2, 1));
      stage_fetch(buf, TAP_CA2 + r, b.corr, wrap(c + b.p2, b.p1));
   }

   // start of a step (after front_advance): request the next step's taps, then wait for this step's
   NFC_HD void stage_advance()
   {
      const u32 s = stgState;
      u32 kind = 0;
      if (s & STG_ON)
      {
         if (F.lock == LOCK_NONE && !(F.k < F.gate)) // the next step is past the detector gate
            kind = KIND_SEARCH;
         else if (F.lock == LOCK_A)
         {
            const u32 frameType = L.c.t[TECH_A].fs.frameType;
            if (frameType == FT_Poll)
               kind = KIND_POLL + F.lockRate;
            else if (frameType == FT_Listen && F.lockRate == 0) // A_listen_step: ASK at 106 kbps, BPSK above
               kind = KIND_LISTEN_ASK + F.lockRate;
         }
      }

      const u32 next = (F.k + 1) & 1;
      if (kind == KIND_SEARCH)
         stage_search(next);
      else if (kind >= KIND_LISTEN_ASK)
         stage_a(next, kind - KIND_LISTEN_ASK, NFCB200_OFF_I);
      else if (kind)
         stage_a(next, kind - KIND_POLL, NFCB200_OFF_X);
      else if (F.lock != LOCK_NONE)
         prefetch_locked_taps(1);

#if defined(__CUDA_ARCH__)
      asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 1;" ::: "memory");
#endif
      // the next step's stage becomes this step's
      stgState = (s & STG_ON) | ((s >> 3) & 7u) | (kind << 3) | ((s >> 8) & 0x1F00u);
   }

   NFC_HD void prefetch_slot(u32 off, u32 index)
   {
#if defined(__CUDA_ARCH__)
      const float *ptr = &rg[(off + index) * STRIDE];
      asm volatile("prefetch.global.L2 [%0];" ::"l"(ptr));
#else
      (void) off;
      (void) index;
#endif
   }

   NFC_HD static u32 wrap(u32 slot, u32 period)
   {
      return slot >= period ? slot - period : slot;
   }

   // ring slot of the sample `delay` steps before the step `ahead` steps from now (front_advance() already ran)
   NFC_HD u32 slot_at(u32 delay, u32 ahead) const
   {
      return (F.k + F.kbase + ahead - delay) & (NFCB200_RING - 1);
   }

   // the symbol decoders of a locked lane read a handful of taps at fixed delays of their own rate
   NFC_HD void prefetch_locked_taps(u32 ahead)
   {
#if defined(__CUDA_ARCH__)
      const RateParams &b = locked_rate();
      prefetch_slot(NFCB200_OFF_X, slot_at(b.sdd, ahead));
      prefetch_slot(NFCB200_OFF_X, slot_at(b.sdd + b.p2, ahead));
      prefetch_slot(NFCB200_OFF_W, slot_at(b.sdd, ahead));
      prefetch_slot(NFCB200_OFF_W, slot_at(b.sdd + b.p1, ahead));
      prefetch_slot(NFCB200_OFF_I, slot_at(b.sdd + b.p2, ahead));
      prefetch_slot(NFCB200_OFF_I, slot_at(b.sdd + b.p4, ahead));
      prefetch_slot(NFCB200_OFF_I, slot_at(b.sdd + b.p1, ahead));
#else
      (void) ahead;
#endif
   }

   // ------------------------------------------------------------------------------------------------------------------
   // dispatch: NfcDecoder::Impl::nextFrames inner loops, NfcDecoder.cpp:393-442, one sample per call
   // ------------------------------------------------------------------------------------------------------------------
   NFC_HD void step(float x)
   {
      const bool wasLocked = F.lock != LOCK_NONE;

      step_body(x);

      // the busy mask is only read in search mode: rebuild it after a detector did more than its idle fast path, and
      // when a frame ended (the symbol decoders, process() and the resets rewrite the Mods freely)
      if (slow || (wasLocked && F.lock == LOCK_NONE))
      {
         refresh_busy();
         slow = false;
      }

#if defined(NFCB200_CHECK_BUSY)
      if (F.lock == LOCK_NONE)
      {
         const u32 have = F.busy;
         refresh_busy();
         if (have != F.busy)
            nfcb200_busy_mismatch(F.clk, have, F.busy);
      }
#endif
   }

   NFC_HD void step_body(float x)
   {
      front_advance();

      // the next step's taps are requested now; the envelope gate below is decided by this step's sample and a lane may
      // lock or unlock during this step, so some requests go unused, which is harmless
      if constexpr (TAPS == 2)
         stage_advance();

      if (featMode)
         front_feat();
      else
         front(x);

      if (F.lock == LOCK_NONE)
      {
         if (F.k > F.warm)
            detect_carrier();

         // `signalClock < BUFFER_SIZE` and `signalEnvelope < powerLevelThreshold` gates of every detectModulation
         if (F.k - 1 < F.gate || F.env < P.power)
         {
            if (!(F.k - 1 < F.gateSum) && !(F.env < P.power))
               sums_only();
            return;
         }

         if ((P.enabled & EN_A) && A_detect())
            L.lockedMask |= 1u << TECH_A;
         else if ((P.enabled & EN_B) && B_detect())
            L.lockedMask |= 1u << TECH_B;
         else if ((P.enabled & EN_F) && F_detect())
            L.lockedMask |= 1u << TECH_F;
         else if ((P.enabled & EN_V) && V_detect())
            L.lockedMask |= 1u << TECH_V;

         return;
      }

      u32 frameType;

      switch (F.lock)
      {
         case LOCK_A:
            frameType = L.c.t[TECH_A].fs.frameType;
            if (frameType == FT_Poll)
               A_poll_step();
            else if (frameType == FT_Listen)
               A_listen_step();
            break;
         case LOCK_B:
            frameType = L.c.t[TECH_B].fs.frameType;
            if (frameType == FT_Poll)
               B_poll_step();
            else if (frameType == FT_Listen)
               B_listen_step();
            break;
         case LOCK_F:
            frameType = L.c.t[TECH_F].fs.frameType;
            if (frameType == FT_Poll)
               F_poll_step();
            else if (frameType == FT_Listen)
               F_listen_step();
            break;
         default:
            frameType = L.c.t[TECH_V].fs.frameType;
            if (frameType == FT_Poll)
               V_poll_step();
            else if (frameType == FT_Listen)
               V_listen_step();
            break;
      }
   }

   // true when no timed event is pending: every future transition then needs a detector trigger, which the screening
   // kernel flags conservatively (DESIGN.md "dormant state")
   NFC_HD static bool mod_dormant(const Mod &m, u32 clk, u32 horizon)
   {
      if (m.searchStartTime && m.searchStartTime + horizon >= clk)
         return false;
      if (m.searchEndTime && m.searchEndTime + horizon >= clk)
         return false;
      if (m.searchSyncTime && m.searchSyncTime + horizon >= clk)
         return false;
      // a tracked peak always has a pending action: the "recover status" blocks (NfcA.cpp:268, NfcB.cpp:265,
      // NfcF.cpp:260, NfcV.cpp:287) clear it one period later, on the next search-mode sample at the latest
      if (m.correlatedPeakTime || m.detectorPeakTime)
         return false;
      return true;
   }

   NFC_HD bool dormant() const
   {
      if (F.lock != LOCK_NONE)
         return false;

      if (F.closed >= 16) // envelope not settled
         return false;

      const u32 clk = F.clk;
      const u32 horizon = P.V.p0 + 2; // longest recover timeout (NfcV.cpp:287) + margin

      for (int r = 0; r < 3; r++)
         if (!mod_dormant(L.c.mA[r], clk, horizon))
            return false;
      for (int r = 0; r < 2; r++)
      {
         if (!mod_dormant(L.c.mB[r], clk, horizon) || !mod_dormant(L.c.mF[r], clk, horizon))
            return false;

         // a stalled NFC-B SOF search reacts to edges above ITS OWN threshold (NfcB.cpp:313, 327, 366, 380); the
         // screening kernel only guarantees to flag edges above modMin * envelope, so a more sensitive residue keeps
         // the lane awake
         if (L.c.mB[r].symbolStartTime && L.c.mB[r].searchValueThreshold < F.env * P.thr[TECH_B].modMin)
            return false;
      }
      return mod_dormant(L.c.mV, clk, horizon);
   }

#undef RG
#undef SMP
};

// ---------------------------------------------------------------------------------------------------------------------
// lane construction
// ---------------------------------------------------------------------------------------------------------------------

// power-on carry: NfcX::initialize (NfcA.cpp:195-205 and twins)
NFC_HD void carry_init(Carry &c, const Params &P)
{
   u8 *raw = (u8 *) &c;
   for (u32 i = 0; i < sizeof(Carry); i++)
      raw[i] = 0;

   const u32 def[4][4] = {
      {P.A_sfgt, P.A_fgt, P.A_fwt, P.A_rgt},
      {P.B_sfgt, P.B_fgt, P.B_fwt, P.B_rgt},
      {P.F_sfgt, P.F_fgt, P.F_fwt, P.F_rgt},
      {P.V_sfgt, P.V_fgt, P.V_fwt, P.V_rgt},
   };

   for (int t = 0; t < 4; t++)
   {
      c.t[t].ps.maxFrameSize = 256;
      c.t[t].ps.startUpGuardTime = def[t][0];
      c.t[t].ps.frameGuardTime = def[t][1];
      c.t[t].ps.frameWaitingTime = def[t][2];
      c.t[t].ps.requestGuardTime = def[t][3];
      c.t[t].fs.startUpGuardTime = def[t][0];
      c.t[t].fs.frameGuardTime = def[t][1];
      c.t[t].fs.frameWaitingTime = def[t][2];
      c.t[t].fs.requestGuardTime = def[t][3];
   }
}

// ---------------------------------------------------------------------------------------------------------------------
// carry canonical form.  A retired (dormant, unlocked) lane leaves values behind that no later code path can read
// before overwriting them; zeroing those makes the carries of independent lanes comparable (DESIGN.md "carry groups").
//   * running sums restart with the rings in the next lane
//   * a detector whose search state is idle (no times, no peaks) rewrites every other Mod field before reading it:
//       NFC-B searchValueThreshold is reassigned each sample (NfcB.cpp:280); NFC-F searchLastPhase / LastValue /
//       Corr0Value / SyncValue are set by the first peak of a new search (NfcF.cpp:286-300, 344) -- but NFC-F's
//       searchValueThreshold and searchPulseWidth survive the "recover" path (NfcF.cpp:260-271) and ARE read by the
//       next search (:307-313), so an NFC-F Mod only counts as idle when those are zero too
//   * NfcFrameStatus: everything except lastCommand is reassigned by process() / detectModulation before use
//   * carrier times only matter as set / unset once their frame has been emitted (NfcDecoder.cpp:477, 502, 451)
// ---------------------------------------------------------------------------------------------------------------------
NFC_HD bool mod_idle(const Mod &m, bool isF)
{
   if (m.symbolStartTime | m.symbolEndTime | m.searchStartTime | m.searchEndTime | m.searchSyncTime | m.correlatedPeakTime | m.detectorPeakTime)
      return false;
   if (m.correlatedPeakValue != 0 || m.detectorPeakValue != 0)
      return false;
   if (isF && (m.searchPulseWidth != 0 || m.searchValueThreshold != 0))
      return false;
   return true;
}

NFC_HD void mod_canon(Mod &m, bool isF)
{
   m.filterIntegrate = 0;
   m.phaseIntegrate = 0;

   if (mod_idle(m, isF))
   {
      u32 *raw = (u32 *) &m;
      for (u32 i = 0; i < sizeof(Mod) / 4; i++)
         raw[i] = 0;
   }
   if (isF && m.searchPulseWidth > 94)
      m.searchPulseWidth = 94; // only ever read by `searchPulseWidth++ < 94` (NfcF.cpp:307, 844): every value from 94 on behaves alike

   if (!mod_idle(m, isF) && isF && !(m.searchSyncTime | m.searchEndTime))
   {
      // NFC-F residue (pulse counter / threshold survive between searches, NfcF.cpp:307-345) with no window pending: the
      // next window can only be opened by a fresh peak, which assigns searchSyncValue and searchCorr0Value before the
      // window end reads them (NfcF.cpp:283-292) -- the stale values are dead, and carrying them would make every later
      // lane depend on them
      m.searchSyncValue = 0;
      m.searchCorr0Value = 0;
   }
}

NFC_HD void carry_canon(Carry &c)
{
   for (int r = 0; r < 3; r++)
      mod_canon(c.mA[r], false);
   for (int r = 0; r < 2; r++)
   {
      mod_canon(c.mB[r], false);
      mod_canon(c.mF[r], true);
   }
   mod_canon(c.mV, false);

   for (int t = 0; t < 4; t++)
   {
      FrameSt &fs = c.t[t].fs;
      fs.frameType = fs.symbolRate = fs.frameStart = fs.frameEnd = fs.guardEnd = fs.waitingEnd = 0;
      fs.frameGuardTime = fs.frameWaitingTime = fs.startUpGuardTime = fs.requestGuardTime = 0;
   }

   c.carrierOn = c.carrierOn ? 1 : 0;
   c.carrierOff = c.carrierOff ? 1 : 0;
}

// carry groups: 0..3 detector residue of tech A/B/F/V (always live: the detectors run on every search-mode sample),
// 4..7 protocol state of tech A/B/F/V (only read or written while that tech is LOCKED), 8 carrier flags
#define NFCB200_GROUPS 9

NFC_HD void carry_group(Carry &c, int g, u32 *&ptr, u32 &words)
{
   switch (g)
   {
      case 0:
         ptr = (u32 *) c.mA;
         words = 3 * sizeof(Mod) / 4;
         break;
      case 1:
         ptr = (u32 *) c.mB;
         words = 2 * sizeof(Mod) / 4;
         break;
      case 2:
         ptr = (u32 *) c.mF;
         words = 2 * sizeof(Mod) / 4;
         break;
      case 3:
         ptr = (u32 *) &c.mV;
         words = sizeof(Mod) / 4;
         break;
      case 8:
         ptr = &c.carrierOn;
         words = 3;
         break;
      default:
         ptr = (u32 *) &c.t[g - 4];
         words = sizeof(TechSt) / 4;
         break;
   }
}

NFC_HD bool group_equal(Carry &a, Carry &b, int g)
{
   u32 *pa, *pb, wa, wb;
   carry_group(a, g, pa, wa);
   carry_group(b, g, pb, wb);
   for (u32 i = 0; i < wa; i++)
      if (pa[i] != pb[i])
         return false;
   return true;
}

NFC_HD void group_copy(Carry &dst, Carry &src, int g)
{
   u32 *pd, *ps, wd, ws;
   carry_group(dst, g, pd, wd);
   carry_group(src, g, ps, ws);
   for (u32 i = 0; i < wd; i++)
      pd[i] = ps[i];
}

// start a lane at absolute sample index `first` (the first sample it will be fed).  first == 0 is the exact reference
// start; otherwise this is the cold start of DESIGN.md: front end and rings restart from zero, carrier detection is
// held off for `warm` local steps while the averages converge, detectors for NFCB200_RING steps as in the reference.
// Out of line: it clears the whole Lane, and inlined into the thread lanes' kernel it set the register peak that made
// the step loop spill (DESIGN.md §5).
static NFC_HDN void lane_begin(Lane &L, const Params &P, const Carry &carry, u32 first, u32 warm)
{
   u8 *raw = (u8 *) &L;
   for (u32 i = 0; i < sizeof(Lane); i++)
      raw[i] = 0;

   L.c = carry;

   // accumulators restart with the rings (DESIGN.md "running sums")
   for (int r = 0; r < 3; r++)
      L.c.mA[r].filterIntegrate = L.c.mA[r].phaseIntegrate = 0;
   for (int r = 0; r < 2; r++)
   {
      L.c.mB[r].filterIntegrate = L.c.mB[r].phaseIntegrate = 0;
      L.c.mF[r].filterIntegrate = L.c.mF[r].phaseIntegrate = 0;
   }
   L.c.mV.filterIntegrate = L.c.mV.phaseIntegrate = 0;

   L.fe.clk = first - 1; // signalClock starts at -1 (NfcTech.h:338)
   L.fe.k = 0;
   L.fe.edgeTime = carry.edgeTime;

   for (int r = 0; r < 3; r++)
      L.fe.cA[r] = P.A[r].c1 ? P.A[r].c1 - 1 : P.A[r].p1 - 1; // incremented before use
   for (int r = 0; r < 2; r++)
      L.fe.cF[r] = P.F[r + 1].c1 ? P.F[r + 1].c1 - 1 : P.F[r + 1].p1 - 1;
   L.fe.cV1 = P.V.c1 ? P.V.c1 - 1 : P.V.p1 - 1;
   L.fe.cV0 = P.V.c0 ? P.V.c0 - 1 : P.V.p0 - 1;

   L.fe.warm = first ? warm : 0;
   // detectors stay off for the first 1024 samples of a stream like in the reference (signalClock < BUFFER_SIZE); a
   // cold-started lane keeps them off until 512 samples before its own region: enough to refill the correlation rings
   // (longest period 378), while the front end alone converges over the rest of the halo
   L.fe.gate = (first && warm > NFCB200_RING + 512) ? warm - 512 : NFCB200_RING;
   L.fe.gateSum = L.fe.gate;
   L.fe.edgeHold = first ? 64 : 0;
}

}

#endif
