/*
 * nfc_chain.h -- segment construction and the speculative carry chain (host + device).
 *
 * The reference decoder is one sequential state machine per capture stream (NfcDecoder.cpp:393-442).  Here a stream is
 * cut into SEGMENTS around the blocks the dense screening pass flagged; every segment is decoded by an independent lane
 * that cold-starts HALO samples early (front end and rings re-converge bit-exactly, SURVEY.md 8e) from a SPECULATED
 * carry.  chain_walk() then walks the lanes of one stream in time order, composes the true carry, and marks the lanes
 * whose speculation was wrong; those are re-run.  At the fixed point every lane ran from exactly the carry its
 * predecessor left, i.e. the lanes together performed the reference's sequential computation.
 *
 * Nothing here has a counterpart in the reference (which has no parallelism on this path).
 */
#ifndef NFCB200_CHAIN_H
#define NFCB200_CHAIN_H

#include "nfc_core.h"

namespace nfcb200 {

#define NFCB200_BLOCK 256       /* samples per screening block                                   */
#define NFCB200_HALO 4096       /* lane warm-up, samples                                          */
#ifndef NFCB200_HALO_SHORT
#define NFCB200_HALO_SHORT 1536 /* warm-up of a lane that never comes near the carrier thresholds */
#endif
#define NFCB200_PRE_BLOCKS 2    /* active margin before a flagged block                           */
#ifndef NFCB200_POST_BLOCKS
#define NFCB200_POST_BLOCKS 4   /* active margin after a flagged block                            */
#endif
#define NFCB200_GAP_BLOCKS 32   /* regions closer than this form one segment (>= 2 * HALO / BLOCK) */
#define NFCB200_START_BLOCKS 8  /* the stream start is always a segment                           */

// screening flag bits (one byte per block)
enum { SCR_TRIGGER = 1, SCR_ACTIVE = 2, SCR_START = 4, SCR_BAND = 8 };

struct LaneRec
{
   u32 stream;
   u32 begin;      // own region [begin, end), samples, block aligned (end clipped to the stream length)
   u32 end;
   u32 end0;       // end of the region as segmented (end grows when the lane takes over its successors)
   u32 first;      // first sample fed to the lane (begin - HALO, or 0)
   u32 stop;       // first sample NOT consumed by the last run
   u32 lockedMask; // techs locked during the last run
   u32 gen;        // number of runs so far (frames carry the generation that produced them)
   u32 dirty;      // must (re-)run
   u32 dead;       // swallowed by its predecessor
   u32 nframes;    // frames emitted by the last run
   // what the last run observed of its incoming carry (copied from Lane, see nfc_core.h)
   u32 lcWritten, lcLive, fZeroed, fThrWritten, fThrRead;
   u32 fInc0[2];
   float fThrSync[2];
   u32 edgeWritten, edgeLive;
   u32 seg0;       // index of the lane's first segment in the segment table (nfc_wlane.h)
   Carry in;       // carry the last run started from
   Carry out;      // canonical carry the last run retired with
};

/*
 * First sample of the lane whose own region starts at block `bb`.  The warm-up exists for the front-end recurrences to
 * re-converge bit-exactly; the slowest is the carrier average (0.995 per sample, ~3500 samples), which only feeds
 * detect_carrier()'s comparisons against the power thresholds.  SCR_BAND marks the blocks in which that average (block
 * model of segment_flags_kernel, 20 % margins) can come near a threshold.  Without such a block anywhere between the long
 * warm-up start and the point where the average is exact again, the 0.05 % the average is still off after the short
 * warm-up cannot change a comparison: the lane may start HALO_SHORT samples early (the deviation EMA, 0.98 per sample,
 * the envelope and the DC filter converge in < 1000 samples, the sample rings fill in 1024, the detectors open 512
 * samples before the region either way).
 */
NFC_HD u32 lane_first_sample(const u8 *flags, u32 nb, u32 bb, bool allowShort = true)
{
   const u32 begin = bb * NFCB200_BLOCK;
   if (begin <= NFCB200_HALO)
      return 0;
   if (!allowShort)
      return begin - NFCB200_HALO;
   const u32 lo = bb - NFCB200_HALO / NFCB200_BLOCK;
   u32 hi = bb + (NFCB200_HALO - NFCB200_HALO_SHORT) / NFCB200_BLOCK + 1;
   if (hi > nb)
      hi = nb;
   for (u32 b = lo; b < hi; b++)
      if (flags[b] & SCR_BAND)
         return begin - NFCB200_HALO;
   return begin - NFCB200_HALO_SHORT;
}

// dilate the raw trigger flags into active blocks, in place: bit SCR_ACTIVE.  streamStart: the buffer begins at the stream's
// first sample.  false for a window that continues a capture from an injected carry: its first START_BLOCKS blocks are
// warm-up (the screen's own start-up transient triggers there; what they hold belongs to the predecessor's window)
NFC_HD void blocks_activate(u8 *flags, u32 nb, bool streamStart = true)
{
   // forward reach (POST) and backward reach (PRE) of every trigger
   int reach = 0;
   for (u32 b = 0; b < nb; b++)
   {
      if ((flags[b] & SCR_TRIGGER) && (streamStart || b >= NFCB200_START_BLOCKS))
         reach = NFCB200_POST_BLOCKS + 1;
      if (reach > 0 || (streamStart && b < NFCB200_START_BLOCKS))
         flags[b] |= SCR_ACTIVE;
      if (reach > 0)
         reach--;
   }
   reach = 0;
   for (u32 b = nb; b-- > 0;)
   {
      if ((flags[b] & SCR_TRIGGER) && (streamStart || b >= NFCB200_START_BLOCKS))
         reach = NFCB200_PRE_BLOCKS + 1;
      if (reach > 0)
         flags[b] |= SCR_ACTIVE;
      if (reach > 0)
         reach--;
   }
}

// emit the lanes of one stream: every lane owns `group` consecutive segments (it skips the idle stretches between them
// itself, re-warming from its own exact carry); returns the number of lanes (only `cap` are stored)
NFC_HD u32 blocks_segments(const u8 *flags, u32 nb, u32 nsamples, u32 stream, LaneRec *out, u32 cap, u32 group = 1)
{
   u32 count = 0;
   u32 b = 0;
   u32 inGroup = 0;

   while (b < nb)
   {
      if (!(flags[b] & SCR_ACTIVE))
      {
         b++;
         continue;
      }

      u32 last = b;
      u32 e = b;

      while (e < nb && ((flags[e] & SCR_ACTIVE) || e - last < NFCB200_GAP_BLOCKS))
      {
         if (flags[e] & SCR_ACTIVE)
            last = e;
         e++;
      }

      u32 segEnd = (last + 1) * NFCB200_BLOCK;
      if (segEnd > nsamples)
         segEnd = nsamples;

      if (inGroup == 0)
      {
         if (count < cap)
         {
            LaneRec &l = out[count];
            l.stream = stream;
            l.begin = b * NFCB200_BLOCK;
            l.end = segEnd;
            l.end0 = segEnd;
            l.first = lane_first_sample(flags, nb, b);
            l.stop = 0;
            l.lockedMask = 0;
            l.gen = 0;
            l.dirty = 1;
            l.dead = 0;
            l.nframes = 0;
         }
         count++;
      }
      else if (count - 1 < cap)
      {
         out[count - 1].end = segEnd;
         out[count - 1].end0 = segEnd;
      }

      if (++inGroup >= group)
         inGroup = 0;

      b = last + 1;
   }

   return count;
}

// the lanes that follow a running lane in its stream (time ordered, contiguous in the lane table).  Only first / end0 /
// stream of those records are read: they never change after the segment pass
struct LaneSucc
{
   const LaneRec *lanes;
   u32 k, n;       // next candidate, table size
   u32 stream;
   u32 nextFirst;  // lanes[k].first, or 0xFFFFFFFF when the stream has no further lane

   NFC_HD void init(const LaneRec *table, u32 self, u32 count)
   {
      lanes = table;
      n = count;
      k = self + 1;
      stream = table ? table[self].stream : 0;
      load();
   }
   NFC_HD void load() { nextFirst = (lanes && k < n && lanes[k].stream == stream) ? lanes[k].first : 0xFFFFFFFFu; }
   NFC_HD void take(u32 pos, u32 &end)
   {
      while (pos > nextFirst)
      {
         if (lanes[k].end0 > end)
            end = lanes[k].end0;
         k++;
         load();
      }
   }
};

// restart a lane at `target` from its own canonical carry (lane_iterate's skip-ahead), out of line: it runs a few times
// per lane and takes no part in the register allocation of the step loop
static NFC_HDN void lane_restart(Lane &L, const Params &P, u32 target, u32 kw)
{
   Carry carry = L.c;
   carry.edgeTime = L.fe.edgeTime;
   carry_canon(carry);
   // what the run has recorded so far about its use of the INCOMING carry (chain_walk reads it) survives the restart:
   // the run goes on from its own exact carry, it does not start a new dependency history
   const u32 locked = L.lockedMask, lcWritten = L.lcWritten, lcLive = L.lcLive, fZeroed = L.fZeroed, fThrWritten = L.fThrWritten,
             fThrRead = L.fThrRead, fInc00 = L.fInc0[0], fInc01 = L.fInc0[1];
   const float fThrSync0 = L.fThrSync[0], fThrSync1 = L.fThrSync[1];
   const u32 edgeWritten = L.edgeWritten, edgeLive = L.edgeLive;
   lane_begin(L, P, carry, target, NFCB200_HALO);
   L.lockedMask = locked;
   L.lcWritten = lcWritten;
   L.lcLive = lcLive;
   L.fZeroed = fZeroed;
   L.fThrWritten = fThrWritten;
   L.fThrRead = fThrRead;
   L.fInc0[0] = fInc00;
   L.fInc0[1] = fInc01;
   L.fThrSync[0] = fThrSync0;
   L.fThrSync[1] = fThrSync1;
   L.edgeWritten = edgeWritten;
   L.edgeLive = edgeLive;
   L.fe.kbase = kw;
}

/*
 * Drive one lane from R.first until it retires past R.end (or the stream ends).  Inside its own region the lane skips
 * idle stretches: when it is dormant outside every active block it jumps to HALO samples before the next active block
 * and re-warms from its own canonical carry -- exactly what a separate lane with a verified carry would do.
 *   LOAD(pos)    -> magnitude sample at absolute index pos
 *   ACTIVE(pos)  -> block of pos is active
 *   ZERO()       -> wipe the correlation rings of the lane's scratch
 *   kw           -> warp-uniform iteration counter (ring slot labels), advanced by the caller's loop on the device;
 *                   the host build passes its own counter
 * One call = one iteration (at most one sample).  Returns false when the lane has retired.
 */
template <class MACH, class LOAD, class ACTIVE, class ZERO>
NFC_HD bool lane_iterate(MACH &M, Lane &L, const Params &P, u32 &pos, u32 &end, u32 n, u32 kw, u32 &stepped, LOAD load, ACTIVE active, ZERO zero,
                         LaneSucc &succ)
{
   if (pos >= n)
      return false;

   // still running past the point where the next lane of the stream started its warm-up: that lane will be swallowed
   // (chain_walk), so its region is taken over right away instead of in a re-run over the extended region
   if ((pos & 31) == 0 && pos > succ.nextFirst)
      succ.take(pos, end);

   // retirement / skip-ahead is only examined every 32 samples (it costs a walk over all detector states)
   if ((pos & 31) == 0 && !active(pos) && M.dormant())
   {
      if (pos >= end)
         return false;

      // next active block inside the own region (end is the end of an active block, so one exists)
      u32 b = pos >> 8;
      while (((b + 1) << 8) < end && !active(b << 8))
         b++;

      u32 begin = b << 8;

      if (begin > pos + NFCB200_HALO)
      {
         const u32 target = begin - NFCB200_HALO;
         zero();
         lane_restart(L, P, target, kw);
         M.reload_front();
         pos = target;
      }
   }

   M.step(load(pos));
   pos++;
   stepped++;
   return true;
}

// carry composed in front of the first live lane that begins at or after `sample` (valid once the chain has converged);
// laneBegin receives that lane's begin (or 0xFFFFFFFF when the stream has no such lane: the carry is then the final one)
NFC_HD void carry_before(LaneRec *lanes, u32 n, const Params &P, const Carry *init, u32 sample, Carry &out, u32 &laneBegin);

// copy the outcome of a finished run into its record
NFC_HD void lane_record(LaneRec &R, const Lane &L, u32 stop, u32 gen, u32 nframes, u32 end)
{
   R.stop = stop;
   R.end = end; // grown over the successors the run took over (lane_iterate)
   R.lockedMask = L.lockedMask;
   R.out = L.c;
   R.out.edgeTime = L.fe.edgeTime;
   carry_canon(R.out);
   R.gen = gen;
   R.dirty = 0;
   R.nframes = nframes;
   R.lcWritten = L.lcWritten;
   R.lcLive = L.lcLive;
   R.fZeroed = L.fZeroed;
   R.fThrWritten = L.fThrWritten;
   R.fThrRead = L.fThrRead;
   R.fInc0[0] = L.fInc0[0];
   R.fInc0[1] = L.fInc0[1];
   R.fThrSync[0] = L.fThrSync[0];
   R.fThrSync[1] = L.fThrSync[1];
   R.edgeWritten = L.edgeWritten;
   R.edgeLive = L.edgeLive;
}

// word offsets inside Mod / TechSt used by the relaxed dependency rules
#define NFCB200_MOD_WORDS (sizeof(Mod) / 4)
#define NFCB200_W_PULSE 4 /* Mod::searchPulseWidth     */
#define NFCB200_W_THR 5   /* Mod::searchValueThreshold */
#define NFCB200_W_LASTPHASE 7 /* Mod::searchLastPhase   */
#define NFCB200_W_LASTVALUE 8 /* Mod::searchLastValue   */

NFC_HD float u32_as_float(u32 v)
{
   union
   {
      u32 u;
      float f;
   } c;
   c.u = v;
   return c.f;
}

// what the last run of a lane recorded about its use of the incoming carry (copied from LaneRec: the word rules below
// are shared by the scalar walk and by the warp-parallel device walk)
struct LaneObs
{
   u32 edgeWritten, edgeLive;
   u32 lcWritten, lcLive, fZeroed, fThrWritten, fThrRead;
   u32 fInc0[2];
   float fThrSync[2];
   u32 inert;      // bit t: the TRUE carry in front of the run has maxFrameSize == 0 for tech t (set by the composing caller)
};

// a zero maxFrameSize (an RFU frame-size code in ATTRIB / RATS, NfcB.cpp:1235, NfcA.cpp:1664) truncates every later frame of
// that technology at its first byte: no command is recognised any more, the protocol status is never assigned again.
// Only used to PREDICT the carry behind a run that must be repeated: the repeat will assign nothing
NFC_HD u32 carry_inert_mask(const Carry &c)
{
   u32 m = 0;
   for (int t = 0; t < 4; t++)
      if (c.t[t].ps.maxFrameSize == 0)
         m |= 1u << t;
   return m;
}

NFC_HD LaneObs lane_obs(const LaneRec &L)
{
   LaneObs o;
   o.inert = 0;
   o.edgeWritten = L.edgeWritten;
   o.edgeLive = L.edgeLive;
   o.lcWritten = L.lcWritten;
   o.lcLive = L.lcLive;
   o.fZeroed = L.fZeroed;
   o.fThrWritten = L.fThrWritten;
   o.fThrRead = L.fThrRead;
   o.fInc0[0] = L.fInc0[0];
   o.fInc0[1] = L.fInc0[1];
   o.fThrSync[0] = L.fThrSync[0];
   o.fThrSync[1] = L.fThrSync[1];
   return o;
}

/*
 * Word w of carry group g differs between the carry the run assumed (a) and the true carry (t): could the run have
 * observed the difference?  Plain word equality decides, except for three values whose only reads are known:
 *   - frameStatus.lastCommand (word 0 of the protocol groups): read only by the listen-frame classifiers; a run whose
 *     first classified listen frame followed an assignment in the same run never saw the carried value (lcLive)
 *   - NFC-F searchPulseWidth: read only by `searchPulseWidth++ < 94` (NfcF.cpp:307, 844); until its first reset the run
 *     executed fInc0 such tests, all with the same outcome under both carries iff both stay below / above 94 throughout
 *   - NFC-F searchValueThreshold: until its first assignment it is compared once, against fThrSync (NfcF.cpp:313, 331)
 *   - NFC-F searchLastValue / searchLastPhase: stale values of an earlier search that the reference never clears; read
 *     only at a threshold pass (LastValue, NfcF.cpp:344) and at the preamble's final test (LastPhase, :349), normally after
 *     the run's own assignment (:300, :344) -- the run notes when it was not (fThrRead bits 2.. / 4..)
 */
NFC_HD bool word_observed_equal(const LaneObs &L, int g, u32 w, u32 a, u32 t)
{
   if (a == t)
      return true;

   if (g >= 4 && g < 8 && w == 0)
      return !((L.lcLive >> (g - 4)) & 1);

   if (g == 8 && w == 2) // carrier edge time: read only when a carrier frame is stamped, before the run's own first assignment
      return !L.edgeLive;

   if (g == 2)
   {
      u32 r = w / NFCB200_MOD_WORDS, f = w % NFCB200_MOD_WORDS;

      if (f == NFCB200_W_PULSE)
      {
         u32 n = L.fInc0[r];
         u32 hi = a > t ? a : t;
         u32 lo = a > t ? t : a;
         return n == 0 || hi + n <= 94 || lo >= 94;
      }

      if (f == NFCB200_W_THR)
      {
         if (!((L.fThrRead >> r) & 1))
            return true;
         float sv = L.fThrSync[r], fa = u32_as_float(a), ft = u32_as_float(t);
         return (sv < fa) == (sv < ft) && (sv > fa) == (sv > ft);
      }

      if (f == NFCB200_W_LASTVALUE)
         return !((L.fThrRead >> (2 + r)) & 1);

      if (f == NFCB200_W_LASTPHASE)
         return !((L.fThrRead >> (4 + r)) & 1);
   }

   return false;
}

// did the last run of L observe anything of carry group g that differs between L.in and the true carry `cur`?
NFC_HD bool group_observed_equal(LaneRec &L, Carry &cur, int g)
{
   u32 *pa, *pb, wa, wb;
   carry_group(L.in, g, pa, wa);
   carry_group(cur, g, pb, wb);
   const LaneObs obs = lane_obs(L);

   for (u32 w = 0; w < wa; w++)
      if (!word_observed_equal(obs, g, w, pa[w], pb[w]))
         return false;

   return true;
}

/*
 * Word w of carry group g after the last run of a lane, given the true carry word before it (n), the word the run
 * retired with (o) and the word it started from (i): a word the run left unchanged passes the (corrected) incoming value
 * through, any other keeps the run's value; the three special values follow their own bookkeeping.
 */
NFC_HD u32 compose_word(const LaneObs &L, int g, u32 w, u32 n, u32 o, u32 i)
{
   if (g >= 4 && g < 8 && w == 0)
      return ((L.lcWritten >> (g - 4)) & 1) ? o : n;

   // protocol status (TechSt words 11..15): assigned by the run, or passed through
   if (g >= 4 && g < 8 && w >= sizeof(FrameSt) / 4 && w < (sizeof(FrameSt) + sizeof(Proto)) / 4)
   {
      if ((L.inert >> (g - 4)) & 1)
         return n; // whatever the run assigned, it did so from a state in which frames decode; from the true state none does
      return ((L.lcWritten >> (8 + 5 * (g - 4) + (w - sizeof(FrameSt) / 4))) & 1) ? o : n;
   }

   if (g == 8 && w == 2)
      return L.edgeWritten ? o : n;

   if (g == 2)
   {
      u32 r = w / NFCB200_MOD_WORDS, f = w % NFCB200_MOD_WORDS;

      if (f == NFCB200_W_PULSE)
      {
         // not reset: the run added one per window-end test (fInc0); the canonical form saturates at 94 (mod_canon)
         if ((L.fZeroed >> r) & 1)
            return o;
         const u32 v = n + L.fInc0[r];
         return v > 94 ? 94 : v;
      }

      if (f == NFCB200_W_THR)
         return ((L.fThrWritten >> r) & 1) ? o : n;

      if (f == NFCB200_W_LASTVALUE)
         return ((L.fThrWritten >> (2 + r)) & 1) ? o : n;

      if (f == NFCB200_W_LASTPHASE)
         return ((L.fThrWritten >> (4 + r)) & 1) ? o : n;
   }

   return o != i ? o : n;
}

// carry after the last run of L, given the true carry `cur` before it (exact when the run is valid, a prediction else)
NFC_HD void carry_compose(LaneRec &L, Carry &cur, Carry &next, u32 touched)
{
   next = cur;
   LaneObs obs = lane_obs(L);
   obs.inert = carry_inert_mask(cur);

   for (int g = 0; g < NFCB200_GROUPS; g++)
   {
      if (!((touched >> g) & 1))
         continue;

      u32 *pn, *po, *pi, wn, wo, wi;
      carry_group(next, g, pn, wn);
      carry_group(L.out, g, po, wo);
      carry_group(L.in, g, pi, wi);

      for (u32 w = 0; w < wn; w++)
         pn[w] = compose_word(obs, g, w, pn[w], po[w], pi[w]);
   }
}

// speculated carry of a lane that does not start at sample 0: power-on state with the carrier already detected
NFC_HD void carry_speculate(Carry &c, const Params &P)
{
   carry_init(c, P);
   carry_canon(c);
   c.carrierOn = 1;
}

/*
 * Walk the lanes [0, n) of ONE stream (time ordered).  Returns the number of lanes left dirty.
 *   - a lane whose predecessor was still busy after the lane's own warm-up had started is swallowed: the
 *     predecessor's region is extended over it (and the predecessor re-runs if it had already retired earlier)
 *   - otherwise the lane's last run is valid iff, on every carry group it can observe, it started from the carry
 *     composed so far; groups it cannot observe (protocol state of techs it never locked) pass through
 *   - the carry after a lane is PREDICTED for lanes that must re-run: groups the last run left unchanged are assumed
 *     to pass the corrected value through (pure heuristic -- validity is only ever established by the equality test)
 */
NFC_HD u32 chain_walk(LaneRec *lanes, u32 n, const Params &P, const Carry *init = nullptr)
{
   Carry cur;
   if (init)
      cur = *init; // the stream does not start at power-on: a time shard of a longer capture continues its predecessor's carry
   else
   {
      carry_init(cur, P);
      carry_canon(cur);
   }

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

         // Q's reach: where its last run stopped, or -- once its region was extended -- at least the new region end
         u32 reach = Q.stop > Q.end ? Q.stop : Q.end;

         if (Q.gen > 0 && (!Q.dirty || Q.stop < Q.end) && reach > L.first)
         {
            L.dead = 1;
            L.dirty = 0;
            if (Q.end < L.end)
               Q.end = L.end;
            if (Q.stop < Q.end && !Q.dirty)
            {
               Q.dirty = 1;
               ndirty++;
            }
            continue;
         }
      }

      const bool ran = L.gen > 0;
      u32 touched = 0x10F | ((L.lockedMask & 0xF) << 4); // groups 0..3 and 8 always, 4 + t when tech t was locked
      bool ok = ran;

      if (ran)
      {
         for (int g = 0; g < NFCB200_GROUPS; g++)
            if ((touched >> g) & 1)
               if (!group_observed_equal(L, cur, g))
               {
                  ok = false;
#ifdef NFCB200_CHAIN_DEBUG
                  printf("   lane %u [%u,%u) gen %u: group %d differs\n", j, L.begin, L.end, L.gen, g);
                  u32 *pa, *pb, wa, wb;
                  carry_group(L.in, g, pa, wa);
                  carry_group(cur, g, pb, wb);
                  for (u32 i = 0; i < wa; i++)
                     if (!word_observed_equal(lane_obs(L), g, i, pa[i], pb[i]))
                        printf("        word %u: assumed %08x true %08x\n", i, pa[i], pb[i]);
#endif
               }
      }

      // carry after this lane
      Carry next = cur;

      if (ran)
         carry_compose(L, cur, next, touched);

      if (!ok)
      {
         if (ran)
            L.in = cur; // a lane that never ran keeps the carry it was created with (power-on or speculated)
         L.dirty = 1;
      }

      if (L.dirty)
         ndirty++;

#ifdef NFCB200_CHAIN_DEBUG
      printf("   lane %u [%u,%u) first %u gen %u ran %d ok %d locked %x lcW %x lcL %x: lastCommand in %02x/%02x out %02x/%02x -> carry %02x/%02x (A/B)\n", j, L.begin,
             L.end, L.first, L.gen, (int) ran, (int) ok, L.lockedMask, L.lcWritten, L.lcLive, L.in.t[0].fs.lastCommand, L.in.t[1].fs.lastCommand,
             L.out.t[0].fs.lastCommand, L.out.t[1].fs.lastCommand, next.t[0].fs.lastCommand, next.t[1].fs.lastCommand);
#endif

      cur = next;
      prev = (int) j;
   }

   return ndirty;
}


NFC_HD void carry_before(LaneRec *lanes, u32 n, const Params &P, const Carry *init, u32 sample, Carry &out, u32 &laneBegin)
{
   Carry cur;
   if (init)
      cur = *init;
   else
   {
      carry_init(cur, P);
      carry_canon(cur);
   }

   laneBegin = 0xFFFFFFFFu;

   for (u32 j = 0; j < n; j++)
   {
      LaneRec &L = lanes[j];
      if (L.dead)
         continue;
      if (L.begin >= sample)
      {
         laneBegin = L.begin;
         break;
      }
      if (L.gen > 0)
      {
         Carry next = cur;
         carry_compose(L, cur, next, 0x10F | ((L.lockedMask & 0xF) << 4));
         cur = next;
      }
   }

   out = cur;
}

}

#endif
