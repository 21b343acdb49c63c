/*
 * tests/native/host_sim.cpp -- TEST-ONLY host build of the device lane machine (csrc/nfc_core.h).
 *
 * The product has no CPU path: nfc_core.h is device code and the shipped library (libnfcb200.so) only runs it inside
 * CUDA kernels.  This file compiles the same header with g++ so that the lane logic can be exercised in the GPU-less
 * CI container (`pytest -m "not gpu"`) against the reference oracle; it is never linked into the product library and
 * nothing in nfc_laboratory_b200/ imports it.
 *
 * Build (tests/conftest.py does this): g++ -O2 -msse2 -mfpmath=sse -ffp-contract=off -shared -fPIC
 */
#include <cmath>
#include <cstring>
#include <cstdlib>
#include <vector>
#include <cstdio>

// the host build always cross-checks the detectors' busy mask against the Mod fields it summarises (nfc_core.h step())
#define NFCB200_CHECK_BUSY 1
static inline void nfcb200_busy_mismatch(unsigned clk, unsigned have, unsigned want)
{
   std::fprintf(stderr, "host_sim: busy mask out of date at clock %u: have %02x, fields say %02x\n", clk, have, want);
   std::abort();
}

// per-sample value tap (nfc_core.h NFC_TRACE): rows of 8 floats [x, w, dev, avg, ch4, ch5, locked, 0], NaN = not written
#define NFCB200_TRACE_VALUES 1
static float *g_trace_row = nullptr;
static inline void nfcb200_trace_value(int channel, float value)
{
   if (g_trace_row && channel >= 0 && channel < 6)
      g_trace_row[channel] = value;
}

#include "../../nfc_laboratory_b200/csrc/nfc_wlane.h"

// tap fetch variant of the lane machine under test: the one the device library ships (nfcb200.cu laneTaps)
#ifndef NFCB200_SIM_TAPS
#define NFCB200_SIM_TAPS 2
#endif

using namespace nfcb200;

extern "C" {

struct sim_frame
{
   uint32_t tech, type, flags, phase, rate, start, end, len;
   uint8_t data[512];
};

struct sim_result
{
   uint32_t stop;     // absolute index of the first sample NOT consumed
   uint32_t dormant;  // lane state at stop
   uint32_t locked;
   uint32_t reserved;
};

}

struct Sink
{
   sim_frame *out;
   long cap;
   long count;

   void frame(const FrameOut &f, const u8 *payload)
   {
      if (count < cap)
      {
         sim_frame &o = out[count];
         o.tech = f.tech;
         o.type = f.type;
         o.flags = f.flags;
         o.phase = f.phase;
         o.rate = f.rate;
         o.start = f.start;
         o.end = f.end;
         o.len = f.len;
         std::memset(o.data, 0, sizeof(o.data));
         std::memcpy(o.data, payload, f.len);
      }
      count++;
   }
};

extern "C" {

int hostsim_carry_size(void)
{
   return (int) sizeof(Carry);
}

// decoder settings every later run takes (setup_params in nfcb200.cu): the power level and per tech the correlation and
// modulation thresholds; hostsim_set_settings(NULL, ...) goes back to the reference defaults
static bool g_settings = false;
static float g_power;
static TechThresholds g_thr[4];

void hostsim_set_settings(const float *corr, const float *modMin, const float *modMax, float power)
{
   g_settings = corr != nullptr;
   if (!g_settings)
      return;
   g_power = power;
   for (int t = 0; t < 4; t++)
      g_thr[t] = TechThresholds {corr[t], modMin[t], modMax[t]};
}

int hostsim_params(uint32_t sampleRate, uint32_t enabled, Params *P)
{
   std::memset(P, 0, sizeof(*P));
   params_defaults(P);
   P->enabled = enabled;
   if (g_settings)
   {
      P->power = g_power;
      for (int t = 0; t < 4; t++)
         P->thr[t] = g_thr[t];
   }
   params_init(P, sampleRate);
   return P->valid;
}

/* speculative carry of a lane that does not start at sample 0: power-on state, carrier already on */
void hostsim_default_carry(uint32_t sampleRate, void *out)
{
   Params P;
   hostsim_params(sampleRate, 0xF, &P);
   Carry c;
   carry_speculate(c, P);
   std::memcpy(out, &c, sizeof(Carry));
}

int hostsim_params_size(void)
{
   return (int) sizeof(Params);
}

/*
 * Run one lane over mag[first .. n) (mag indexed by absolute sample).  carry_in == NULL: power-on carry.
 * The lane stops at n, or -- when own_end > 0 -- at the first sample >= own_end where it is dormant and outside
 * every flagged block (flags: one byte per `block` samples, may be NULL).
 */
long hostsim_run(const float *mag, uint64_t n, uint32_t sampleRate, uint32_t enabled, uint32_t first, uint32_t warm, uint32_t own_end,
                 const void *carry_in, void *carry_out, sim_frame *out, long cap, sim_result *res, const uint8_t *flags, uint32_t block)
{
   Params P;
   if (!hostsim_params(sampleRate, enabled, &P))
      return -1;

   std::vector<float> scratch(NFCB200_SCRATCH_FLOATS, 0.0f);
   std::vector<u8> sb(512, 0);

   Carry carry;
   if (carry_in)
      std::memcpy(&carry, carry_in, sizeof(Carry));
   else
      carry_init(carry, P);

   Lane L;
   lane_begin(L, P, carry, first, warm);

   Sink sink {out, cap, 0};
   Machine<1, Sink, NFCB200_SIM_TAPS> M(P, L, L.fe, scratch.data(), sb.data(), sink);
   M.reload_front();

   uint64_t pos = first;

   for (; pos < n; pos++)
   {
      // a lane retires at the first sample past its own region where nothing is pending and the screen saw nothing
      if (own_end && pos >= own_end && !(flags && flags[pos / block]) && M.dormant())
         break;

      M.step(mag[pos]);
   }

   if (carry_out)
   {
      Carry c = L.c;
      c.edgeTime = L.fe.edgeTime;
      carry_canon(c);
      std::memcpy(carry_out, &c, sizeof(Carry));
   }

   if (res)
   {
      res->stop = (uint32_t) pos;
      res->dormant = M.dormant();
      res->locked = L.fe.lock;
      res->reserved = 0;
   }

   return sink.count;
}


/*
 * One lane from sample `first` (0 = the exact stream start; otherwise a cold start with `warm` warm-up samples), every
 * sample stepped, with the value tap on: rows[8 * i] for sample first + i.  Channel 6 = lock state after the step.
 */
long hostsim_trace(const float *mag, uint64_t n, uint32_t sampleRate, uint32_t enabled, uint32_t first, uint32_t warm, float *rows)
{
   Params P;
   if (!hostsim_params(sampleRate, enabled, &P))
      return -1;

   std::vector<float> scratch(NFCB200_SCRATCH_FLOATS, 0.0f);
   std::vector<u8> sb(512, 0);
   std::vector<sim_frame> frames(4096);

   Carry carry;
   if (first)
      carry_speculate(carry, P);
   else
   {
      carry_init(carry, P);
      carry_canon(carry);
   }

   Lane L;
   lane_begin(L, P, carry, first, warm);

   Sink sink {frames.data(), (long) frames.size(), 0};
   Machine<1, Sink, NFCB200_SIM_TAPS> M(P, L, L.fe, scratch.data(), sb.data(), sink);
   M.reload_front();

   const float nan = std::nanf("");
   for (uint64_t pos = first; pos < n; pos++)
   {
      float *row = rows + 8 * (pos - first);
      for (int c = 0; c < 8; c++)
         row[c] = nan;
      g_trace_row = row;
      M.step(mag[pos]);
      row[6] = (float) L.fe.lock;
      row[7] = 0;
   }
   g_trace_row = nullptr;
   return (long) (n - first);
}

// first sample of the lane whose own region starts at block bb (nfc_chain.h lane_first_sample)
uint32_t hostsim_first_sample(const uint8_t *flags, uint32_t nb, uint32_t bb)
{
   return lane_first_sample(flags, nb, bb);
}

/*
 * Whole-stream model of the product pipeline: segments from the screening flags (one byte per block, bit 0 = trigger),
 * one lane per segment, carry chain to the fixed point.  stats: [0] lanes [1] live lanes [2] rounds [3] lane runs
 * [4] samples stepped [5] active blocks
 */
struct HostSrc
{
   const float *mag;
   const Feat *pool;
   const uint8_t *flags;
   const float *bmeans;
   const SegRec *segs;
   uint32_t nsegs;
   bool exactInt;

   float x(uint32_t pos) const { return mag[pos]; }
   Feat feat(unsigned long long i) const { return pool[i]; }
   bool active(uint32_t pos) const { return (flags[pos / NFCB200_BLOCK] & SCR_ACTIVE) != 0; }
   float bmean(uint32_t b) const { return bmeans[b]; }
   const SegRec &seg(uint32_t i) const { return segs[i]; }
   uint32_t nseg() const { return nsegs; }
   bool exact_int() const { return exactInt; }
};

int g_hostsim_noff = 0;
int g_hostsim_nofeat = 0; // 1: no front pass, no feature pool: the warp lanes run the front-end recurrences themselves (the straggler pass)
int g_hostsim_bail = -1; // >= 0: a thread lane that runs this many samples past its queued length gives up and is decoded again by a warp
                         // lane without features (the straggler pass of the product, here without the "queue is empty" condition)
int g_hostsim_no_takeover = 0; // 1: lanes never take over their successors in-run (the chain walk alone extends regions)

static long pipeline_impl(const float *mag, uint64_t n, uint32_t sampleRate, uint32_t enabled, uint8_t *flags, uint32_t nb, sim_frame *out, long cap,
                          uint64_t *stats, uint32_t group, const Carry *init, uint32_t query, Carry *qOut, uint32_t *qBegin)
{
   Params P;
   if (!hostsim_params(sampleRate, enabled, &P))
      return -1;

   blocks_activate(flags, nb, init == nullptr);

   if (group < 1)
      group = 1;

   uint32_t nseg = blocks_segments(flags, nb, (uint32_t) n, 0, nullptr, 0, group);
   std::vector<LaneRec> lanes(nseg);
   blocks_segments(flags, nb, (uint32_t) n, 0, lanes.data(), nseg, group);

   for (uint32_t j = 0; j < nseg; j++)
   {
      // as segment_fill_kernel (nfc_decode.cuh): an injected carry stands in front of the first lane and is what the later
      // lanes speculate on
      if (init)
      {
         lanes[j].in = *init;
         if (lanes[j].first == 0)
            lanes[j].first = 1;
      }
      else if (lanes[j].first == 0)
      {
         carry_init(lanes[j].in, P);
         carry_canon(lanes[j].in);
      }
      else
         carry_speculate(lanes[j].in, P);
   }

   std::vector<std::vector<sim_frame>> frames(nseg);
   std::vector<float> scratch(NFCB200_SCRATCH_FLOATS);
   std::vector<u8> sb(512);

   uint64_t rounds = 0, runs = 0, work = 0, bails = 0;

   // segment table and block means for the straggler pass (group 1: lane j is segment j)
   std::vector<SegRec> segs(nseg);
   std::vector<float> bmeans(g_hostsim_bail >= 0 ? nb : 0);
   if (g_hostsim_bail >= 0)
   {
      for (uint32_t j = 0; j < nseg; j++)
      {
         std::memset(&segs[j], 0, sizeof(SegRec));
         segs[j].first = lanes[j].first;
         segs[j].begin = lanes[j].begin;
         segs[j].end = lanes[j].end0;
      }
      for (uint32_t b = 0; b < nb; b++)
      {
         double acc = 0;
         uint64_t cnt = 0;
         for (uint64_t i = (uint64_t) b * NFCB200_BLOCK; i < n && i < (uint64_t) (b + 1) * NFCB200_BLOCK; i++, cnt++)
            acc += mag[i];
         bmeans[b] = cnt ? (float) (acc / cnt) : 0.0f;
      }
   }

   for (;;)
   {
      bool any = false;
      std::vector<char> ranNow(nseg, 0);

      for (uint32_t j = 0; j < nseg; j++)
      {
         LaneRec &R = lanes[j];

         if (R.dead || !R.dirty)
            continue;

         any = true;
         ranNow[j] = 1;

         std::fill(scratch.begin(), scratch.end(), 0.0f);
         std::fill(sb.begin(), sb.end(), 0);

         std::vector<sim_frame> buf(4096);
         Sink sink {buf.data(), (long) buf.size(), 0};

         Lane L;
         lane_begin(L, P, R.in, R.first, R.begin - R.first);

         Machine<1, Sink, NFCB200_SIM_TAPS> M(P, L, L.fe, scratch.data(), sb.data(), sink);
   M.reload_front();

         uint32_t pos = R.first, kw = 0, stepped = 0;

         auto load = [&](uint32_t p) { return mag[p]; };
         auto active = [&](uint32_t p) { return (flags[p / NFCB200_BLOCK] & SCR_ACTIVE) != 0; };
         auto zero = [&]() { std::fill(scratch.begin() + NFCB200_OFF_CA, scratch.end(), 0.0f); };

         uint32_t end = R.end;
         LaneSucc succ;
         succ.init(lanes.data(), j, nseg);
         if (g_hostsim_no_takeover)
            succ.nextFirst = 0xFFFFFFFFu;

         bool bailed = false;
         const uint32_t patience = g_hostsim_bail >= 0 ? R.end - R.first + (uint32_t) g_hostsim_bail : 0xFFFFFFFFu;
         while (lane_iterate(M, L, P, pos, end, (uint32_t) n, kw, stepped, load, active, zero, succ))
         {
            kw++;
            if (stepped > patience)
            {
               bailed = true;
               break;
            }
         }

         if (bailed)
         {
            // the product's straggler pass: the lane again, by a warp lane that runs the front end itself
            bails++;
            work += stepped;
            std::fill(scratch.begin(), scratch.end(), 0.0f);
            std::fill(sb.begin(), sb.end(), 0);
            sink.count = 0;
            Lane WLn;
            WShared sh;
            std::memset(&sh, 0, sizeof(sh));
            HostSrc src {mag, nullptr, flags, bmeans.data(), segs.data(), nseg, false};
            WLane<HostWarp, Sink, HostSrc> WL(P, WLn, scratch.data(), sb.data(), sink, sh, src);
            WL.run(R, j, (uint32_t) n);
            lane_record(R, WLn, sh.pos, R.gen + 2, (uint32_t) sink.count, R.end);
            buf.resize(sink.count);
            frames[j] = buf;
            runs++;
            work += sh.stepped;
            continue;
         }

         lane_record(R, L, pos, R.gen + 1, (uint32_t) sink.count, R.end); // the committed region only moves in chain_walk
         buf.resize(sink.count);
         frames[j] = buf;

         runs++;
         work += stepped;
      }

      if (!any)
         break;

      rounds++;

      if (getenv("HOSTSIM_ROUNDS"))
      {
         fprintf(stderr, "round %llu ran:", (unsigned long long) rounds);
         for (uint32_t j = 0; j < nseg; j++)
            if (!lanes[j].dead && lanes[j].dirty == 0 && lanes[j].gen > 0 && lanes[j].nframes + 1 > 0 && lanes[j].stop && ranNow[j])
               fprintf(stderr, " %u", j);
         fprintf(stderr, "\n");
      }

      chain_walk(lanes.data(), nseg, P, init);
   }

   if (qOut)
      carry_before(lanes.data(), nseg, P, init, query, *qOut, *qBegin);

   if (getenv("HOSTSIM_LANES"))
      for (uint32_t j = 0; j < nseg; j++)
         fprintf(stderr, "lane %u first %u begin %u end %u stop %u dead %u gen %u frames %u\n", j, lanes[j].first, lanes[j].begin, lanes[j].end, lanes[j].stop,
                 lanes[j].dead, lanes[j].gen, lanes[j].nframes);

   long count = 0;
   uint64_t live = 0;

   for (uint32_t j = 0; j < nseg; j++)
   {
      if (lanes[j].dead)
         continue;

      live++;

      for (const sim_frame &f: frames[j])
      {
         if (count < cap)
            out[count] = f;
         count++;
      }
   }

   if (stats)
   {
      uint64_t act = 0;
      for (uint32_t b = 0; b < nb; b++)
         act += (flags[b] & SCR_ACTIVE) ? 1 : 0;
      stats[0] = nseg;
      stats[1] = live;
      stats[2] = rounds;
      stats[3] = runs;
      stats[4] = work;
      stats[5] = act;
      stats[6] = bails;
   }

   return count;
}


long hostsim_pipeline(const float *mag, uint64_t n, uint32_t sampleRate, uint32_t enabled, uint8_t *flags, uint32_t nb, sim_frame *out, long cap,
                      uint64_t *stats, uint32_t group)
{
   return pipeline_impl(mag, n, sampleRate, enabled, flags, nb, out, cap, stats, group, nullptr, 0, nullptr, nullptr);
}

/*
 * One window of a time-sharded capture (nfcb200_set_carry / nfcb200_carry_before on the host): carry_in (or null) stands in
 * front of the window's first lane; carry_out / lane_begin answer the carry query at `query` (lane_begin 0xFFFFFFFF: no lane
 * begins at or after it)
 */
long hostsim_window(const float *mag, uint64_t n, uint32_t sampleRate, uint32_t enabled, uint8_t *flags, uint32_t nb, sim_frame *out, long cap,
                    const void *carry_in, uint32_t query, void *carry_out, uint32_t *lane_begin)
{
   Carry in, q;
   if (carry_in)
   {
      memcpy(&in, carry_in, sizeof(Carry));
      carry_canon(in);
   }
   uint32_t b = 0xFFFFFFFFu;
   long r = pipeline_impl(mag, n, sampleRate, enabled, flags, nb, out, cap, nullptr, 1, carry_in ? &in : nullptr, query, &q, &b);
   if (carry_out)
      memcpy(carry_out, &q, sizeof(Carry));
   if (lane_begin)
      *lane_begin = b;
   return r;
}


/*
 * Whole-stream model of the round-2 product pipeline (nfc_wlane.h): segments from the screening flags, the front pass per
 * segment into a feature pool, one WARP LANE (here: a one-thread warp) per group of segments, carry chain to the fixed point.
 * group == 0: ONE lane for the whole stream (exact running sums, no speculation).  noff != 0: every sample goes through the
 * per-sample machine (fast-forward paths off) -- the self-check of the fast paths.
 * stats: [0] lanes [1] live lanes [2] rounds [3] lane runs [4] samples stepped [5] active blocks [6] segments [7] feature samples
 */

long hostsim_pipeline2(const float *mag, uint64_t n, uint32_t sampleRate, uint32_t enabled, uint8_t *flags, uint32_t nb, sim_frame *out, long cap,
                       uint64_t *stats, uint32_t group, uint32_t exactInt)
{
   Params P;
   if (!hostsim_params(sampleRate, enabled, &P))
      return -1;

   blocks_activate(flags, nb);

   // block means (the device takes them from the screening pass)
   std::vector<float> bmeans(nb);
   for (uint32_t b = 0; b < nb; b++)
   {
      double acc = 0;
      uint64_t cnt = 0;
      for (uint64_t i = (uint64_t) b * NFCB200_BLOCK; i < n && i < (uint64_t) (b + 1) * NFCB200_BLOCK; i++, cnt++)
         acc += mag[i];
      bmeans[b] = cnt ? (float) (acc / cnt) : 0.0f;
   }

   // segments and their feature ranges
   uint32_t nseg = blocks_segments(flags, nb, (uint32_t) n, 0, nullptr, 0, 1);
   std::vector<LaneRec> segl(nseg);
   blocks_segments(flags, nb, (uint32_t) n, 0, segl.data(), nseg, 1);
   std::vector<SegRec> segs(nseg);
   uint64_t total = 0;
   for (uint32_t i = 0; i < nseg; i++)
   {
      SegRec &S = segs[i];
      std::memset(&S, 0, sizeof(S));
      S.stream = 0;
      S.first = segl[i].first;
      S.begin = segl[i].begin;
      S.end = segl[i].end;
      S.featOff = total;
      total += S.end - S.first;
   }
   std::vector<Feat> pool(g_hostsim_nofeat ? 1 : total);
   for (uint32_t i = 0; i < nseg && !g_hostsim_nofeat; i++)
   {
      SegRec &S = segs[i];
      Feat *dst = pool.data() + S.featOff;
      front_pass(P, S.first, S.end, [&](uint32_t p) { return mag[p]; },
                 [&](uint32_t i, float w, float env, float dev, float avg) { dst[i] = Feat {w, env, dev, avg}; }, S);
      S.hasFeat = 1;
   }

   // lanes
   const uint32_t grp = group ? group : (nseg ? nseg : 1);
   uint32_t nlanes = blocks_segments(flags, nb, (uint32_t) n, 0, nullptr, 0, grp);
   std::vector<LaneRec> lanes(nlanes);
   blocks_segments(flags, nb, (uint32_t) n, 0, lanes.data(), nlanes, grp);
   std::vector<uint32_t> seg0(nlanes);
   for (uint32_t j = 0, i = 0; j < nlanes; j++)
   {
      while (i < nseg && segs[i].begin != lanes[j].begin)
         i++;
      seg0[j] = i;
      if (lanes[j].first == 0)
      {
         carry_init(lanes[j].in, P);
         carry_canon(lanes[j].in);
      }
      else
         carry_speculate(lanes[j].in, P);
   }

   HostSrc src {mag, pool.data(), flags, bmeans.data(), segs.data(), nseg, exactInt != 0};

   std::vector<std::vector<sim_frame>> frames(nlanes);
   std::vector<float> scratch(NFCB200_SCRATCH_FLOATS);
   std::vector<u8> sb(512);
   uint64_t rounds = 0, runs = 0, work = 0;

   for (;;)
   {
      bool any = false;

      for (uint32_t j = 0; j < nlanes; j++)
      {
         LaneRec &R = lanes[j];
         if (R.dead || !R.dirty)
            continue;
         any = true;

         std::fill(scratch.begin(), scratch.end(), 0.0f);
         std::fill(sb.begin(), sb.end(), 0);
         std::vector<sim_frame> buf(65536);
         Sink sink {buf.data(), (long) buf.size(), 0};

         Lane L;
         WShared sh;
         std::memset(&sh, 0, sizeof(sh));
         WLane<HostWarp, Sink, HostSrc> WL(P, L, scratch.data(), sb.data(), sink, sh, src);
         WL.noff = g_hostsim_noff != 0;
         WL.run(R, seg0[j], (uint32_t) n);

         if (getenv("HOSTSIM_PHASES"))
            fprintf(stderr, "lane %u [%u,%u) stop %u: control %llu fill %llu search %llu machine %llu walk %llu jump %llu scalar %llu locked %llu\n", j, R.first,
                    R.end, sh.pos, sh.cnt[0], sh.cnt[1], sh.cnt[2], sh.cnt[3], sh.cnt[4], sh.cnt[5], sh.cnt[6], sh.cnt[7]);

         lane_record(R, L, sh.pos, R.gen + 1, (uint32_t) sink.count, R.end);
         buf.resize(std::min<long>(sink.count, (long) buf.size()));
         frames[j] = buf;
         runs++;
         work += sh.stepped;
      }

      if (!any)
         break;
      rounds++;
      chain_walk(lanes.data(), nlanes, P);
   }

   long count = 0;
   uint64_t live = 0;
   for (uint32_t j = 0; j < nlanes; j++)
   {
      if (lanes[j].dead)
         continue;
      live++;
      for (const sim_frame &f: frames[j])
      {
         if (count < cap)
            out[count] = f;
         count++;
      }
   }

   if (stats)
   {
      uint64_t act = 0;
      for (uint32_t b = 0; b < nb; b++)
         act += (flags[b] & SCR_ACTIVE) ? 1 : 0;
      stats[0] = nlanes;
      stats[1] = live;
      stats[2] = rounds;
      stats[3] = runs;
      stats[4] = work;
      stats[5] = act;
      stats[6] = nseg;
      stats[7] = total;
   }
   return count;
}

void hostsim_set_no_takeover(int v)
{
   g_hostsim_no_takeover = v;
}

void hostsim_set_bail(int v)
{
   g_hostsim_bail = v;
}

void hostsim_set_nofeat(int v)
{
   g_hostsim_nofeat = v;
}

void hostsim_set_noff(int v)
{
   g_hostsim_noff = v;
}

}
