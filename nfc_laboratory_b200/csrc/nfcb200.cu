/*
 * nfcb200.cu -- C ABI (include/nfcb200.h) and host orchestration of the H100 NFC demodulation path: the handle, batch
 * decode, streaming, the carry of time shards and the frame gather.  The spectrum and the ISO 7816 decoder have their own
 * units (spectrum.cu, iso7816.cu); what the units share is in host.h.
 *
 * The kernels live in nfc_screen.cuh / nfc_decode.cuh, the exact lane machine in nfc_core.h.
 * Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -fmad=false -shared -Xcompiler -fPIC
 * (-fmad=false: the reference's x86 build has no FMA, CMakeLists.txt:36-40; lane decisions must be bit-identical).
 *
 * There is no CPU fallback in this library: every entry point that decodes requires a CUDA device.
 */
#include <chrono>
#include <cmath>
#include <cstdarg>
#include <cstddef>
#include <numeric>

#include "host.h"
#include "nfc_decode.cuh"

using namespace nfcb200;

// ---------------------------------------------------------------------------------------------------------------------
// errors
// ---------------------------------------------------------------------------------------------------------------------
static thread_local char g_error[512] = "";

int nfcb200::fail(int code, const char *fmt, ...)
{
   va_list ap;
   va_start(ap, fmt);
   vsnprintf(g_error, sizeof(g_error), fmt, ap);
   va_end(ap);
   return code;
}

struct Counters
{
   u32 poolCount;
   u32 extCount;
   u32 queueCount;
   u32 cursor;
   u32 overrunCount; // lanes that gave up in the thread-lane kernel (stragglers), decoded again by warp lanes
   u32 pad0;
   unsigned long long work;
   unsigned long long live;
   u32 segTotal;
   u32 activeBlocks;
   unsigned long long featTotal;
   unsigned long long phase[16];
};

// host-side milestones of a call, printed when NFCB200_TRACE is set (debug aid)
struct Trace
{
   bool on;
   std::chrono::steady_clock::time_point t0, last;
   Trace() : on(getenv("NFCB200_TRACE") != nullptr), t0(std::chrono::steady_clock::now()), last(t0) {}
   double ms() const { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count(); }
   void mark(const char *what)
   {
      if (!on)
         return;
      auto now = std::chrono::steady_clock::now();
      fprintf(stderr, "[nfcb200] %-28s +%8.2f ms (%8.2f)\n", what, std::chrono::duration<double, std::milli>(now - last).count(),
              std::chrono::duration<double, std::milli>(now - t0).count());
      last = now;
   }
};

static int setup_params(nfcb200_handle *h, u32 sampleRate)
{
   Params &P = h->P;
   h->paramsRate = 0; // the block is rebuilt in place: a rejected rate must not leave the previous rate marked as current
   memset(&P, 0, sizeof(P));
   params_defaults(&P);
   P.enabled = h->cfg.enabled & 0xF;
   P.streamTime = h->cfg.stream_time;
   P.power = h->cfg.power_level_threshold;
   for (int t = 0; t < 4; t++)
   {
      P.thr[t].corr = h->cfg.correlation_threshold[t];
      P.thr[t].modMin = h->cfg.modulation_min[t];
      P.thr[t].modMax = h->cfg.modulation_max[t];
   }
   params_init(&P, sampleRate);

   if (!P.valid)
      return fail(NFCB200_ERR_UNSUPPORTED, "sample rate %u is outside the supported range of the device ring layout", sampleRate);

   // the screening tile keeps SCR_HALO samples of history: every correlator tap must fit
   if (P.V.p1 + 2 > SCR_HALO || P.A[0].p1 + 2 > SCR_HALO || NFCB200_BLOCK * 2 > SCR_HALO)
      return fail(NFCB200_ERR_UNSUPPORTED, "sample rate %u needs a longer screening halo than %d samples", sampleRate, SCR_HALO);

   h->paramsRate = sampleRate;
   return 0;
}

// K1 launch: one instantiation per sample format, persistent grid of 2 CTAs per SM
static void launch_screen(const nfcb200_handle *h, const ScreenConfig &sc, uint32_t items, cudaStream_t st)
{
   const u32 grid = std::min<u32>(items, (u32) h->smCount * 2);
   switch (sc.sigtype)
   {
      case SIG_IQ_F32:
         screen_kernel<SIG_IQ_F32, false><<<grid, SCR_THREADS, sizeof(ScreenSmem), st>>>(sc, items);
         break;
      case SIG_MAG_F32:
         screen_kernel<SIG_MAG_F32, false><<<grid, SCR_THREADS, sizeof(ScreenSmem), st>>>(sc, items);
         break;
      case SIG_MAG_S16:
         screen_kernel<SIG_MAG_S16, false><<<grid, SCR_THREADS, sizeof(ScreenSmem), st>>>(sc, items);
         break;
      default:
         screen_kernel<SIG_IQ_S16, false><<<grid, SCR_THREADS, sizeof(ScreenSmem), st>>>(sc, items);
         break;
   }
}

// front pass: one instantiation per sample format
static void launch_front(const FrontConfig &fc, const Params &P, cudaStream_t st)
{
   const u32 grid = (fc.n_segs + FRONT_THREADS - 1) / FRONT_THREADS;
   switch (fc.sigtype)
   {
      case SIG_IQ_F32:
         front_kernel<SIG_IQ_F32><<<grid, FRONT_THREADS, 0, st>>>(fc, P);
         break;
      case SIG_MAG_F32:
         front_kernel<SIG_MAG_F32><<<grid, FRONT_THREADS, 0, st>>>(fc, P);
         break;
      case SIG_MAG_S16:
         front_kernel<SIG_MAG_S16><<<grid, FRONT_THREADS, 0, st>>>(fc, P);
         break;
      default:
         front_kernel<SIG_IQ_S16><<<grid, FRONT_THREADS, 0, st>>>(fc, P);
         break;
   }
}

// K1, shared by the batch decode and streaming: screening of [n_streams][n_samples] samples into per-block flags and
// sums.  `useTma` returns whether the bulk copies were allowed.
static int screen(const nfcb200_handle *h, const void *samples, int sigtype, u32 n_streams, uint64_t n_samples, DevBuf &flags, DevBuf &bsum,
                  cudaStream_t st, int &useTma)
{
   const u32 n_blocks = (u32) ((n_samples + NFCB200_BLOCK - 1) / NFCB200_BLOCK);
   const u32 tiles = (u32) ((n_samples + SCR_TILE - 1) / SCR_TILE);
   int rc = flags.reserve((size_t) n_streams * n_blocks);
   rc = rc ? rc : bsum.reserve((size_t) n_streams * n_blocks * sizeof(float));
   if (rc)
      return rc;

   ScreenConfig sc;
   memset(&sc, 0, sizeof(sc));
   sc.samples = samples;
   sc.n_samples = n_samples;
   sc.n_streams = n_streams;
   sc.sigtype = sigtype;
   sc.n_blocks = n_blocks;
   sc.tiles_per_stream = tiles;
   sc.flags = flags.as<uint8_t>();
   sc.bsum = bsum.as<float>();
   const Params &P = h->P;
   const float margin = 0.9f;
   for (int r = 0; r < 3; r++)
   {
      sc.p1[r] = P.A[r].p1;
      sc.p2[r] = P.A[r].p2;
   }
   sc.vp1 = P.V.p1;
   sc.vp2 = P.V.p2;
   // rate 106 is only used by NFC-A; 212 / 424 by NFC-A and NFC-F; disabled techs still screen (conservative).
   // thr = min(0.9 T p2, T p2 - 1.25) / 2, lowered by the change the decimated evaluation can miss (nfc_screen.cuh)
   const float cA = P.thr[TECH_A].corr, cF = P.thr[TECH_F].corr, cV = P.thr[TECH_V].corr;
   const float T[3] = {cA, std::min(cA, cF), std::min(cA, cF)};
   for (int r = 0; r < 3; r++)
   {
      float p2 = (float) P.A[r].p2;
      sc.thrA[r] = std::min(margin * T[r] * p2, T[r] * p2 - 1.25f) * 0.5f;
   }
   // decimated evaluation: |C[t] - C[t-q]| moves by at most 2 xmax = 2.5 env per sample
   sc.thrA[1] -= 1 * 2.5f;   // 212k: every 2nd sample
   sc.thrA[0] -= 3 * 2.5f;   // 106k: every 4th sample
   {
      float p2 = (float) P.V.p2;
      // NFC-V: S0 = (C[t-q] - C[t]) / p2 > T env (NfcV.cpp:274, 305); every 8th sample
      sc.thrV = std::min(margin * cV * p2, cV * p2 - 1.25f) - 7 * 2.5f;
   }
   for (int r = 0; r < 3; r++)
      sc.thrA[r] = std::max(sc.thrA[r], 0.25f);
   sc.thrV = std::max(sc.thrV, 0.25f);
   sc.kB = margin * P.thr[TECH_B].modMin;
   // quiet bound of a warp span (nfc_screen.cuh): no test can fire while max - min <= quiet * min
   {
      float q = sc.kB;
      for (int r = 0; r < 3; r++)
         q = std::min(q, sc.thrA[r] / (float) P.A[r].p2);
      q = std::min(q, sc.thrV / (float) P.V.p2);
      sc.quiet = 0.999f * q;
   }
   sc.use_tma = h->cfg.use_tma ? 1 : 0;
   // cp.async.bulk needs 16-byte aligned global addresses: stream pitch and base pointer
   if ((((uintptr_t) samples) & 15) || ((n_samples * sig_bytes(sigtype)) & 15))
      sc.use_tma = 0;

   const uint64_t items = (uint64_t) n_streams * tiles;
   if (items >= 0xFFFF0000ull)
      return fail(NFCB200_ERR_CAPACITY, "batch of %llu screening tiles exceeds one launch", (unsigned long long) items);
   launch_screen(h, sc, (u32) items, st);
   CUDA_TRY(cudaGetLastError());
   useTma = sc.use_tma;
   return 0;
}

// block flags after the screen, shared by the batch decode and streaming: level shifts and the carrier band, dilated into
// active blocks.  The batch decode extends the returned configuration for its later segment kernels.
static SegmentConfig flag_blocks(const nfcb200_handle *h, const DevBuf &flags, const DevBuf &bsum, u32 n_streams, uint64_t n_samples,
                                 const Carry *carryIn, u32 *activeTotal, cudaStream_t st)
{
   SegmentConfig sg;
   memset(&sg, 0, sizeof(sg));
   sg.flags = flags.as<uint8_t>();
   sg.bsum = bsum.as<float>();
   sg.n_streams = n_streams;
   sg.n_blocks = (u32) ((n_samples + NFCB200_BLOCK - 1) / NFCB200_BLOCK);
   sg.n_samples = n_samples;
   sg.low = h->P.lowThr;
   sg.high = h->P.highThr;
   sg.meanW = powf(h->P.meanW0, (float) NFCB200_BLOCK);
   sg.group = 1;
   sg.carryIn = carryIn;
   sg.activeTotal = activeTotal;
   const u32 bgrid = (u32) (((uint64_t) n_streams * sg.n_blocks + 255) / 256);
   segment_flags_kernel<<<bgrid, 256, 0, st>>>(sg);
   segment_activate_kernel<<<bgrid, 256, 0, st>>>(sg);
   return sg;
}

// the device frame pool of the batch decode and of streaming: `cap` records, `extCap` 128-byte chunks, counted in dC
static int frame_pool(DevBuf &recs, DevBuf &ext, u32 cap, u32 extCap, Counters *dC, FramePool &pool)
{
   int rc = recs.reserve((size_t) cap * sizeof(FrameRec));
   rc = rc ? rc : ext.reserve((size_t) extCap * 128);
   if (rc)
      return rc;
   pool.recs = recs.as<FrameRec>();
   pool.cap = cap;
   pool.count = &dC->poolCount;
   pool.ext = ext.as<u8>();
   pool.extCap = extCap;
   pool.extCount = &dC->extCount;
   return 0;
}

// convert one pool record to the ABI frame
static void emit_frame(const nfcb200_handle *h, const FrameRec &r, const unsigned char *ext, size_t extBytes, u32 stream, u32 sampleRate, nfcb200_frame &o)
{
   // header, payload, and zeros up to the next 64-byte boundary after the payload (the rest of data[] is not touched:
   // a batch of 4e5 frames would otherwise write 250 MB of zeros)
   memset(&o, 0, offsetof(nfcb200_frame, data));
   o.stream = stream;
   o.tech_type = r.tech;
   o.frame_type = r.type;
   o.frame_flags = r.flags;
   o.frame_phase = r.phase;
   o.frame_rate = r.rate;
   o.sample_start = r.start;
   o.sample_end = r.end;
   o.sample_rate = sampleRate;
   o.time_start = (double) r.start / (double) sampleRate;
   o.time_end = (double) r.end / (double) sampleRate;
   o.date_time = (double) h->P.streamTime + o.time_start;
   u32 len = r.len > 512 ? 512 : r.len;
   u32 inl = len < 80 ? len : 80;
   memcpy(o.data, r.data, inl);
   if (len > 80)
   {
      if (r.ext != 0xFFFFFFFFu && (size_t) r.ext * 128 + (len - 80) <= extBytes)
         memcpy(o.data + 80, ext + (size_t) r.ext * 128, len - 80);
      else
         len = 80; // extension chunk missing (pool exhausted, reported by the caller): truncated payload
   }
   o.length = len;
   u32 padEnd = (len + 63u) & ~63u;
   if (padEnd > 512)
      padEnd = 512;
   if (padEnd > len)
      memset(o.data + len, 0, padEnd - len);
}

// packed records -> ABI frames on a few host threads (4e5 frames per batch): a record's payload continues in chunk
// r.ext - extBase of `ext`, its stream is r.lane + streamOffset
static void convert_records(const nfcb200_handle *h, const FrameRec *recs, uint64_t count, const unsigned char *ext, size_t extBytes, u32 extBase,
                            u32 streamOffset, u32 sampleRate, nfcb200_frame *out)
{
   parallel_for(count, 4096, [&](uint64_t lo, uint64_t hi) {
      for (uint64_t i = lo; i < hi; i++)
      {
         FrameRec r = recs[i];
         if (r.ext != 0xFFFFFFFFu)
            r.ext -= extBase;
         emit_frame(h, r, ext, extBytes, r.lane + streamOffset, sampleRate, out[i]);
      }
   });
}

// one device-resident chunk of a batch decode, and what its phases hand each other (streamBase: the stream index of its
// first stream in the call)
struct Chunk
{
   nfcb200_handle *h;
   nfcb200_handle::NfcBatch &B;
   cudaStream_t st;
   const void *samples;
   uint64_t n_samples;
   int sigtype;
   u32 n_streams, n_blocks, sample_rate, streamBase;
   bool exact;
   Trace tr;
   nfcb200_stats cs = {};           // the chunk's statistics, merged into the call's at the end
   Counters *dC = nullptr;          // 1: device counters
   const Carry *carryIn = nullptr;  // 1: the carry a single-stream decode continues from (nfcb200_set_carry, one shot), or null
   int useTma = 0;                  // 1: bulk copies allowed
   SegmentConfig sg;                // 1, 2: segment kernels' configuration
   u32 nLanes = 0, nSegs = 0;       // 2
   FramePool pool;                  // 4: the frames the lanes wrote
};

// the counts and times of one chunk into the call's statistics: sums, except rounds (the most any chunk needed)
static void merge_stats(nfcb200_stats &S, const nfcb200_stats &c)
{
   S.samples += c.samples;
   S.blocks += c.blocks;
   S.active_blocks += c.active_blocks;
   S.segments += c.segments;
   S.lanes += c.lanes;
   S.live_lanes += c.live_lanes;
   S.lane_runs += c.lane_runs;
   S.lane_samples += c.lane_samples;
   S.rounds = std::max(S.rounds, c.rounds);
   S.frames += c.frames;
   S.kernel_launches += c.kernel_launches;
   S.ms_screen += c.ms_screen;
   S.ms_segment += c.ms_segment;
   S.ms_lanes += c.ms_lanes;
   S.ms_gather += c.ms_gather;
   S.ms_front += c.ms_front;
   S.straggler_lanes += c.straggler_lanes;
   S.feature_samples += c.feature_samples;
}

// 1. screen, flag blocks, count segments
static int screen_phase(Chunk &c)
{
   auto &B = c.B;
   {
      int rc = B.counts.reserve((size_t) c.n_streams * sizeof(u32));
      rc = rc ? rc : B.offsets.reserve((size_t) c.n_streams * sizeof(u32));
      rc = rc ? rc : B.segCounts.reserve((size_t) c.n_streams * sizeof(u32));
      rc = rc ? rc : B.segOffsets.reserve((size_t) c.n_streams * sizeof(u32));
      rc = rc ? rc : B.counters.reserve(sizeof(Counters));
      rc = rc ? rc : B.carryDev.reserve(2 * sizeof(Carry) + 16);
      if (rc)
         return rc;
   }
   c.dC = B.counters.as<Counters>();
   if (!B.carryIn.empty() && c.n_streams == 1 && c.streamBase == 0)
   {
      CUDA_TRY(cudaMemcpyAsync(B.carryDev.ptr, B.carryIn.data(), sizeof(Carry), cudaMemcpyHostToDevice, c.st));
      c.carryIn = B.carryDev.as<Carry>();
   }

   if (int rc = screen(c.h, c.samples, c.sigtype, c.n_streams, c.n_samples, B.flags, B.bsum, c.st, c.useTma))
      return rc;
   cudaEventRecord(B.ev[EV_SCREENED], c.st);

   CUDA_TRY(cudaMemsetAsync(c.dC, 0, sizeof(Counters), c.st));
   CUDA_TRY(cudaMemsetAsync(B.counts.ptr, 0, (size_t) c.n_streams * sizeof(u32), c.st));
   c.sg = flag_blocks(c.h, B.flags, B.bsum, c.n_streams, c.n_samples, c.carryIn, &c.dC->activeBlocks, c.st);
   c.sg.counts = B.counts.as<u32>();
   c.sg.offsets = B.offsets.as<u32>();
   c.sg.segTotal = &c.dC->segTotal;
   c.sg.shortHalo = (u32) B.shortHalo;
   segment_starts_kernel<<<(u32) (((uint64_t) c.n_streams * c.n_blocks + 255) / 256), 256, 0, c.st>>>(c.sg);
   c.cs.kernel_launches += 4;
   CUDA_TRY(cudaGetLastError());
   return 0;
}

// 2. segments and lanes: grouping, the segment table and lane records of every stream, and the first-round queue
static int lanes_phase(Chunk &c)
{
   auto &B = c.B;
   u32 segTotal = 0;
   CUDA_TRY(cudaMemcpyAsync(&segTotal, &c.dC->segTotal, sizeof(u32), cudaMemcpyDeviceToHost, c.st));
   CUDA_TRY(cudaMemcpyAsync(B.segCounts.ptr, B.counts.ptr, (size_t) c.n_streams * sizeof(u32), cudaMemcpyDeviceToDevice, c.st));
   CUDA_TRY(cudaStreamSynchronize(c.st));
   // Segments per lane.  Exact mode: ONE warp lane decodes the whole stream -- the detectors' running sums carry their rounding
   // history (NfcA.cpp:246-250), which only a run over the whole capture reproduces bit for bit (nfc_wlane.h).  Throughput
   // mode: thread lanes, one per group of segments, cold-started sums (exact on 16-bit input), as many lanes as fill the
   // machine a few times over (every lane pays a warm-up halo; longer lanes keep more of the carry chain inside one sequential run).
   SegmentConfig &sg = c.sg;
   if (c.h->cfg.segments_per_lane)
      sg.group = c.h->cfg.segments_per_lane;
   else if (c.exact && c.sigtype == SIG_MAG_S16 && (uint64_t) c.n_streams < (uint64_t) c.h->smCount * (uint64_t) B.wlanesPerSm)
   {
      // 16-bit mono input adds exactly whatever the history of a running sum: a stream may be cut into several warp lanes
      // (cold starts + carry chain) without losing a bit -- small batches fill the machine that way
      const uint64_t resident = (uint64_t) c.h->smCount * (uint64_t) B.wlanesPerSm;
      sg.group = (u32) std::max<uint64_t>(1, segTotal / (resident * 2));
   }
   else if (c.exact)
      sg.group = 0xFFFFFFFFu; // one lane per stream
   else
   {
      const uint64_t residentLanes = (uint64_t) c.h->smCount * (uint64_t) B.laneBlocks * (LANE_THREADS / 32) * 32;
      sg.group = (u32) std::min<uint64_t>(64, std::max<uint64_t>(1, segTotal / std::max<uint64_t>(1, residentLanes * 2)));
   }
   if (sg.group > 1)
   {
      segment_group_kernel<<<(c.n_streams + 63) / 64, 64, 0, c.st>>>(sg);
      c.cs.kernel_launches++;
      CUDA_TRY(cudaGetLastError());
   }
   c.cs.segments = segTotal;
   c.tr.mark("screen + segments");

   std::vector<u32> counts(c.n_streams), offsets(c.n_streams), segCounts(c.n_streams), segOffsets(c.n_streams);
   CUDA_TRY(cudaMemcpyAsync(counts.data(), B.counts.ptr, c.n_streams * sizeof(u32), cudaMemcpyDeviceToHost, c.st));
   CUDA_TRY(cudaMemcpyAsync(segCounts.data(), B.segCounts.ptr, c.n_streams * sizeof(u32), cudaMemcpyDeviceToHost, c.st));
   CUDA_TRY(cudaStreamSynchronize(c.st));

   const uint64_t nLanes64 = std::accumulate(counts.begin(), counts.end(), 0ull), nSegs64 = std::accumulate(segCounts.begin(), segCounts.end(), 0ull);
   if (nLanes64 >= 0x7FFFFFFFull || nSegs64 >= 0x7FFFFFFFull)
      return fail(NFCB200_ERR_CAPACITY, "too many segments (%llu)", (unsigned long long) nSegs64);
   std::exclusive_scan(counts.begin(), counts.end(), offsets.begin(), 0u);
   std::exclusive_scan(segCounts.begin(), segCounts.end(), segOffsets.begin(), 0u);
   const u32 nLanes = c.nLanes = (u32) nLanes64;
   c.nSegs = (u32) nSegs64;
   c.cs.lanes = nLanes;

   {
      int rc = B.lanes.reserve((size_t) nLanes * sizeof(LaneRec));
      rc = rc ? rc : B.segs.reserve((size_t) std::max<u32>(c.nSegs, 1) * sizeof(SegRec));
      rc = rc ? rc : B.queue.reserve((size_t) nLanes * sizeof(u32));
      rc = rc ? rc : B.meta.reserve((size_t) (nLanes + 1) * sizeof(u32));
      if (rc)
         return rc;
   }

   CUDA_TRY(cudaMemcpyAsync(B.offsets.ptr, offsets.data(), c.n_streams * sizeof(u32), cudaMemcpyHostToDevice, c.st));
   CUDA_TRY(cudaMemcpyAsync(B.segOffsets.ptr, segOffsets.data(), c.n_streams * sizeof(u32), cudaMemcpyHostToDevice, c.st));
   sg.lanes = B.lanes.as<LaneRec>();
   sg.queue = B.queue.as<u32>();
   sg.segCounts = B.segCounts.as<u32>();
   sg.segOffsets = B.segOffsets.as<u32>();
   sg.segs = B.segs.as<SegRec>();
   sg.featTotal = &c.dC->featTotal;
   segment_fill_kernel<<<c.n_streams, 32, 0, c.st>>>(sg, c.h->P);
   c.cs.kernel_launches++;
   CUDA_TRY(cudaGetLastError());

   // first-round queue ordered by decreasing lane length (counting sort on the host: the lengths are 4 bytes per lane)
   if (!c.exact && nLanes > 64)
   {
      lane_length_kernel<<<(nLanes + 255) / 256, 256, 0, c.st>>>(B.lanes.as<LaneRec>(), nLanes, B.meta.as<u32>());
      c.cs.kernel_launches++;
      std::vector<u32> len(nLanes), order(nLanes);
      CUDA_TRY(cudaMemcpyAsync(len.data(), B.meta.ptr, (size_t) nLanes * sizeof(u32), cudaMemcpyDeviceToHost, c.st));
      CUDA_TRY(cudaStreamSynchronize(c.st));
      const u32 shift = 8, buckets = 1u << 16;
      std::vector<u32> hist(buckets + 1, 0);
      auto key = [&](u32 v) { u32 k = v >> shift; return k >= buckets ? 0u : buckets - 1 - k; }; // descending
      for (u32 i = 0; i < nLanes; i++)
         hist[key(len[i]) + 1]++;
      for (u32 b = 0; b < buckets; b++)
         hist[b + 1] += hist[b];
      for (u32 i = 0; i < nLanes; i++)
         order[hist[key(len[i])]++] = i;
      CUDA_TRY(cudaMemcpyAsync(B.queue.ptr, order.data(), (size_t) nLanes * sizeof(u32), cudaMemcpyHostToDevice, c.st));
      CUDA_TRY(cudaStreamSynchronize(c.st));
   }
   return 0;
}

// 3. front pass (exact mode): the sequential float recurrences of nextSample, one thread per segment -> feature pool
static int front_phase(Chunk &c)
{
   unsigned long long featTotal = 0;
   CUDA_TRY(cudaMemcpyAsync(&featTotal, &c.dC->featTotal, sizeof(featTotal), cudaMemcpyDeviceToHost, c.st));
   CUDA_TRY(cudaStreamSynchronize(c.st));
   if (int rc = c.B.feats.reserve((size_t) std::max<unsigned long long>(c.exact ? featTotal : 0, 1) * sizeof(float4)))
      return rc;
   c.cs.feature_samples = featTotal;
   cudaEventRecord(c.B.ev[EV_FRONT], c.st);
   if (c.nSegs && c.exact)
   {
      FrontConfig fc;
      fc.samples = c.samples;
      fc.n_samples = c.n_samples;
      fc.sigtype = c.sigtype;
      fc.segs = c.B.segs.as<SegRec>();
      fc.n_segs = c.nSegs;
      fc.pool = c.B.feats.as<float4>();
      launch_front(fc, c.h->P, c.st);
      c.cs.kernel_launches++;
      CUDA_TRY(cudaGetLastError());
   }
   return 0;
}

// one round of thread lanes; with the straggler hand-over on, `overrun` lanes gave up and ran again on warp lanes (`lc`)
static int thread_lanes(Chunk &c, u32 queueCount, WLaneConfig &lc, u32 &overrun)
{
   auto &B = c.B;
   const u32 warpsPerBlock = LANE_THREADS / 32;
   const u32 maxThreadWarps = (u32) c.h->smCount * (u32) B.laneBlocks * warpsPerBlock; // the kernel is persistent
   u32 warps = std::min(maxThreadWarps, (queueCount + 31) / 32);
   const u32 blocks = (warps + warpsPerBlock - 1) / warpsPerBlock;
   warps = blocks * warpsPerBlock;

   int rc = B.scratch.reserve((size_t) warps * NFCB200_SCRATCH_FLOATS * 32 * sizeof(float));
   rc = rc ? rc : B.sbuf.reserve((size_t) warps * 32 * 512);
   if (rc)
      return rc;

   LaneConfig tc;
   memset(&tc, 0, sizeof(tc));
   tc.samples = c.samples;
   tc.n_samples = c.n_samples;
   tc.sigtype = c.sigtype;
   tc.flags = B.flags.as<uint8_t>();
   tc.n_blocks = c.n_blocks;
   tc.lanes = B.lanes.as<LaneRec>();
   tc.n_lanes = c.nLanes;
   tc.queue = B.queue.as<u32>();
   tc.queue_count = queueCount;
   tc.cursor = &c.dC->cursor;
   tc.scratch = B.scratch.as<float>();
   tc.sbuf = B.sbuf.as<uint8_t>();
   tc.pool = c.pool;
   tc.work = &c.dC->work;
   tc.bail_margin = B.stragglerMargin;
   tc.bail_always = B.stragglerAlways ? 1u : 0u;
   tc.overrun = B.meta.as<u32>(); // free between the queue ordering and the gather
   tc.overrun_count = &c.dC->overrunCount;
   CUDA_TRY(cudaMemsetAsync(&c.dC->overrunCount, 0, sizeof(u32), c.st));
   overrun = 0;
   if (!tc.bail_margin)
   {
      lanes_kernel<false><<<blocks, LANE_THREADS, 0, c.st>>>(tc, c.h->P);
      return 0;
   }
   lanes_kernel<true><<<blocks, LANE_THREADS, 0, c.st>>>(tc, c.h->P);
   CUDA_TRY(cudaMemcpyAsync(&overrun, &c.dC->overrunCount, sizeof(u32), cudaMemcpyDeviceToHost, c.st));
   CUDA_TRY(cudaStreamSynchronize(c.st));
   c.tr.mark("  thread lanes");
   if (overrun)
   {
      // the stragglers again, each by a whole warp with its history in shared memory; without a feature pool the
      // warp lane runs the front end itself (SegRec::hasFeat is 0 in throughput mode)
      CUDA_TRY(cudaMemsetAsync(&c.dC->cursor, 0, sizeof(u32), c.st));
      lc.queue = B.meta.as<u32>();
      lc.queue_count = overrun;
      wlanes_kernel<<<std::min((u32) c.h->smCount * (u32) B.wlanesPerSm, overrun), 32, sizeof(WLaneSmem), c.st>>>(lc, c.h->P);
      c.cs.kernel_launches++;
      c.cs.lane_runs += overrun;
      if (c.tr.on)
      {
         cudaStreamSynchronize(c.st);
         char what[64];
         snprintf(what, sizeof(what), "  %u straggler(s) on warp lanes", overrun);
         c.tr.mark(what);
      }
   }
   return 0;
}

// 4. lanes and chain to the fixed point: each round runs the queued lanes, then the chain queues those whose carry changed
static int chain_phase(Chunk &c)
{
   auto &B = c.B;
   Counters *dC = c.dC;
   const u32 poolCap = (u32) std::min<uint64_t>(32u << 20, std::max<uint64_t>(1u << 16, (uint64_t) c.n_streams * c.n_samples / 512 + (uint64_t) c.nLanes * 8));
   if (int rc = frame_pool(B.pool, B.ext, poolCap, std::max<u32>(1u << 12, poolCap / 8), dC, c.pool))
      return rc;

   const u32 maxWarps = (u32) c.h->smCount * (u32) B.wlanesPerSm; // resident warp lanes: the kernel is persistent
   WLaneConfig lc;
   memset(&lc, 0, sizeof(lc));
   lc.samples = c.samples;
   lc.n_samples = c.n_samples;
   lc.sigtype = c.sigtype;
   lc.flags = B.flags.as<uint8_t>();
   lc.bsum = B.bsum.as<float>();
   lc.n_blocks = c.n_blocks;
   lc.lanes = B.lanes.as<LaneRec>();
   lc.queue = B.queue.as<u32>();
   lc.cursor = &dC->cursor;
   lc.segs = B.segs.as<SegRec>();
   lc.n_segs = c.nSegs;
   lc.pool = B.feats.as<float4>();
   lc.frames = c.pool;
   lc.work = &dC->work;
   lc.use_tma = c.useTma;
   lc.phase = dC->phase;

   ChainConfig cc;
   cc.carryIn = c.carryIn;
   cc.lanes = B.lanes.as<LaneRec>();
   cc.offsets = B.offsets.as<u32>();
   cc.counts = B.counts.as<u32>();
   cc.n_streams = c.n_streams;
   cc.queue = B.queue.as<u32>();
   cc.queue_count = &dC->queueCount;

   u32 queueCount = c.nLanes;
   const u32 maxRounds = c.h->cfg.max_rounds ? c.h->cfg.max_rounds : 4096;
   u32 rounds = 0;
   u32 stragglers = 0;
   while (queueCount > 0)
   {
      if (rounds >= maxRounds)
         return fail(NFCB200_ERR_CAPACITY, "carry chain did not converge in %u rounds", maxRounds);

      CUDA_TRY(cudaMemsetAsync(&dC->cursor, 0, sizeof(u32), c.st));
      if (c.exact)
      {
         lc.queue_count = queueCount;
         wlanes_kernel<<<std::min(maxWarps, queueCount), 32, sizeof(WLaneSmem), c.st>>>(lc, c.h->P);
      }
      else
      {
         u32 overrun = 0;
         if (int rc = thread_lanes(c, queueCount, lc, overrun))
            return rc;
         stragglers += overrun;
      }
      c.cs.kernel_launches++;
      CUDA_TRY(cudaGetLastError());

      c.cs.lane_runs += queueCount;
      rounds++;

      CUDA_TRY(cudaMemsetAsync(&dC->queueCount, 0, sizeof(u32), c.st));
      chain_warp_kernel<<<(c.n_streams + CHAIN_WARPS - 1) / CHAIN_WARPS, CHAIN_WARPS * 32, 0, c.st>>>(cc, c.h->P);
      c.cs.kernel_launches++;
      CUDA_TRY(cudaGetLastError());

      const u32 ran = queueCount;
      CUDA_TRY(cudaMemcpyAsync(&queueCount, &dC->queueCount, sizeof(u32), cudaMemcpyDeviceToHost, c.st));
      CUDA_TRY(cudaStreamSynchronize(c.st));
      if (c.tr.on)
      {
         char what[64];
         snprintf(what, sizeof(what), "  round %u: %u lanes", rounds, ran);
         c.tr.mark(what);
      }
   }

   c.cs.rounds = rounds;
   c.cs.straggler_lanes = (float) stragglers;
   c.tr.mark("lanes + chain");
   return 0;
}

// NFCB200_TRACE diagnostics of the lanes: how far they ran, the thread lanes' profile, where the warp lanes' cycles went
static void trace_lanes(Chunk &c, const Counters &hc)
{
   if (!c.tr.on)
      return;
   const u32 nLanes = c.nLanes;
   if (nLanes)
   {
      // the longest run bounds the lane kernel from below whatever the total work is
      if (c.B.scratch.reserve(65 * sizeof(unsigned long long)) == 0)
      {
         unsigned long long *dStat = (unsigned long long *) c.B.scratch.ptr;
         unsigned long long hs[65];
         cudaMemsetAsync(dStat, 0, sizeof(hs), c.st);
         lane_run_stat_kernel<<<(nLanes + 255) / 256, 256, 0, c.st>>>(c.B.lanes.as<LaneRec>(), nLanes, dStat);
         cudaMemcpyAsync(hs, dStat, sizeof(hs), cudaMemcpyDeviceToHost, c.st);
         cudaStreamSynchronize(c.st);
         LaneRec lr;
         const u32 li = (u32) (hs[64] & 0xFFFFFFFFu);
         cudaMemcpy(&lr, c.B.lanes.as<LaneRec>() + li, sizeof(LaneRec), cudaMemcpyDeviceToHost);
         fprintf(stderr, "[nfcb200] longest lane run: %llu samples (lane %u, stream %u, first %u begin %u end0 %u end %u stop %u, %u frames)\n[nfcb200] runs by length / 4096:",
                 hs[64] >> 32, li, lr.stream, lr.first, lr.begin, lr.end0, lr.end, lr.stop, lr.nframes);
         for (int b = 0; b < 64; b++)
            if (hs[b])
               fprintf(stderr, " %d:%llu", b, hs[b]);
         fprintf(stderr, "\n");
         c.tr.mark("(lane run statistics)");
      }
#if defined(NFCB200_LANE_PROFILE)
      {
         // where the thread lanes' warp steps and cycles went in this call (make DEFS=-DNFCB200_LANE_PROFILE)
         static const char *names[NFCB200_PROF_CLASSES] = {"gated", "search", "A poll", "A listen start", "A listen symbol", "other locked", "retire / skip"};
         unsigned long long hp[2 * NFCB200_PROF_CLASSES], zero[2 * NFCB200_PROF_CLASSES] = {};
         cudaMemcpyFromSymbol(hp, nfcb200_lane_prof, sizeof(hp));
         cudaMemcpyToSymbol(nfcb200_lane_prof, zero, sizeof(zero));
         unsigned long long steps = 0, cycles = 0;
         for (int i = 0; i < NFCB200_PROF_CLASSES; i++)
         {
            steps += hp[i];
            cycles += hp[NFCB200_PROF_CLASSES + i];
         }
         fprintf(stderr, "[nfcb200] lane profile: class | warp steps | share | cycles / warp step | share of cycles\n");
         for (int i = 0; i < NFCB200_PROF_CLASSES; i++)
            fprintf(stderr, "[nfcb200]   %-16s %14llu %6.2f%% %10.0f %6.2f%%\n", names[i], hp[i], steps ? 100.0 * hp[i] / steps : 0.0,
                    hp[i] ? (double) hp[NFCB200_PROF_CLASSES + i] / hp[i] : 0.0, cycles ? 100.0 * hp[NFCB200_PROF_CLASSES + i] / cycles : 0.0);
         fprintf(stderr, "[nfcb200]   %-16s %14llu %7s %10.0f\n", "total", steps, "", steps ? (double) cycles / steps : 0.0);
      }
#endif
   }
   if (c.exact || c.cs.straggler_lanes > 0)
   {
      static const char *names[8] = {"control", "fill", "search", "machine", "walk", "jump", "scalar", "locked"};
      unsigned long long tot = 0;
      for (int i = 0; i < 8; i++)
         tot += hc.phase[i];
      for (int i = 0; i < 8; i++)
         fprintf(stderr, "[nfcb200] lanes %-8s %5.1f %% of cycles, %12llu samples, %8.1f cycles / sample\n", names[i], 100.0 * hc.phase[i] / (double) (tot ? tot : 1),
                 hc.phase[8 + i], hc.phase[8 + i] ? (double) hc.phase[i] / (double) hc.phase[8 + i] : 0.0);
   }
}

// 5. gather: frames ordered and packed on the device after those of the call's earlier chunks, one copy to the host,
// conversion to out[outOffset ...) (bounded by cap)
static int gather_phase(Chunk &c, nfcb200_frame *out, uint64_t cap, uint64_t outOffset)
{
   auto &B = c.B;
   const u32 nLanes = c.nLanes;
   u32 *dLaneOff = B.meta.as<u32>(); // [nLanes + 1]
   frame_offsets_kernel<<<1, 1024, 0, c.st>>>(B.lanes.as<LaneRec>(), nLanes, dLaneOff, &c.dC->live);
   c.cs.kernel_launches++;
   CUDA_TRY(cudaGetLastError());

   Counters hc;
   u32 nf32 = 0;
   CUDA_TRY(cudaMemcpyAsync(&hc, c.dC, sizeof(Counters), cudaMemcpyDeviceToHost, c.st));
   CUDA_TRY(cudaMemcpyAsync(&nf32, dLaneOff + nLanes, sizeof(u32), cudaMemcpyDeviceToHost, c.st));
   CUDA_TRY(cudaStreamSynchronize(c.st));
   trace_lanes(c, hc);
   c.cs.lane_samples = hc.work;
   c.cs.live_lanes = hc.live;
   c.cs.active_blocks = hc.activeBlocks;

   if (hc.poolCount > c.pool.cap || hc.extCount > c.pool.extCap)
      return fail(NFCB200_ERR_CAPACITY, "frame pool exhausted (%u frames, %u extension chunks)", hc.poolCount, hc.extCount);

   const uint64_t nf = nf32;
   const u32 extBefore = B.packedExtCount;
   {
      int rc = B.packed.reserve_keep((size_t) (B.packedCount + nf) * sizeof(FrameRec), (size_t) B.packedCount * sizeof(FrameRec), c.st);
      rc = rc ? rc : B.packedExt.reserve_keep((size_t) (extBefore + hc.extCount + 1) * 128, (size_t) extBefore * 128, c.st);
      rc = rc ? rc : B.packCtr.reserve(sizeof(u32));
      if (rc)
         return rc;
   }
   const u32 packedExtCap = (u32) std::min<size_t>(B.packedExt.cap / 128, 0xFFFFFFFFu);
   CUDA_TRY(cudaMemcpyAsync(B.packCtr.ptr, &extBefore, sizeof(u32), cudaMemcpyHostToDevice, c.st));

   FrameRec *dPacked = B.packed.as<FrameRec>() + B.packedCount;
   if (hc.poolCount)
   {
      const u32 grid = std::min<u32>((hc.poolCount + 255) / 256, (u32) c.h->smCount * 8);
      frame_compact_kernel<<<grid, 256, 0, c.st>>>(B.pool.as<FrameRec>(), hc.poolCount, B.lanes.as<LaneRec>(), nLanes, dLaneOff, B.ext.as<u8>(), hc.extCount,
                                                    c.streamBase, dPacked, B.packedExt.as<u8>(), packedExtCap, B.packCtr.as<u32>());
      c.cs.kernel_launches++;
      CUDA_TRY(cudaGetLastError());
   }

   u32 extAfter = extBefore;
   CUDA_TRY(cudaMemcpyAsync(&extAfter, B.packCtr.ptr, sizeof(u32), cudaMemcpyDeviceToHost, c.st));
   CUDA_TRY(cudaStreamSynchronize(c.st));
   if (extAfter > packedExtCap)
      extAfter = packedExtCap;

   {
      int rc = B.hRecs.reserve((size_t) std::max<uint64_t>(nf, 1) * sizeof(FrameRec));
      rc = rc ? rc : B.hExt.reserve((size_t) std::max<u32>(extAfter - extBefore, 1) * 128);
      if (rc)
         return rc;
   }

   if (nf)
      CUDA_TRY(cudaMemcpyAsync(B.hRecs.ptr, dPacked, (size_t) nf * sizeof(FrameRec), cudaMemcpyDeviceToHost, c.st));
   if (extAfter > extBefore)
      CUDA_TRY(cudaMemcpyAsync(B.hExt.ptr, B.packedExt.as<u8>() + (size_t) extBefore * 128, (size_t) (extAfter - extBefore) * 128, cudaMemcpyDeviceToHost, c.st));

   cudaEventRecord(B.ev[EV_GATHERED], c.st);
   CUDA_TRY(cudaStreamSynchronize(c.st));
   c.tr.mark("frames d2h");

   B.packedCount += nf;
   B.packedExtCount = extAfter;

   const uint64_t count = outOffset >= cap ? 0 : std::min<uint64_t>(nf, cap - outOffset);
   if (count)
      convert_records(c.h, B.hRecs.as<FrameRec>(), count, B.hExt.as<unsigned char>(), (size_t) (extAfter - extBefore) * 128, extBefore, 0, c.sample_rate,
                      out + outOffset);
   c.tr.mark("emit");
   c.cs.frames = nf;
   return 0;
}

// decode one device-resident batch [n_streams][n_samples]; frames are written to out[outOffset ...) (bounded by cap) with
// stream indices offset by streamBase; statistics are ACCUMULATED into the call's
static int decode_resident(nfcb200_handle *h, const void *dSamples, int sigtype, uint32_t n_streams, uint64_t n_samples, uint32_t sample_rate,
                           uint32_t streamBase, nfcb200_frame *out, uint64_t cap, uint64_t outOffset, uint64_t *produced)
{
   auto &B = h->batch;
   Chunk c = {h, B, h->stream, dSamples, n_samples, sigtype, n_streams, (u32) ((n_samples + NFCB200_BLOCK - 1) / NFCB200_BLOCK), sample_rate,
              streamBase, h->cfg.exact != 0};
   c.cs.samples = (uint64_t) n_streams * n_samples;
   c.cs.blocks = (uint64_t) n_streams * c.n_blocks;
   cudaEventRecord(B.ev[EV_SCREEN], c.st);

   int rc = screen_phase(c);
   rc = rc ? rc : lanes_phase(c);
   rc = rc ? rc : front_phase(c);
   if (rc)
      return rc;
   c.tr.mark("lane fill + front pass");
   cudaEventRecord(B.ev[EV_LANES], c.st);
   if ((rc = chain_phase(c)))
      return rc;
   cudaEventRecord(B.ev[EV_GATHER], c.st);
   if ((rc = gather_phase(c, out, cap, outOffset)))
      return rc;
   *produced = c.cs.frames;

   B.lastStreams = n_streams;
   B.lastBlocks = c.n_blocks;
   B.lastLanes = n_streams == 1 ? c.nLanes : 0;
   B.lastCarryInUsed = c.carryIn != nullptr;
   if (c.carryIn)
      B.carryIn.clear(); // one shot

   cudaEventElapsedTime(&c.cs.ms_front, B.ev[EV_FRONT], B.ev[EV_LANES]);
   cudaEventElapsedTime(&c.cs.ms_screen, B.ev[EV_SCREEN], B.ev[EV_SCREENED]);
   cudaEventElapsedTime(&c.cs.ms_segment, B.ev[EV_SCREENED], B.ev[EV_LANES]); // the front pass included
   cudaEventElapsedTime(&c.cs.ms_lanes, B.ev[EV_LANES], B.ev[EV_GATHER]);
   cudaEventElapsedTime(&c.cs.ms_gather, B.ev[EV_GATHER], B.ev[EV_GATHERED]);
   merge_stats(B.stats, c.cs);
   return 0;
}

// decode the retained buffer up to its end (the stream's end when `flush`): its frames go onto the pending list, where what
// does not fit the caller's buffer waits for the next call; `hs` returns the lane's state
static int stream_decode(nfcb200_handle *h, bool flush, StreamState &hs)
{
   auto &S = h->strm;
   cudaStream_t st = h->stream;
   // the buffer always starts on a block boundary, so buffer block i is absolute block base / 256 + i
   const u32 n_blocks = (S.count + NFCB200_BLOCK - 1) / NFCB200_BLOCK;
   if (S.count)
   {
      int useTma = 0;
      if (int rc = screen(h, S.samples.ptr, S.sig, 1, S.count, S.flags, S.bsum, st, useTma))
         return rc;
      // note: the stream-start margin of blocks_activate applies to buffer block 0; at the true stream start that is
      // exactly the reference start, later it only makes a few retained blocks active (harmless)
      flag_blocks(h, S.flags, S.bsum, 1, S.count, nullptr, nullptr, st);
      CUDA_TRY(cudaGetLastError());
   }

   // frame pool for this push
   Counters *dC = S.counters.as<Counters>();
   StreamConfig cfg;
   memset(&cfg, 0, sizeof(cfg));
   if (int rc = frame_pool(S.pool, S.ext, 1u << 14, 1u << 12, dC, cfg.pool))
      return rc;
   CUDA_TRY(cudaMemsetAsync(dC, 0, sizeof(Counters), st));

   cfg.samples = S.samples.ptr;
   cfg.base = S.base;
   cfg.count = S.count;
   cfg.sigtype = S.sig;
   cfg.flags = S.flags.as<uint8_t>();
   cfg.flagBase = S.base / NFCB200_BLOCK;
   cfg.flagCount = n_blocks;
   cfg.limit = S.base + S.count;
   cfg.final = flush ? 1 : 0;
   cfg.state = S.state.as<StreamState>();
   cfg.scratch = S.scratch.as<float>();
   cfg.sbuf = S.sbuf.as<uint8_t>();

   stream_kernel<<<1, 32, 0, st>>>(cfg, h->P);
   CUDA_TRY(cudaGetLastError());

   Counters hc;
   CUDA_TRY(cudaMemcpyAsync(&hc, dC, sizeof(Counters), cudaMemcpyDeviceToHost, st));
   CUDA_TRY(cudaMemcpyAsync(&hs, S.state.ptr, sizeof(StreamState), cudaMemcpyDeviceToHost, st));
   CUDA_TRY(cudaStreamSynchronize(st));

   if (hc.poolCount > cfg.pool.cap || hc.extCount > cfg.pool.extCap)
      return fail(NFCB200_ERR_CAPACITY, "stream frame pool exhausted");

   std::vector<FrameRec> recs(hc.poolCount);
   std::vector<unsigned char> ext((size_t) hc.extCount * 128);
   if (hc.poolCount)
      CUDA_TRY(cudaMemcpy(recs.data(), S.pool.ptr, (size_t) hc.poolCount * sizeof(FrameRec), cudaMemcpyDeviceToHost));
   if (hc.extCount)
      CUDA_TRY(cudaMemcpy(ext.data(), S.ext.ptr, ext.size(), cudaMemcpyDeviceToHost));

   std::sort(recs.begin(), recs.end(), [](const FrameRec &a, const FrameRec &b) { return a.seq < b.seq; });

   for (const FrameRec &r: recs)
   {
      S.pending.emplace_back();
      emit_frame(h, r, ext.data(), ext.size(), 0, S.rate, S.pending.back());
   }

   if (flush)
   {
      // nextFrames({}): one carrier frame at the current clock (NfcDecoder.cpp:449-463)
      u32 clock = hs.pos - 1;
      bool on = hs.running ? hs.L.c.carrierOn != 0 : hs.carry.carrierOn != 0;
      S.pending.emplace_back();
      nfcb200_frame &o = S.pending.back();
      memset(&o, 0, sizeof(o));
      o.tech_type = TT_Any;
      o.frame_type = on ? FT_CarrierOn : FT_CarrierOff;
      o.frame_phase = PH_Carrier;
      o.sample_start = o.sample_end = clock;
      o.sample_rate = S.rate;
      o.time_start = o.time_end = (double) clock / (double) S.rate;
      o.date_time = (double) h->P.streamTime + o.time_start;
   }
   return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------------------------------
extern "C" {

const char *nfcb200_last_error(void)
{
   return g_error;
}

const char *nfcb200_version(void)
{
   return "nfcb200 0.1 sm_90a";
}

void nfcb200_config_default(nfcb200_config *cfg)
{
   memset(cfg, 0, sizeof(*cfg));
   Params P;
   params_defaults(&P);
   cfg->device = 0;
   cfg->enabled = P.enabled;
   cfg->power_level_threshold = P.power;
   for (int t = 0; t < 4; t++)
   {
      cfg->correlation_threshold[t] = P.thr[t].corr;
      cfg->modulation_min[t] = P.thr[t].modMin;
      cfg->modulation_max[t] = P.thr[t].modMax;
   }
   cfg->stream_time = 0;
   cfg->use_tma = 1;
   cfg->max_rounds = 0;
}

int nfcb200_create(const nfcb200_config *cfg, nfcb200_handle **out)
{
   if (!out)
      return fail(NFCB200_ERR_INVALID, "null output handle");

   *out = nullptr;

   int count = 0;
   cudaError_t e = cudaGetDeviceCount(&count);
   if (e != cudaSuccess || count == 0)
      return fail(NFCB200_ERR_NO_DEVICE, "no CUDA device available (%s): this library has no CPU path", e == cudaSuccess ? "0 devices" : cudaGetErrorString(e));

   nfcb200_config c;
   if (cfg)
      c = *cfg;
   else
      nfcb200_config_default(&c);

   if (c.device < 0 || c.device >= count)
      return fail(NFCB200_ERR_INVALID, "device %d out of range (0..%d)", c.device, count - 1);

   CUDA_TRY(cudaSetDevice(c.device));

   // Host threads SLEEP while they wait for the device (the default is to spin).  A decode waits ~0.2 s per batch on a
   // stream; with one process per GPU and a CPU quota shared by all of them (16 cores for 8 ranks on this pool) spinning
   // waiters exhaust the quota and the whole cgroup is throttled for tens of milliseconds at arbitrary points -- measured
   // as 50-125 ms stalls inside trivial host code at 2 GPUs, and as the 0.59 weak-scaling efficiency of round 1 at 4 / 8.
   cudaSetDeviceFlags(cudaDeviceScheduleBlockingSync);
   cudaGetLastError(); // older runtimes refuse to change the flags of an initialised context: not fatal

   nfcb200_handle *h = new nfcb200_handle();
   h->cfg = c;
   h->device = c.device;

   cudaDeviceProp prop;
   if (cudaGetDeviceProperties(&prop, c.device) == cudaSuccess)
      h->smCount = prop.multiProcessorCount;

   e = cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking);
   if (e != cudaSuccess)
   {
      delete h;
      return fail(NFCB200_ERR_CUDA, "cudaStreamCreate failed: %s", cudaGetErrorString(e));
   }

   for (auto &ev: h->batch.ev)
      cudaEventCreate(&ev);

   if (const char *e = getenv("NFCB200_HALO_SHORT"))
      h->batch.shortHalo = atoi(e) ? 1 : 0;
   if (const char *e = getenv("NFCB200_STRAGGLER"))
   {
      // N > 0: margin in samples; 0: off; N < 0 (tests): margin |N|, and a lane gives up whether the queue is empty or not
      const int v = atoi(e);
      h->batch.stragglerMargin = (u32) (v < 0 ? -v : v);
      h->batch.stragglerAlways = v < 0;
   }
#define NFCB200_SMEM_ATTR(K) cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) sizeof(ScreenSmem))
   NFCB200_SMEM_ATTR((screen_kernel<SIG_IQ_F32, false>));
   NFCB200_SMEM_ATTR((screen_kernel<SIG_MAG_F32, false>));
   NFCB200_SMEM_ATTR((screen_kernel<SIG_MAG_S16, false>));
   NFCB200_SMEM_ATTR((screen_kernel<SIG_IQ_S16, false>));
#undef NFCB200_SMEM_ATTR
   cudaFuncSetAttribute(wlanes_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) sizeof(WLaneSmem));
   {
      // resident warp lanes per SM: what the shared memory of one SM holds
      int perSm = 0;
      if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, wlanes_kernel, 32, sizeof(WLaneSmem)) == cudaSuccess && perSm > 0)
         h->batch.wlanesPerSm = perSm;
   }
   {
      // the persistent thread-lane grid and its scratch are sized from laneBlocks: never more blocks than fit (registers,
      // and the shared memory of the Front array plus the tap stages)
      int plain = 0, bail = 0;
      if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&plain, lanes_kernel<false>, LANE_THREADS, 0) == cudaSuccess &&
          cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bail, lanes_kernel<true>, LANE_THREADS, 0) == cudaSuccess)
      {
         const int fit = std::min(plain, bail);
         if (fit > 0 && fit < h->batch.laneBlocks)
         {
            fprintf(stderr, "nfcb200: only %d thread-lane blocks fit per SM (expected %d)\n", fit, h->batch.laneBlocks);
            h->batch.laneBlocks = fit;
         }
      }
   }

   *out = h;
   return 0;
}

void nfcb200_destroy(nfcb200_handle *h)
{
   if (!h)
      return;
   cudaSetDevice(h->device);
   cudaStreamSynchronize(h->stream);
#if defined(NFCB200_CHECK_TAPS)
   {
      // totals of the device so far (make DEFS=-DNFCB200_CHECK_TAPS): staged ring taps used, and those that differed from
      // the ring word they stand for (must be 0)
      unsigned long long used = 0, differ = 0, kind[8] = {};
      cudaMemcpyFromSymbol(&used, nfcb200_taps_used, sizeof(used));
      cudaMemcpyFromSymbol(&differ, nfcb200_taps_differ, sizeof(differ));
      cudaMemcpyFromSymbol(kind, nfcb200_taps_kind, sizeof(kind));
      fprintf(stderr, "nfcb200 taps check: %llu staged taps used (search %llu, A poll %llu, A listen %llu), %llu differ\n", used, kind[1],
              kind[2] + kind[3] + kind[4], kind[5] + kind[6] + kind[7], differ);
   }
#endif
   for (cudaEvent_t ev: h->batch.ev)
      if (ev)
         cudaEventDestroy(ev);
   for (cudaEvent_t ev: h->batch.copied)
      if (ev)
         cudaEventDestroy(ev);
   if (h->batch.copyStream)
      cudaStreamDestroy(h->batch.copyStream);
   if (h->stream)
      cudaStreamDestroy(h->stream);
   delete h; // the buffers free themselves
}

int nfcb200_configure(nfcb200_handle *h, const nfcb200_config *cfg)
{
   if (!h || !cfg)
      return fail(NFCB200_ERR_INVALID, "null argument");
   if (cfg->device != h->device)
      return fail(NFCB200_ERR_INVALID, "the device of a handle cannot change");
   h->cfg = *cfg;
   h->paramsRate = 0; // parameters are re-derived at the next decode (NfcDecoder::initialize)
   return 0;
}

int nfcb200_get_stats(nfcb200_handle *h, nfcb200_stats *stats)
{
   if (!h || !stats)
      return fail(NFCB200_ERR_INVALID, "null argument");
   *stats = h->batch.stats;
   return 0;
}

int nfcb200_get_block_flags(nfcb200_handle *h, uint8_t *out, uint64_t cap, uint64_t *n_blocks_per_stream)
{
   if (!h)
      return fail(NFCB200_ERR_INVALID, "null handle");
   if (n_blocks_per_stream)
      *n_blocks_per_stream = h->batch.lastBlocks;
   uint64_t total = (uint64_t) h->batch.lastStreams * h->batch.lastBlocks;
   if (!out)
      return 0;
   if (cap < total)
      return fail(NFCB200_ERR_CAPACITY, "flag buffer too small: need %llu bytes", (unsigned long long) total);
   CUDA_TRY(cudaSetDevice(h->device));
   CUDA_TRY(cudaMemcpy(out, h->batch.flags.ptr, total, cudaMemcpyDeviceToHost));
   return 0;
}

int nfcb200_decode_batch(nfcb200_handle *h, const void *samples, int samples_on_device, int sigtype, uint32_t n_streams, uint64_t n_samples,
                         uint32_t sample_rate, nfcb200_frame *out, uint64_t cap, uint64_t *n_out)
{

   if (!h)
      return fail(NFCB200_ERR_INVALID, "null handle");
   if (n_out)
      *n_out = 0;
   if (sigtype < SIG_IQ_F32 || sigtype > SIG_IQ_S16)
      return fail(NFCB200_ERR_INVALID, "unknown signal type %d", sigtype);
   if (!samples || n_streams == 0 || n_samples == 0)
      return fail(NFCB200_ERR_INVALID, "empty batch");
   if (n_samples >= 0xFFFF0000ull)
      return fail(NFCB200_ERR_UNSUPPORTED, "streams of 2^32 samples or more exceed the 32-bit sample clock of the frame format (NfcTech.h:338)");
   if (cap && !out)
      return fail(NFCB200_ERR_INVALID, "null frame buffer");

   CUDA_TRY(cudaSetDevice(h->device));

   if (h->paramsRate != sample_rate)
   {
      int rc = setup_params(h, sample_rate);
      if (rc)
         return rc;
   }

   auto &B = h->batch;
   cudaStream_t st = h->stream;
   const u32 bs = sig_bytes(sigtype);
   const uint64_t total = (uint64_t) n_streams * n_samples;

   memset(&B.stats, 0, sizeof(B.stats));
   B.packedCount = 0;      // the packed frames of a call: every chunk of this call appends
   B.packedExtCount = 0;
   nfcb200_stats &S = B.stats;
   Trace wall;

   cudaEventRecord(B.ev[EV_CALL], st);

   uint64_t nf = 0;

   if (samples_on_device)
   {
      int rc = decode_resident(h, samples, sigtype, n_streams, n_samples, sample_rate, 0, out, cap, 0, &nf);
      if (rc)
         return rc;
   }
   else
   {
      // host input: the batch is cut into stream chunks and the copy of chunk i + 1 (second CUDA stream, double-buffered
      // device staging) overlaps the decode of chunk i, so that a large batch runs at the host link's speed
      const uint64_t streamBytes = n_samples * bs;
      uint32_t chunkStreams = n_streams;
      if (total * bs > (1ull << 30) && n_streams >= 16)
      {
         // 16 chunks (8 below 4 GB): only the first copy and the last decode are not overlapped
         const uint32_t parts = total * bs > (4ull << 30) && n_streams >= 64 ? 16 : 8;
         chunkStreams = (n_streams + parts - 1) / parts;
         while (chunkStreams > 1 && (uint64_t) chunkStreams * streamBytes > (12ull << 30))
            chunkStreams = (chunkStreams + 1) / 2;
      }
      const uint64_t chunkBytes = (((uint64_t) chunkStreams * streamBytes) + 255) & ~255ull;
      const uint32_t nChunks = (n_streams + chunkStreams - 1) / chunkStreams;

      int rc = B.samples.reserve((nChunks > 1 ? 2 : 1) * chunkBytes + 64);
      if (rc)
         return rc;

      if (!B.copyStream)
      {
         CUDA_TRY(cudaStreamCreateWithFlags(&B.copyStream, cudaStreamNonBlocking));
         CUDA_TRY(cudaEventCreateWithFlags(&B.copied[0], cudaEventDisableTiming));
         CUDA_TRY(cudaEventCreateWithFlags(&B.copied[1], cudaEventDisableTiming));
      }

      auto issue = [&](uint32_t c) -> cudaError_t {
         const uint32_t s0 = c * chunkStreams;
         const uint32_t sc = std::min(chunkStreams, n_streams - s0);
         unsigned char *dst = B.samples.as<unsigned char>() + (c & 1) * chunkBytes;
         cudaError_t e = cudaMemcpyAsync(dst, (const unsigned char *) samples + (uint64_t) s0 * streamBytes, (uint64_t) sc * streamBytes, cudaMemcpyHostToDevice,
                                         B.copyStream);
         if (e != cudaSuccess)
            return e;
         return cudaEventRecord(B.copied[c & 1], B.copyStream);
      };

      CUDA_TRY(issue(0));

      float msCopyWait = 0;

      for (uint32_t c = 0; c < nChunks; c++)
      {
         const uint32_t s0 = c * chunkStreams;
         const uint32_t sc = std::min(chunkStreams, n_streams - s0);

         cudaEventRecord(B.ev[EV_COPY_WAIT], st);
         CUDA_TRY(cudaStreamWaitEvent(st, B.copied[c & 1], 0));
         cudaEventRecord(B.ev[EV_COPIED], st);

         // the other staging buffer is free (its decode returned): start the next copy before decoding this chunk
         if (c + 1 < nChunks)
            CUDA_TRY(issue(c + 1));

         uint64_t got = 0;
         rc = decode_resident(h, B.samples.as<unsigned char>() + (c & 1) * chunkBytes, sigtype, sc, n_samples, sample_rate, s0, out, cap, nf, &got);
         if (rc)
         {
            cudaStreamSynchronize(B.copyStream); // the next chunk's copy still reads the caller's buffer
            return rc;
         }
         nf += got;

         float w = 0;
         cudaEventElapsedTime(&w, B.ev[EV_COPY_WAIT], B.ev[EV_COPIED]);
         msCopyWait += w;
      }

      S.ms_h2d = msCopyWait; // time the decode stream spent waiting for input
   }

   cudaEventRecord(B.ev[EV_END], st);
   CUDA_TRY(cudaStreamSynchronize(st));
   cudaEventElapsedTime(&S.ms_total, B.ev[EV_CALL], B.ev[EV_END]);
   S.ms_wall = (float) wall.ms();

   if (n_out)
      *n_out = nf;

   if (nf > cap)
      return fail(NFCB200_ERR_CAPACITY, "%llu frames decoded but room for %llu only", (unsigned long long) nf, (unsigned long long) cap);

   return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// multi-GPU frame gather without a host round trip: the frames of the last decode, ordered and packed, as they sit in
// device memory (128-byte records + 128-byte payload extension chunks), and the conversion of such records to ABI frames
// ---------------------------------------------------------------------------------------------------------------------
/*
 * Time shards of ONE long capture (BASELINE.json configs[4], dist.decode_long_capture): a shard that does not start at the
 * capture's first sample continues its predecessor's decoder.  nfcb200_carry_before returns, after a single-stream decode,
 * the carry in front of the first lane that begins at or after `sample` (and that lane's begin: an idle point of the
 * capture); nfcb200_set_carry hands it to the next single-stream decode of this handle (one shot), with clock_shift
 * subtracted from the absolute sample times inside (the next window counts from its own first sample).  The blob is
 * opaque (a `Carry`, nfc_core.h): protocol state (FSD / FWT / SFGT, the Encrypted flag, lastCommand), carrier flags, the
 * carrier edge time.  Running sums and front-end state are not part of it: they re-converge over the window's overlap.
 */
int nfcb200_carry_size(void)
{
   return (int) sizeof(Carry);
}

int nfcb200_default_carry(nfcb200_handle *h, void *blob, uint64_t cap)
{
   if (!h || !blob || cap < sizeof(Carry))
      return fail(NFCB200_ERR_INVALID, "carry blob needs %zu bytes", sizeof(Carry));
   if (!h->paramsRate)
      return fail(NFCB200_ERR_INVALID, "no decode yet: the protocol defaults depend on the sample rate");
   Carry c;
   carry_speculate(c, h->P);
   memcpy(blob, &c, sizeof(Carry));
   return 0;
}

int nfcb200_set_carry(nfcb200_handle *h, const void *blob, uint64_t size, uint32_t clock_shift)
{
   if (!h)
      return fail(NFCB200_ERR_INVALID, "null handle");
   std::vector<unsigned char> &carry = h->batch.carryIn;
   if (!blob || size == 0)
   {
      carry.clear();
      return 0;
   }
   if (size != sizeof(Carry))
      return fail(NFCB200_ERR_INVALID, "carry blob of %llu bytes, expected %zu", (unsigned long long) size, sizeof(Carry));
   carry.assign((const unsigned char *) blob, (const unsigned char *) blob + sizeof(Carry));
   Carry &c = *(Carry *) carry.data();
   carry_canon(c);
   if (c.edgeTime)
      c.edgeTime = c.edgeTime > clock_shift ? c.edgeTime - clock_shift : 1;
   return 0;
}

int nfcb200_carry_before(nfcb200_handle *h, uint64_t sample, void *blob, uint64_t cap, uint64_t *size, uint64_t *lane_begin)
{
   if (!h)
      return fail(NFCB200_ERR_INVALID, "null handle");
   if (size)
      *size = sizeof(Carry);
   if (!blob || cap < sizeof(Carry))
      return fail(NFCB200_ERR_CAPACITY, "carry blob needs %zu bytes", sizeof(Carry));
   if (h->batch.lastStreams != 1)
      return fail(NFCB200_ERR_INVALID, "the carry query needs a single-stream decode before it");
   CUDA_TRY(cudaSetDevice(h->device));
   cudaStream_t st = h->stream;
   Carry *dOut = h->batch.carryDev.as<Carry>() + 1;
   u32 *dBegin = (u32 *) (h->batch.carryDev.as<Carry>() + 2);
   carry_before_kernel<<<1, 32, 0, st>>>(h->batch.lanes.as<LaneRec>(), h->batch.lastLanes, h->batch.lastCarryInUsed ? h->batch.carryDev.as<Carry>() : nullptr,
                                          (u32) std::min<uint64_t>(sample, 0xFFFFFFFFull), dOut, dBegin, h->P);
   CUDA_TRY(cudaGetLastError());
   u32 b = 0;
   CUDA_TRY(cudaMemcpyAsync(blob, dOut, sizeof(Carry), cudaMemcpyDeviceToHost, st));
   CUDA_TRY(cudaMemcpyAsync(&b, dBegin, sizeof(u32), cudaMemcpyDeviceToHost, st));
   CUDA_TRY(cudaStreamSynchronize(st));
   if (lane_begin)
      *lane_begin = b == 0xFFFFFFFFu ? ~0ull : b;
   return 0;
}

int nfcb200_device_frames(nfcb200_handle *h, const void **records, uint64_t *n_records, const void **ext, uint64_t *n_ext_chunks)
{
   if (!h)
      return fail(NFCB200_ERR_INVALID, "null handle");
   if (records)
      *records = h->batch.packed.ptr;
   if (n_records)
      *n_records = h->batch.packedCount;
   if (ext)
      *ext = h->batch.packedExt.ptr;
   if (n_ext_chunks)
      *n_ext_chunks = h->batch.packedExtCount;
   return 0;
}

int nfcb200_emit_records(nfcb200_handle *h, const void *records, uint64_t n_records, const void *ext, uint64_t n_ext_chunks, uint32_t stream_offset,
                         uint32_t sample_rate, nfcb200_frame *out, uint64_t cap, uint64_t *n_out)
{
   if (!h)
      return fail(NFCB200_ERR_INVALID, "null handle");
   if (n_out)
      *n_out = n_records;
   if (n_records > cap)
      return fail(NFCB200_ERR_CAPACITY, "%llu records but room for %llu frames", (unsigned long long) n_records, (unsigned long long) cap);
   if (n_records && (!records || !out))
      return fail(NFCB200_ERR_INVALID, "null buffer");
   convert_records(h, (const FrameRec *) records, n_records, (const unsigned char *) ext, (size_t) n_ext_chunks * 128, 0, stream_offset, sample_rate, out);
   return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// wire format of the host-side frame gather (gloo / CPU tests): [u64 count][count x 80-byte headers][payloads back to back]
// ---------------------------------------------------------------------------------------------------------------------
int nfcb200_pack_frames(const nfcb200_frame *frames, uint64_t n, uint32_t stream_offset, uint8_t *out, uint64_t cap, uint64_t *n_bytes)
{
   if (n && !frames)
      return fail(NFCB200_ERR_INVALID, "null frames");
   const size_t headBytes = offsetof(nfcb200_frame, data);

   std::vector<uint64_t> offs(n + 1);
   uint64_t payload = 0;
   for (uint64_t i = 0; i < n; i++)
   {
      offs[i] = payload;
      payload += frames[i].length > 512 ? 512 : frames[i].length;
   }
   offs[n] = payload;

   const uint64_t need = 8 + n * headBytes + payload;
   if (n_bytes)
      *n_bytes = need;
   if (!out)
      return 0;
   if (cap < need)
      return fail(NFCB200_ERR_CAPACITY, "%llu bytes needed, room for %llu", (unsigned long long) need, (unsigned long long) cap);

   memcpy(out, &n, 8);
   uint8_t *head = out + 8;
   uint8_t *pay = head + n * headBytes;

   parallel_for(n, 8192, [&](uint64_t lo, uint64_t hi) {
      for (uint64_t i = lo; i < hi; i++)
      {
         memcpy(head + i * headBytes, &frames[i], headBytes);
         uint32_t stream = frames[i].stream + stream_offset;
         memcpy(head + i * headBytes, &stream, 4);
         memcpy(pay + offs[i], frames[i].data, offs[i + 1] - offs[i]);
      }
   });
   return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// streaming
// ---------------------------------------------------------------------------------------------------------------------
int nfcb200_stream_reset(nfcb200_handle *h)
{
   if (!h)
      return fail(NFCB200_ERR_INVALID, "null handle");
   auto &S = h->strm;
   S.init = false;
   S.base = 0;
   S.count = 0;
   S.hostTail.clear();
   S.pending.clear();
   return 0;
}

int nfcb200_stream_pending(nfcb200_handle *h, nfcb200_frame *out, uint64_t cap, uint64_t *n_out, uint64_t *n_left)
{
   if (!h)
      return fail(NFCB200_ERR_INVALID, "null handle");
   auto &S = h->strm;
   const uint64_t deliver = std::min<uint64_t>(S.pending.size(), out ? cap : 0);
   for (uint64_t i = 0; i < deliver; i++)
      out[i] = S.pending[i];
   S.pending.erase(S.pending.begin(), S.pending.begin() + (size_t) deliver);
   if (n_out)
      *n_out = deliver;
   if (n_left)
      *n_left = S.pending.size();
   return 0;
}

int nfcb200_stream_push(nfcb200_handle *h, const void *samples, int sigtype, uint64_t n, uint32_t sample_rate, nfcb200_frame *out, uint64_t cap,
                        uint64_t *n_out)
{
   if (!h)
      return fail(NFCB200_ERR_INVALID, "null handle");
   if (n_out)
      *n_out = 0;
   if (n && (sigtype < SIG_IQ_F32 || sigtype > SIG_IQ_S16))
      return fail(NFCB200_ERR_INVALID, "unknown signal type %d", sigtype);
   if (n && !samples)
      return fail(NFCB200_ERR_INVALID, "null samples");
   if (n > (1u << 28))
      return fail(NFCB200_ERR_INVALID, "push of more than 2^28 samples: use nfcb200_decode_batch");

   CUDA_TRY(cudaSetDevice(h->device));
   cudaStream_t st = h->stream;
   auto &S = h->strm;

   const bool flush = n == 0;

   if (flush && !S.init)
   {
      // nextFrames({}) on a decoder that never saw a sample: one carrier-off frame at clock -1 (NfcDecoder.cpp:449-463)
      if (cap < 1)
         return fail(NFCB200_ERR_CAPACITY, "room for the flush frame needed");
      memset(&out[0], 0, sizeof(nfcb200_frame));
      out[0].tech_type = TT_Any;
      out[0].frame_type = FT_CarrierOff;
      out[0].frame_phase = PH_Carrier;
      out[0].sample_start = out[0].sample_end = 0xFFFFFFFFull;
      // the reference divides that clock by its sample rate, still 0: the times are +inf like its frame's
      out[0].time_start = out[0].time_end = (double) out[0].sample_start / (double) out[0].sample_rate;
      out[0].date_time = (double) h->cfg.stream_time + out[0].time_start;
      if (n_out)
         *n_out = 1;
      return 0;
   }

   // a sample-rate (or format) change re-initialises the decoder (NfcDecoder.cpp:383-388)
   if (!flush && (!S.init || S.rate != sample_rate || S.sig != sigtype))
   {
      nfcb200_stream_reset(h);
      int rc = 0;
      if (h->paramsRate != sample_rate)
         rc = setup_params(h, sample_rate);
      if (rc)
         return rc;

      rc = S.state.reserve(sizeof(StreamState));
      rc = rc ? rc : S.scratch.reserve(NFCB200_SCRATCH_FLOATS * sizeof(float));
      rc = rc ? rc : S.sbuf.reserve(512);
      rc = rc ? rc : S.counters.reserve(sizeof(Counters));
      if (rc)
         return rc;

      StreamState init;
      memset(&init, 0, sizeof(init));
      carry_init(init.carry, h->P);
      carry_canon(init.carry);
      CUDA_TRY(cudaMemcpyAsync(S.state.ptr, &init, sizeof(init), cudaMemcpyHostToDevice, st));
      CUDA_TRY(cudaMemsetAsync(S.scratch.ptr, 0, NFCB200_SCRATCH_FLOATS * sizeof(float), st));
      CUDA_TRY(cudaStreamSynchronize(st));

      S.rate = sample_rate;
      S.sig = sigtype;
      S.init = true;
   }
   else if (h->paramsRate != S.rate)
   {
      int rc = setup_params(h, S.rate);
      if (rc)
         return rc;
   }

   const u32 bs = sig_bytes(S.sig);

   // The streaming lane keeps absolute sample positions in 32 bits like the reference's signalClock (NfcTech.h:338).  The
   // reference wraps silently after 2^32 samples (7 minutes at 10 MS/s); here the position space must not wrap (retention and
   // the flag window are indexed by it), so the stream refuses further samples with an explicit error instead of stalling.
   if ((uint64_t) S.base + S.count + n >= 0xFFFF0000ull)
      return fail(NFCB200_ERR_UNSUPPORTED, "stream position would pass 2^32 samples: call nfcb200_stream_reset (the reference's 32-bit sample clock wraps here)");

   // retained host-side tail + new samples -> device buffer covering absolute samples [base, base + count + n); the host
   // copy stays for the next retention step
   const u32 newCount = S.count + (u32) n;
   if (int rc = S.samples.reserve((size_t) newCount * bs + 64))
      return rc;
   S.hostTail.insert(S.hostTail.end(), (const unsigned char *) samples, (const unsigned char *) samples + (size_t) n * bs);
   S.count = newCount;
   if (newCount)
      CUDA_TRY(cudaMemcpyAsync(S.samples.ptr, S.hostTail.data(), (size_t) newCount * bs, cudaMemcpyHostToDevice, st));

      StreamState hs;
   if (int rc = stream_decode(h, flush, hs))
      return rc;

   const uint64_t nf = S.pending.size();
   uint64_t deliver = 0;
   nfcb200_stream_pending(h, out, cap, &deliver, nullptr);

   // retention: keep what the parked / running lane can still need.  A running lane only reads forward (its history is in
   // its rings); a parked lane may cold start HALO samples before a later active block or be resumed at pos.
   {
      u32 keepFrom = hs.pos > NFCB200_HALO + 2 * NFCB200_BLOCK ? hs.pos - NFCB200_HALO - 2 * NFCB200_BLOCK : 0;
      if (hs.running)
         keepFrom = hs.pos > SCR_HALO + NFCB200_BLOCK ? hs.pos - SCR_HALO - NFCB200_BLOCK : 0; // screening history only
      keepFrom &= ~(u32) (NFCB200_BLOCK - 1); // block aligned
      if (keepFrom < S.base)
         keepFrom = S.base;
      u32 drop = keepFrom - S.base;
      if (drop)
      {
         S.hostTail.erase(S.hostTail.begin(), S.hostTail.begin() + (size_t) drop * bs);
         S.base += drop;
         S.count -= drop;
      }
   }

   if (n_out)
      *n_out = deliver;

   if (nf > cap)
      return fail(NFCB200_ERR_CAPACITY, "%llu frames decoded but room for %llu only: the rest waits in nfcb200_stream_pending", (unsigned long long) nf,
                  (unsigned long long) cap);

   return 0;
}

}
