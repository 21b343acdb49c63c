/*
 * nfcb200.cu -- C ABI (include/nfcb200.h) and host orchestration of the H100 NFC demodulation path.
 *
 * One translation unit: the kernels live in nfc_screen.cuh / nfc_decode.cuh, the exact lane machine in nfc_core.h.
 * Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -fmad=false -shared -Xcompiler -fPIC
 * (-fmad=false: the reference's x86 build has no FMA, CMakeLists.txt:36-40; lane decisions must be bit-identical).
 *
 * There is no CPU fallback in this library: every entry point that decodes requires a CUDA device.
 */
#include <cuda_runtime.h>
#include <sched.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdarg>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <atomic>
#include <functional>
#include <vector>

#include "../../include/nfcb200.h"
#include "nfc_decode.cuh"
#include "nfc_spectrum.cuh"
#include "iso_decode.cuh"

using namespace nfcb200;

// ---------------------------------------------------------------------------------------------------------------------
// errors
// ---------------------------------------------------------------------------------------------------------------------
static thread_local char g_error[512] = "";

static int fail(int code, const char *fmt, ...)
{
   va_list ap;
   va_start(ap, fmt);
   vsnprintf(g_error, sizeof(g_error), fmt, ap);
   va_end(ap);
   return code;
}

#define CUDA_TRY(expr)                                                                                              \
   do                                                                                                               \
   {                                                                                                                \
      cudaError_t e_ = (expr);                                                                                      \
      if (e_ != cudaSuccess)                                                                                        \
         return fail(NFCB200_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); \
   }                                                                                                                \
   while (0)

// ---------------------------------------------------------------------------------------------------------------------
// device buffer that only grows
// ---------------------------------------------------------------------------------------------------------------------
struct DevBuf
{
   void *ptr = nullptr;
   size_t cap = 0;

   int reserve(size_t bytes)
   {
      if (bytes <= cap)
         return 0;
      if (ptr)
         cudaFree(ptr);
      ptr = nullptr;
      cap = 0;
      size_t want = bytes + bytes / 8 + 256;
      cudaError_t e = cudaMalloc(&ptr, want);
      if (e != cudaSuccess)
         return fail(NFCB200_ERR_CUDA, "cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e));
      cap = want;
      return 0;
   }

   // grow, preserving the first `keep` bytes (the packed frames of the earlier chunks of one call)
   int reserve_keep(size_t bytes, size_t keep, cudaStream_t st)
   {
      if (bytes <= cap)
         return 0;
      size_t want = bytes + bytes / 2 + 256;
      void *np = nullptr;
      cudaError_t e = cudaMalloc(&np, want);
      if (e != cudaSuccess)
         return fail(NFCB200_ERR_CUDA, "cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e));
      if (ptr && keep)
      {
         cudaMemcpyAsync(np, ptr, keep, cudaMemcpyDeviceToDevice, st);
         cudaStreamSynchronize(st);
      }
      if (ptr)
         cudaFree(ptr);
      ptr = np;
      cap = want;
      return 0;
   }

   void release()
   {
      if (ptr)
         cudaFree(ptr);
      ptr = nullptr;
      cap = 0;
   }

   template <class T>
   T *as() const
   {
      return (T *) ptr;
   }
};

// pinned host staging that only grows (frame records travel device -> host at link speed, not through a pageable bounce)
struct HostBuf
{
   void *ptr = nullptr;
   size_t cap = 0;

   int reserve(size_t bytes)
   {
      if (bytes <= cap)
         return 0;
      if (ptr)
         cudaFreeHost(ptr);
      ptr = nullptr;
      cap = 0;
      size_t want = bytes + bytes / 4 + 4096;
      cudaError_t e = cudaHostAlloc(&ptr, want, cudaHostAllocDefault);
      if (e != cudaSuccess)
         return fail(NFCB200_ERR_CUDA, "cudaHostAlloc(%zu) failed: %s", want, cudaGetErrorString(e));
      cap = want;
      return 0;
   }

   void release()
   {
      if (ptr)
         cudaFreeHost(ptr);
      ptr = nullptr;
      cap = 0;
   }

   template <class T>
   T *as() const
   {
      return (T *) ptr;
   }
};

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

// Host threads this process may use for the conversion of frame records: the CPUs it is allowed to run on (affinity, clipped
// by a cgroup CPU quota) divided by the processes that share them (one per GPU under torchrun: LOCAL_WORLD_SIZE).  With 8
// ranks on a 16-CPU quota, 8 x 16 conversion threads exhausted the quota and the kernel throttled the whole job.
static unsigned host_workers()
{
   static unsigned cached = 0;
   if (cached)
      return cached;
   unsigned n = std::max(1u, std::thread::hardware_concurrency());
   cpu_set_t set;
   if (sched_getaffinity(0, sizeof(set), &set) == 0)
      n = std::max(1, CPU_COUNT(&set));
   if (FILE *f = fopen("/sys/fs/cgroup/cpu.max", "r"))
   {
      char q[64] = "";
      double per = 0;
      if (fscanf(f, "%63s %lf", q, &per) == 2 && strcmp(q, "max") != 0 && per > 0)
         n = std::max(1u, std::min(n, (unsigned) (atof(q) / per + 0.5)));
      fclose(f);
   }
   unsigned share = 1;
   if (const char *e = getenv("LOCAL_WORLD_SIZE"))
      share = (unsigned) std::max(1, atoi(e));
   cached = std::max(1u, std::min(16u, n / share));
   return cached;
}

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

struct nfcb200_handle
{
   nfcb200_config cfg;
   Params P;
   u32 paramsRate = 0;
   int device = 0;
   int smCount = 132;
   cudaStream_t stream = nullptr;
   cudaStream_t copyStream = nullptr;
   cudaEvent_t copied[2] = {};
   cudaEvent_t ev[12] = {};

   int wlanesPerSm = 7; // resident warp lanes per SM (shared memory: sizeof(WLaneSmem) each)
   bool stragglerAlways = false;
   u32 stragglerMargin = 0; // thread lanes: samples past its queued length after which a lane that holds the launch gives up
                               // and is decoded again by a warp lane (0: never; development knob NFCB200_STRAGGLER)
   int laneBlocks = 4;  // resident thread-lane blocks per SM (lanes_kernel __launch_bounds__)
   int shortHalo = 1;   // NFCB200_HALO_SHORT=0 forces the long warm-up for every segment (measurement knob)

   HostBuf hRecs, hExt; // gather staging
   DevBuf carryDev;                    // injected carry (nfcb200_set_carry) / carry query result
   Carry carryIn;                      // host copy of the injected carry
   bool haveCarryIn = false;
   bool lastCarryInUsed = false;       // the last decode started from the injected carry
   u32 lastLanes = 0;                  // lanes of the last single-stream decode (nfcb200_carry_before)
   DevBuf packed, packedExt, packCtr; // frames of the current call, ordered and packed on the device (all chunks)
   uint64_t packedCount = 0;           // records in `packed`
   u32 packedExtCount = 0;             // 128-byte chunks in `packedExt`
   u32 packedRate = 0;

   DevBuf samples, flags, bsum, counts, offsets, segCounts, segOffsets, segs, feats, lanes, queue, scratch, sbuf, pool, ext, meta, counters;
   nfcb200_stats stats;

   // last batch geometry (for the flag tap)
   u32 lastStreams = 0, lastBlocks = 0;

   // streaming state
   DevBuf sState, sScratch, sSbuf, sSamples, sFlags, sBsum, sCounts;
   std::vector<unsigned char> sHostTail; // samples retained on the host side of the stream buffer
   u32 sBase = 0;        // absolute index of the first retained sample
   u32 sCount = 0;       // retained samples
   u32 sRate = 0;
   int sSig = 0;
   bool sInit = false;
   u32 sEmitted = 0;     // frames already returned
   std::vector<nfcb200_frame> sPending; // decoded but not yet delivered (the caller's buffer was too small)

   // nfcb200_spectrum: its own buffers, so that a spectrum call leaves every decode state above as it was
   DevBuf specTables, specIn, specOut; // twiddles + window (uploaded once), staged host input, staged host output
   bool specTablesReady = false;

   // nfcb200_iso7816_decode_batch: its own buffers too
   DevBuf isoIn, isoLine, isoLineCount, isoClk, isoClkCount, isoPool, isoCtr, isoStreamCount, isoFirst, isoOrdered;
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

static void fill_screen_config(const nfcb200_handle *h, ScreenConfig &sc)
{
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
   memset(&h->stats, 0, sizeof(h->stats));
   h->packedCount = 0;
   h->packedExtCount = 0;

   cudaDeviceProp prop;
   if (cudaGetDeviceProperties(&prop, c.device) == cudaSuccess)
      h->smCount = prop.multiProcessorCount;

   e = cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking);
   if (e != cudaSuccess)
   {
      delete h;
      return fail(NFCB200_ERR_CUDA, "cudaStreamCreate failed: %s", cudaGetErrorString(e));
   }

   for (auto &ev: h->ev)
      cudaEventCreate(&ev);

   if (const char *e = getenv("NFCB200_HALO_SHORT"))
      h->shortHalo = atoi(e) ? 1 : 0;
   if (const char *e = getenv("NFCB200_STRAGGLER"))
   {
      // N > 0: margin in samples; 0: off; N < 0 (tests): margin |N|, and a lane gives up whether the queue is empty or not
      const int v = atoi(e);
      h->stragglerMargin = (u32) (v < 0 ? -v : v);
      h->stragglerAlways = v < 0;
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
         h->wlanesPerSm = perSm;
   }
   {
      // the persistent thread-lane grid and its scratch are sized from laneBlocks: never more blocks than fit (registers,
      // and the shared memory of the Front array plus the tap stages)
      int plain = 0, bail = 0;
      if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&plain, lanes_kernel<false>, LANE_THREADS, 0) == cudaSuccess &&
          cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bail, lanes_kernel<true>, LANE_THREADS, 0) == cudaSuccess)
      {
         const int fit = std::min(plain, bail);
         if (fit > 0 && fit < h->laneBlocks)
         {
            fprintf(stderr, "nfcb200: only %d thread-lane blocks fit per SM (expected %d)\n", fit, h->laneBlocks);
            h->laneBlocks = fit;
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
   DevBuf *bufs[] = {&h->samples, &h->flags, &h->bsum, &h->counts, &h->offsets, &h->lanes, &h->queue, &h->segCounts, &h->segOffsets, &h->segs, &h->feats, &h->scratch, &h->sbuf, &h->pool, &h->ext, &h->meta, &h->carryDev, &h->packed, &h->packedExt, &h->packCtr,
                     &h->counters, &h->sState, &h->sScratch, &h->sSbuf, &h->sSamples, &h->sFlags, &h->sBsum, &h->sCounts,
                     &h->specTables, &h->specIn, &h->specOut, &h->isoIn, &h->isoLine, &h->isoLineCount, &h->isoClk, &h->isoClkCount,
                     &h->isoPool, &h->isoCtr, &h->isoStreamCount, &h->isoFirst, &h->isoOrdered};
   for (DevBuf *b: bufs)
      b->release();
   HostBuf *hbufs[] = {&h->hRecs, &h->hExt};
   for (HostBuf *b: hbufs)
      b->release();
   for (auto &ev: h->ev)
      if (ev)
         cudaEventDestroy(ev);
   for (auto &ev: h->copied)
      if (ev)
         cudaEventDestroy(ev);
   if (h->copyStream)
      cudaStreamDestroy(h->copyStream);
   if (h->stream)
      cudaStreamDestroy(h->stream);
   delete h;
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
   *stats = h->stats;
   return 0;
}

int nfcb200_get_block_flags(nfcb200_handle *h, uint8_t *out, uint64_t cap, uint64_t *n_blocks_per_stream)
{
   if (!h)
      return fail(NFCB200_ERR_INVALID, "null handle");
   if (n_blocks_per_stream)
      *n_blocks_per_stream = h->lastBlocks;
   uint64_t total = (uint64_t) h->lastStreams * h->lastBlocks;
   if (!out)
      return 0;
   if (cap < total)
      return fail(NFCB200_ERR_CAPACITY, "flag buffer too small: need %llu bytes", (unsigned long long) total);
   CUDA_TRY(cudaSetDevice(h->device));
   CUDA_TRY(cudaMemcpy(out, h->flags.ptr, total, cudaMemcpyDeviceToHost));
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

// decode one device-resident batch [n_streams][n_samples]; frames are written to out[outOffset ...) (bounded by cap) with
// stream indices offset by streamBase; statistics are ACCUMULATED into h->stats
static int decode_resident(nfcb200_handle *h, const void *dSamples, int sigtype, uint32_t n_streams, uint64_t n_samples, uint32_t sample_rate,
                           uint32_t streamBase, nfcb200_frame *out, uint64_t cap, uint64_t outOffset, uint64_t *produced)
{
   cudaStream_t st = h->stream;
   const u32 bs = sig_bytes(sigtype);
   const uint64_t total = (uint64_t) n_streams * n_samples;
   const u32 n_blocks = (u32) ((n_samples + NFCB200_BLOCK - 1) / NFCB200_BLOCK);
   const u32 tiles = (u32) ((n_samples + SCR_TILE - 1) / SCR_TILE);
   uint64_t launches = 0;

   nfcb200_stats &S = h->stats;
   nfcb200_stats prev = S;
   S.lane_runs = 0;
   S.samples += total;
   S.blocks += (uint64_t) n_streams * n_blocks;

   Trace tr;
   cudaEventRecord(h->ev[1], st);

   // ---- K1: screening -------------------------------------------------------------------------------------------------
   {
      int rc = h->flags.reserve((size_t) n_streams * n_blocks);
      rc = rc ? rc : h->bsum.reserve((size_t) n_streams * n_blocks * sizeof(float));
      rc = rc ? rc : h->counts.reserve((size_t) n_streams * sizeof(u32));
      rc = rc ? rc : h->offsets.reserve((size_t) n_streams * sizeof(u32));
      rc = rc ? rc : h->segCounts.reserve((size_t) n_streams * sizeof(u32));
      rc = rc ? rc : h->segOffsets.reserve((size_t) n_streams * sizeof(u32));
      rc = rc ? rc : h->counters.reserve(sizeof(Counters));
      if (rc)
         return rc;
   }

   // a single-stream decode may continue a capture: the carry in front of its first lane (nfcb200_set_carry, one shot)
   const Carry *dCarryIn = nullptr;
   {
      int rc = h->carryDev.reserve(2 * sizeof(Carry) + 16);
      if (rc)
         return rc;
      if (h->haveCarryIn && n_streams == 1 && streamBase == 0)
      {
         CUDA_TRY(cudaMemcpyAsync(h->carryDev.ptr, &h->carryIn, sizeof(Carry), cudaMemcpyHostToDevice, st));
         dCarryIn = h->carryDev.as<Carry>();
      }
   }

   ScreenConfig sc;
   memset(&sc, 0, sizeof(sc));
   sc.samples = dSamples;
   sc.n_samples = n_samples;
   sc.n_streams = n_streams;
   sc.sigtype = sigtype;
   sc.n_blocks = n_blocks;
   sc.tiles_per_stream = tiles;
   sc.flags = h->flags.as<uint8_t>();
   sc.bsum = h->bsum.as<float>();
   fill_screen_config(h, sc);
   // cp.async.bulk needs 16-byte aligned global addresses: stream pitch and base pointer
   if ((((uintptr_t) dSamples) & 15) || ((n_samples * bs) & 15))
      sc.use_tma = 0;

   {
      uint64_t items = (uint64_t) n_streams * tiles;
      if (items >= 0xFFFF0000ull)
         return fail(NFCB200_ERR_CAPACITY, "batch of %llu screening tiles exceeds one launch", (unsigned long long) items);
      launch_screen(h, sc, (u32) items, st);
      launches++;
      CUDA_TRY(cudaGetLastError());
   }

   cudaEventRecord(h->ev[2], st);

   // ---- segments ------------------------------------------------------------------------------------------------------
   SegmentConfig sg;
   memset(&sg, 0, sizeof(sg));
   sg.flags = h->flags.as<uint8_t>();
   sg.bsum = h->bsum.as<float>();
   sg.n_streams = n_streams;
   sg.n_blocks = n_blocks;
   sg.n_samples = n_samples;
   sg.counts = h->counts.as<u32>();
   sg.offsets = h->offsets.as<u32>();
   sg.low = h->P.lowThr;
   sg.high = h->P.highThr;
   sg.meanW = powf(h->P.meanW0, (float) NFCB200_BLOCK);
   sg.shortHalo = (u32) h->shortHalo;

   Counters *dC = h->counters.as<Counters>();
   CUDA_TRY(cudaMemsetAsync(dC, 0, sizeof(Counters), st));
   sg.segTotal = &dC->segTotal;
   sg.activeTotal = &dC->activeBlocks;
   sg.group = 1;
   sg.carryIn = dCarryIn;

   const u32 sgrid = (n_streams + 63) / 64;
   {
      CUDA_TRY(cudaMemsetAsync(h->counts.ptr, 0, (size_t) n_streams * sizeof(u32), st));
      const uint64_t nb = (uint64_t) n_streams * n_blocks;
      const u32 bgrid = (u32) ((nb + 255) / 256);
      segment_flags_kernel<<<bgrid, 256, 0, st>>>(sg);
      segment_activate_kernel<<<bgrid, 256, 0, st>>>(sg);
      segment_starts_kernel<<<bgrid, 256, 0, st>>>(sg);
      launches += 3;
      CUDA_TRY(cudaGetLastError());
   }

   // Lanes.  Exact mode: ONE warp lane decodes the whole stream -- the detectors' running sums carry their rounding history
   // (NfcA.cpp:246-250), which only a run over the whole capture reproduces bit for bit (nfc_wlane.h).  Throughput mode:
   // thread lanes, one per group of segments, cold-started sums (exact on 16-bit input), as many lanes as fill the machine a
   // few times over (every lane pays a warm-up halo; longer lanes keep more of the carry chain inside one sequential run).
   const bool exact = h->cfg.exact != 0;
   u32 segTotal = 0;
   CUDA_TRY(cudaMemcpyAsync(&segTotal, &dC->segTotal, sizeof(u32), cudaMemcpyDeviceToHost, st));
   CUDA_TRY(cudaMemcpyAsync(h->segCounts.ptr, h->counts.ptr, (size_t) n_streams * sizeof(u32), cudaMemcpyDeviceToDevice, st));
   CUDA_TRY(cudaStreamSynchronize(st));
   {
      u32 group;
      if (h->cfg.segments_per_lane)
         group = h->cfg.segments_per_lane;
      else if (exact && sigtype == SIG_MAG_S16 && (uint64_t) n_streams < (uint64_t) h->smCount * (uint64_t) h->wlanesPerSm)
      {
         // 16-bit mono input adds exactly whatever the history of a running sum: a stream may be cut into several warp lanes
         // (cold starts + carry chain) without losing a bit -- small batches fill the machine that way
         const uint64_t resident = (uint64_t) h->smCount * (uint64_t) h->wlanesPerSm;
         group = (u32) std::max<uint64_t>(1, segTotal / (resident * 2));
      }
      else if (exact)
         group = 0xFFFFFFFFu; // one lane per stream
      else
      {
         const uint64_t residentLanes = (uint64_t) h->smCount * (uint64_t) h->laneBlocks * (LANE_THREADS / 32) * 32;
         group = (u32) std::min<uint64_t>(64, std::max<uint64_t>(1, segTotal / std::max<uint64_t>(1, residentLanes * 2)));
      }
      sg.group = group;
      if (group > 1)
      {
         segment_group_kernel<<<sgrid, 64, 0, st>>>(sg);
         launches++;
         CUDA_TRY(cudaGetLastError());
      }
   }
   S.segments = segTotal;
   tr.mark("screen + segments");

   std::vector<u32> counts(n_streams), offsets(n_streams), segCounts(n_streams), segOffsets(n_streams);
   CUDA_TRY(cudaMemcpyAsync(counts.data(), h->counts.ptr, n_streams * sizeof(u32), cudaMemcpyDeviceToHost, st));
   CUDA_TRY(cudaMemcpyAsync(segCounts.data(), h->segCounts.ptr, n_streams * sizeof(u32), cudaMemcpyDeviceToHost, st));
   CUDA_TRY(cudaStreamSynchronize(st));

   uint64_t nLanes64 = 0, nSegs64 = 0;
   for (u32 s = 0; s < n_streams; s++)
   {
      offsets[s] = (u32) nLanes64;
      nLanes64 += counts[s];
      segOffsets[s] = (u32) nSegs64;
      nSegs64 += segCounts[s];
   }
   if (nLanes64 >= 0x7FFFFFFFull || nSegs64 >= 0x7FFFFFFFull)
      return fail(NFCB200_ERR_CAPACITY, "too many segments (%llu)", (unsigned long long) nSegs64);
   const u32 nLanes = (u32) nLanes64;
   const u32 nSegs = (u32) nSegs64;
   S.lanes = nLanes;   // this chunk; accumulated with the previous chunks at the end

   {
      int rc = h->lanes.reserve((size_t) nLanes * sizeof(LaneRec));
      rc = rc ? rc : h->segs.reserve((size_t) std::max<u32>(nSegs, 1) * sizeof(SegRec));
      rc = rc ? rc : h->queue.reserve((size_t) nLanes * sizeof(u32));
      rc = rc ? rc : h->meta.reserve((size_t) (nLanes + 1) * sizeof(u32));
      if (rc)
         return rc;
   }

   CUDA_TRY(cudaMemcpyAsync(h->offsets.ptr, offsets.data(), n_streams * sizeof(u32), cudaMemcpyHostToDevice, st));
   CUDA_TRY(cudaMemcpyAsync(h->segOffsets.ptr, segOffsets.data(), n_streams * sizeof(u32), cudaMemcpyHostToDevice, st));
   sg.lanes = h->lanes.as<LaneRec>();
   sg.queue = h->queue.as<u32>();
   sg.segCounts = h->segCounts.as<u32>();
   sg.segOffsets = h->segOffsets.as<u32>();
   sg.segs = h->segs.as<SegRec>();
   sg.featTotal = &dC->featTotal;
   sg.carryIn = dCarryIn;
   segment_fill_kernel<<<n_streams, 32, 0, st>>>(sg, h->P);
   launches++;
   CUDA_TRY(cudaGetLastError());

   // first-round queue ordered by decreasing lane length (counting sort on the host: the lengths are 4 bytes per lane)
   if (!exact && nLanes > 64)
   {
      lane_length_kernel<<<(nLanes + 255) / 256, 256, 0, st>>>(h->lanes.as<LaneRec>(), nLanes, h->meta.as<u32>());
      launches++;
      std::vector<u32> len(nLanes), order(nLanes);
      CUDA_TRY(cudaMemcpyAsync(len.data(), h->meta.ptr, (size_t) nLanes * sizeof(u32), cudaMemcpyDeviceToHost, st));
      CUDA_TRY(cudaStreamSynchronize(st));
      const u32 shift = 8, buckets = 1u << 16;
      std::vector<u32> hist(buckets + 1, 0);
      auto key = [&](u32 v) { u32 k = v >> shift; return k >= buckets ? 0u : buckets - 1 - k; }; // descending
      for (u32 i = 0; i < nLanes; i++)
         hist[key(len[i]) + 1]++;
      for (u32 b = 0; b < buckets; b++)
         hist[b + 1] += hist[b];
      for (u32 i = 0; i < nLanes; i++)
         order[hist[key(len[i])]++] = i;
      CUDA_TRY(cudaMemcpyAsync(h->queue.ptr, order.data(), (size_t) nLanes * sizeof(u32), cudaMemcpyHostToDevice, st));
      CUDA_TRY(cudaStreamSynchronize(st));
   }

   // ---- front pass: the sequential float recurrences of nextSample, one thread per segment -> feature pool ----------
   unsigned long long featTotal = 0;
   CUDA_TRY(cudaMemcpyAsync(&featTotal, &dC->featTotal, sizeof(featTotal), cudaMemcpyDeviceToHost, st));
   CUDA_TRY(cudaStreamSynchronize(st));
   {
      int rc = h->feats.reserve((size_t) std::max<unsigned long long>(exact ? featTotal : 0, 1) * sizeof(float4));
      if (rc)
         return rc;
   }
   S.feature_samples = featTotal;
   cudaEventRecord(h->ev[8], st);
   if (nSegs && exact)
   {
      FrontConfig fc;
      fc.samples = dSamples;
      fc.n_samples = n_samples;
      fc.sigtype = sigtype;
      fc.segs = h->segs.as<SegRec>();
      fc.n_segs = nSegs;
      fc.pool = h->feats.as<float4>();
      launch_front(fc, h->P, st);
      launches++;
      CUDA_TRY(cudaGetLastError());
   }

   tr.mark("lane fill + front pass");
   cudaEventRecord(h->ev[3], st);

   // ---- frame pool ----------------------------------------------------------------------------------------------------
   u32 poolCap = (u32) std::min<uint64_t>(32u << 20, std::max<uint64_t>(1u << 16, total / 512 + (uint64_t) nLanes * 8));
   u32 extCap = std::max<u32>(1u << 12, poolCap / 8);
   {
      int rc = h->pool.reserve((size_t) poolCap * sizeof(FrameRec));
      rc = rc ? rc : h->ext.reserve((size_t) extCap * 128);
      if (rc)
         return rc;
   }

   FramePool pool;
   pool.recs = h->pool.as<FrameRec>();
   pool.cap = poolCap;
   pool.count = &dC->poolCount;
   pool.ext = h->ext.as<u8>();
   pool.extCap = extCap;
   pool.extCount = &dC->extCount;

   // ---- lanes + chain, to the fixed point -----------------------------------------------------------------------------
   const u32 maxWarps = (u32) h->smCount * (u32) h->wlanesPerSm; // resident warp lanes: the kernel is persistent

   WLaneConfig lc;
   memset(&lc, 0, sizeof(lc));
   lc.samples = dSamples;
   lc.n_samples = n_samples;
   lc.sigtype = sigtype;
   lc.flags = h->flags.as<uint8_t>();
   lc.bsum = h->bsum.as<float>();
   lc.n_blocks = n_blocks;
   lc.lanes = h->lanes.as<LaneRec>();
   lc.queue = h->queue.as<u32>();
   lc.cursor = &dC->cursor;
   lc.segs = h->segs.as<SegRec>();
   lc.n_segs = nSegs;
   lc.pool = h->feats.as<float4>();
   lc.frames = pool;
   lc.work = &dC->work;
   lc.use_tma = sc.use_tma;
   lc.phase = dC->phase;

   ChainConfig cc;
   cc.carryIn = dCarryIn;
   cc.lanes = h->lanes.as<LaneRec>();
   cc.offsets = h->offsets.as<u32>();
   cc.counts = h->counts.as<u32>();
   cc.n_streams = n_streams;
   cc.queue = h->queue.as<u32>();
   cc.queue_count = &dC->queueCount;

   u32 queueCount = nLanes;
   u32 maxRounds = h->cfg.max_rounds ? h->cfg.max_rounds : 4096;
   u32 rounds = 0;
   u32 stragglers = 0;

   while (queueCount > 0)
   {
      if (rounds >= maxRounds)
         return fail(NFCB200_ERR_CAPACITY, "carry chain did not converge in %u rounds", maxRounds);

      CUDA_TRY(cudaMemsetAsync(&dC->cursor, 0, sizeof(u32), st));

      if (exact)
      {
         const u32 blocks = std::min(maxWarps, queueCount);
         lc.queue_count = queueCount;
         wlanes_kernel<<<blocks, 32, sizeof(WLaneSmem), st>>>(lc, h->P);
      }
      else
      {
         const u32 warpsPerBlock = LANE_THREADS / 32;
         const u32 maxThreadWarps = (u32) h->smCount * (u32) h->laneBlocks * warpsPerBlock; // the kernel is persistent
         u32 warps = std::min(maxThreadWarps, (queueCount + 31) / 32);
         const u32 blocks = (warps + warpsPerBlock - 1) / warpsPerBlock;
         warps = blocks * warpsPerBlock;

         int rc = h->scratch.reserve((size_t) warps * NFCB200_SCRATCH_FLOATS * 32 * sizeof(float));
         rc = rc ? rc : h->sbuf.reserve((size_t) warps * 32 * 512);
         if (rc)
            return rc;

         LaneConfig tc;
         memset(&tc, 0, sizeof(tc));
         tc.samples = dSamples;
         tc.n_samples = n_samples;
         tc.sigtype = sigtype;
         tc.flags = h->flags.as<uint8_t>();
         tc.n_blocks = n_blocks;
         tc.lanes = h->lanes.as<LaneRec>();
         tc.n_lanes = nLanes;
         tc.queue = h->queue.as<u32>();
         tc.queue_count = queueCount;
         tc.cursor = &dC->cursor;
         tc.scratch = h->scratch.as<float>();
         tc.sbuf = h->sbuf.as<uint8_t>();
         tc.pool = pool;
         tc.work = &dC->work;
         tc.bail_margin = h->stragglerMargin;
         tc.bail_always = h->stragglerAlways ? 1u : 0u;
         tc.overrun = h->meta.as<u32>(); // free between the queue ordering and the gather
         tc.overrun_count = &dC->overrunCount;
         CUDA_TRY(cudaMemsetAsync(&dC->overrunCount, 0, sizeof(u32), st));
         if (tc.bail_margin)
            lanes_kernel<true><<<blocks, LANE_THREADS, 0, st>>>(tc, h->P);
         else
            lanes_kernel<false><<<blocks, LANE_THREADS, 0, st>>>(tc, h->P);

         if (tc.bail_margin)
         {
            u32 overrun = 0;
            CUDA_TRY(cudaMemcpyAsync(&overrun, &dC->overrunCount, sizeof(u32), cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaStreamSynchronize(st));
            if (tr.on)
               tr.mark("  thread lanes");
            if (overrun)
            {
               // the stragglers again, each by a whole warp with its history in shared memory; without a feature pool the
               // warp lane runs the front end itself (SegRec::hasFeat is 0 in throughput mode)
               CUDA_TRY(cudaMemsetAsync(&dC->cursor, 0, sizeof(u32), st));
               lc.queue = h->meta.as<u32>();
               lc.queue_count = overrun;
               wlanes_kernel<<<std::min(maxWarps, overrun), 32, sizeof(WLaneSmem), st>>>(lc, h->P);
               launches++;
               S.lane_runs += overrun;
               stragglers += overrun;
               if (tr.on)
               {
                  cudaStreamSynchronize(st);
                  char what[64];
                  snprintf(what, sizeof(what), "  %u straggler(s) on warp lanes", overrun);
                  tr.mark(what);
               }
            }
         }
      }
      launches++;
      CUDA_TRY(cudaGetLastError());

      S.lane_runs += queueCount;
      rounds++;

      CUDA_TRY(cudaMemsetAsync(&dC->queueCount, 0, sizeof(u32), st));
      chain_warp_kernel<<<(n_streams + CHAIN_WARPS - 1) / CHAIN_WARPS, CHAIN_WARPS * 32, 0, st>>>(cc, h->P);
      launches++;
      CUDA_TRY(cudaGetLastError());

      const u32 ran = queueCount;
      CUDA_TRY(cudaMemcpyAsync(&queueCount, &dC->queueCount, sizeof(u32), cudaMemcpyDeviceToHost, st));
      CUDA_TRY(cudaStreamSynchronize(st));
      if (tr.on)
      {
         char what[64];
         snprintf(what, sizeof(what), "  round %u: %u lanes", rounds, ran);
         tr.mark(what);
      }
   }

   S.rounds = rounds;
   S.straggler_lanes += (float) stragglers;
   tr.mark("lanes + chain");

   if (tr.on && nLanes)
   {
      // how far the lanes really ran: the longest run bounds the lane kernel from below whatever the total work is
      if (h->scratch.reserve(65 * sizeof(unsigned long long)) == 0)
      {
         unsigned long long *dStat = (unsigned long long *) h->scratch.ptr;
         unsigned long long hs[65];
         cudaMemsetAsync(dStat, 0, sizeof(hs), st);
         lane_run_stat_kernel<<<(nLanes + 255) / 256, 256, 0, st>>>(h->lanes.as<LaneRec>(), nLanes, dStat);
         cudaMemcpyAsync(hs, dStat, sizeof(hs), cudaMemcpyDeviceToHost, st);
         cudaStreamSynchronize(st);
         LaneRec lr;
         const u32 li = (u32) (hs[64] & 0xFFFFFFFFu);
         cudaMemcpy(&lr, h->lanes.as<LaneRec>() + li, sizeof(LaneRec), cudaMemcpyDeviceToHost);
         fprintf(stderr, "[nfcb200] longest lane run: %llu samples (lane %u, stream %u, first %u begin %u end0 %u end %u stop %u, %u frames)\n[nfcb200] runs by length / 4096:",
                 hs[64] >> 32, li, lr.stream, lr.first, lr.begin, lr.end0, lr.end, lr.stop, lr.nframes);
         for (int b = 0; b < 64; b++)
            if (hs[b])
               fprintf(stderr, " %d:%llu", b, hs[b]);
         fprintf(stderr, "\n");
         tr.mark("(lane run statistics)");
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

   cudaEventRecord(h->ev[4], st);

   // ---- gather: ordered and packed on the device, one copy to the host ---------------------------------------------------
   u32 *dLaneOff = h->meta.as<u32>(); // [nLanes + 1]
   frame_offsets_kernel<<<1, 1024, 0, st>>>(h->lanes.as<LaneRec>(), nLanes, dLaneOff, &dC->live);
   launches++;
   CUDA_TRY(cudaGetLastError());

   Counters hc;
   u32 nf32 = 0;
   CUDA_TRY(cudaMemcpyAsync(&hc, dC, sizeof(Counters), cudaMemcpyDeviceToHost, st));
   CUDA_TRY(cudaMemcpyAsync(&nf32, dLaneOff + nLanes, sizeof(u32), cudaMemcpyDeviceToHost, st));
   CUDA_TRY(cudaStreamSynchronize(st));

   S.lane_samples = hc.work;
   if (tr.on && (exact || stragglers))
   {
      static const char *names[8] = {"control", "fill", "search", "machine", "walk", "jump", "scalar", "locked"};
      unsigned long long tot = 0;
      for (int i = 0; i < 8; i++)
         tot += hc.phase[i];
      for (int i = 0; i < 8; i++)
         fprintf(stderr, "[nfcb200] lanes %-8s %5.1f %% of cycles, %12llu samples, %8.1f cycles / sample\n", names[i], 100.0 * hc.phase[i] / (double) (tot ? tot : 1),
                 hc.phase[8 + i], hc.phase[8 + i] ? (double) hc.phase[i] / (double) hc.phase[8 + i] : 0.0);
   }
   S.live_lanes = hc.live;
   S.active_blocks = prev.active_blocks + hc.activeBlocks;

   if (hc.poolCount > poolCap || hc.extCount > extCap)
      return fail(NFCB200_ERR_CAPACITY, "frame pool exhausted (%u frames, %u extension chunks)", hc.poolCount, hc.extCount);

   const uint64_t nf = nf32;
   const u32 extBefore = h->packedExtCount;
   {
      int rc = h->packed.reserve_keep((size_t) (h->packedCount + nf) * sizeof(FrameRec), (size_t) h->packedCount * sizeof(FrameRec), st);
      rc = rc ? rc : h->packedExt.reserve_keep((size_t) (extBefore + hc.extCount + 1) * 128, (size_t) extBefore * 128, st);
      rc = rc ? rc : h->packCtr.reserve(sizeof(u32));
      if (rc)
         return rc;
   }
   const u32 packedExtCap = (u32) std::min<size_t>(h->packedExt.cap / 128, 0xFFFFFFFFu);
   CUDA_TRY(cudaMemcpyAsync(h->packCtr.ptr, &extBefore, sizeof(u32), cudaMemcpyHostToDevice, st));

   FrameRec *dPacked = h->packed.as<FrameRec>() + h->packedCount;
   if (hc.poolCount)
   {
      const u32 grid = std::min<u32>((hc.poolCount + 255) / 256, (u32) h->smCount * 8);
      frame_compact_kernel<<<grid, 256, 0, st>>>(h->pool.as<FrameRec>(), hc.poolCount, h->lanes.as<LaneRec>(), nLanes, dLaneOff, h->ext.as<u8>(), hc.extCount,
                                                  streamBase, dPacked, h->packedExt.as<u8>(), packedExtCap, h->packCtr.as<u32>());
      launches++;
      CUDA_TRY(cudaGetLastError());
   }

   u32 extAfter = extBefore;
   CUDA_TRY(cudaMemcpyAsync(&extAfter, h->packCtr.ptr, sizeof(u32), cudaMemcpyDeviceToHost, st));
   CUDA_TRY(cudaStreamSynchronize(st));
   if (extAfter > packedExtCap)
      extAfter = packedExtCap;

   {
      int rc = h->hRecs.reserve((size_t) std::max<uint64_t>(nf, 1) * sizeof(FrameRec));
      rc = rc ? rc : h->hExt.reserve((size_t) std::max<u32>(extAfter - extBefore, 1) * 128);
      if (rc)
         return rc;
   }

   if (nf)
      CUDA_TRY(cudaMemcpyAsync(h->hRecs.ptr, dPacked, (size_t) nf * sizeof(FrameRec), cudaMemcpyDeviceToHost, st));
   if (extAfter > extBefore)
      CUDA_TRY(cudaMemcpyAsync(h->hExt.ptr, h->packedExt.as<u8>() + (size_t) extBefore * 128, (size_t) (extAfter - extBefore) * 128, cudaMemcpyDeviceToHost, st));

   cudaEventRecord(h->ev[5], st);
   CUDA_TRY(cudaStreamSynchronize(st));
   tr.mark("frames d2h");

   h->packedCount += nf;
   h->packedExtCount = extAfter;
   h->packedRate = sample_rate;

   // conversion to ABI frames on a few host threads (4e5 frames per batch)
   {
      const FrameRec *recs = h->hRecs.as<FrameRec>();
      const unsigned char *ext = h->hExt.as<unsigned char>();
      const uint64_t count = outOffset >= cap ? 0 : std::min<uint64_t>(nf, cap - outOffset);
      const unsigned workers = (unsigned) std::max<uint64_t>(1, std::min<uint64_t>(host_workers(), count / 4096));
      auto work = [&](uint64_t lo, uint64_t hi) {
         for (uint64_t i = lo; i < hi; i++)
         {
            FrameRec r = recs[i];
            if (r.ext != 0xFFFFFFFFu)
               r.ext -= extBefore; // chunk index inside this call's host copy
            emit_frame(h, r, ext, (size_t) (extAfter - extBefore) * 128, r.lane, sample_rate, out[outOffset + i]);
         }
      };
      if (workers <= 1 || count < 8192)
         work(0, count);
      else
      {
         std::vector<std::thread> pool;
         const uint64_t step = (count + workers - 1) / workers;
         for (unsigned w = 0; w < workers; w++)
            pool.emplace_back(work, std::min(count, w * step), std::min(count, (w + 1) * step));
         for (auto &t: pool)
            t.join();
      }
   }

   tr.mark("emit");
   *produced = nf;

   h->lastStreams = n_streams;
   h->lastBlocks = n_blocks;
   h->lastLanes = n_streams == 1 ? nLanes : 0;
   h->lastCarryInUsed = dCarryIn != nullptr;
   if (dCarryIn)
      h->haveCarryIn = false; // one shot

   // accumulate the statistics over the chunks of one call
   float msScreen = 0, msSeg = 0, msLanes = 0, msGather = 0, msFront = 0;
   cudaEventElapsedTime(&msFront, h->ev[8], h->ev[3]);
   cudaEventElapsedTime(&msScreen, h->ev[1], h->ev[2]);
   cudaEventElapsedTime(&msSeg, h->ev[2], h->ev[3]);
   cudaEventElapsedTime(&msLanes, h->ev[3], h->ev[4]);
   cudaEventElapsedTime(&msGather, h->ev[4], h->ev[5]);
   S.ms_screen = prev.ms_screen + msScreen;
   S.ms_segment = prev.ms_segment + msSeg;
   S.ms_lanes = prev.ms_lanes + msLanes;
   S.ms_gather = prev.ms_gather + msGather;
   S.ms_front = prev.ms_front + msFront;
   S.feature_samples += prev.feature_samples;
   S.segments += prev.segments;
   S.lanes += prev.lanes;
   S.live_lanes += prev.live_lanes;
   S.lane_runs += prev.lane_runs;
   S.lane_samples += prev.lane_samples;
   S.rounds = std::max(S.rounds, prev.rounds);
   S.frames = prev.frames + nf;
   S.kernel_launches = prev.kernel_launches + launches;
   (void) bs;
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

   cudaStream_t st = h->stream;
   const u32 bs = sig_bytes(sigtype);
   const uint64_t total = (uint64_t) n_streams * n_samples;

   memset(&h->stats, 0, sizeof(h->stats));
   h->packedCount = 0;      // the packed frames of a call: every chunk of this call appends
   h->packedExtCount = 0;
   nfcb200_stats &S = h->stats;
   Trace wall;

   cudaEventRecord(h->ev[0], st);

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

      int rc = h->samples.reserve((nChunks > 1 ? 2 : 1) * chunkBytes + 64);
      if (rc)
         return rc;

      if (!h->copyStream)
      {
         CUDA_TRY(cudaStreamCreateWithFlags(&h->copyStream, cudaStreamNonBlocking));
         CUDA_TRY(cudaEventCreateWithFlags(&h->copied[0], cudaEventDisableTiming));
         CUDA_TRY(cudaEventCreateWithFlags(&h->copied[1], cudaEventDisableTiming));
      }

      auto issue = [&](uint32_t c) -> cudaError_t {
         const uint32_t s0 = c * chunkStreams;
         const uint32_t sc = std::min(chunkStreams, n_streams - s0);
         unsigned char *dst = (unsigned char *) h->samples.ptr + (c & 1) * chunkBytes;
         cudaError_t e = cudaMemcpyAsync(dst, (const unsigned char *) samples + (uint64_t) s0 * streamBytes, (uint64_t) sc * streamBytes, cudaMemcpyHostToDevice,
                                         h->copyStream);
         if (e != cudaSuccess)
            return e;
         return cudaEventRecord(h->copied[c & 1], h->copyStream);
      };

      CUDA_TRY(issue(0));

      float msCopyWait = 0;

      for (uint32_t c = 0; c < nChunks; c++)
      {
         const uint32_t s0 = c * chunkStreams;
         const uint32_t sc = std::min(chunkStreams, n_streams - s0);

         cudaEventRecord(h->ev[6], st);
         CUDA_TRY(cudaStreamWaitEvent(st, h->copied[c & 1], 0));
         cudaEventRecord(h->ev[7], st);

         // the other staging buffer is free (its decode returned): start the next copy before decoding this chunk
         if (c + 1 < nChunks)
            CUDA_TRY(issue(c + 1));

         uint64_t got = 0;
         rc = decode_resident(h, (unsigned char *) h->samples.ptr + (c & 1) * chunkBytes, sigtype, sc, n_samples, sample_rate, s0, out, cap, nf, &got);
         if (rc)
         {
            cudaStreamSynchronize(h->copyStream); // the next chunk's copy still reads the caller's buffer
            return rc;
         }
         nf += got;

         float w = 0;
         cudaEventElapsedTime(&w, h->ev[6], h->ev[7]);
         msCopyWait += w;
      }

      S.ms_h2d = msCopyWait; // time the decode stream spent waiting for input
   }

   cudaEventRecord(h->ev[5], st);
   CUDA_TRY(cudaStreamSynchronize(st));
   cudaEventElapsedTime(&S.ms_total, h->ev[0], h->ev[5]);
   S.ms_wall = (float) wall.ms();

   if (n_out)
      *n_out = nf;

   if (nf > cap)
      return fail(NFCB200_ERR_CAPACITY, "%llu frames decoded but room for %llu only", (unsigned long long) nf, (unsigned long long) cap);

   return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// FFT spectrum of IQ (FourierProcessTask::process at every hop, nfc_spectrum.cuh)
// ---------------------------------------------------------------------------------------------------------------------
int nfcb200_spectrum_shape(uint64_t n_samples, uint32_t sample_rate, uint64_t hop, uint64_t *n_frames, uint32_t *decimation)
{
   if (hop == 0)
      return fail(NFCB200_ERR_INVALID, "hop of 0 samples");
   if (sample_rate < (uint32_t) SPEC_BANDWIDTH)
      return fail(NFCB200_ERR_UNSUPPORTED, "sample rate %u is below the spectrum's 625 kHz bandwidth (decimation 0)", sample_rate);
   const uint32_t dec = spectrum_decimation(sample_rate);
   if (n_frames)
      *n_frames = spectrum_frames(n_samples, dec, hop);
   if (decimation)
      *decimation = dec;
   return 0;
}

static void launch_spectrum(const nfcb200_handle *h, bool s16, const SpecLaunch &L, cudaStream_t st)
{
   const uint64_t grid = std::min<uint64_t>(L.count, (uint64_t) h->smCount * SPEC_BLOCKS_PER_SM);
   if (s16)
      spectrum_kernel<true><<<(unsigned) grid, SPEC_THREADS, 0, st>>>(L);
   else
      spectrum_kernel<false><<<(unsigned) grid, SPEC_THREADS, 0, st>>>(L);
}

int nfcb200_spectrum(nfcb200_handle *h, const void *samples, int samples_on_device, int sigtype, uint32_t n_streams, uint64_t n_samples,
                     uint32_t sample_rate, uint64_t hop, float *out, int out_on_device, uint64_t cap, uint64_t *n_frames)
{
   if (!h)
      return fail(NFCB200_ERR_INVALID, "null handle");
   if (n_frames)
      *n_frames = 0;
   if (sigtype < SIG_IQ_F32 || sigtype > SIG_IQ_S16)
      return fail(NFCB200_ERR_INVALID, "unknown signal type %d", sigtype);
   if (!samples || n_streams == 0 || n_samples == 0)
      return fail(NFCB200_ERR_INVALID, "empty batch");
   if (cap && !out)
      return fail(NFCB200_ERR_INVALID, "null spectrum buffer");
   if (sigtype != SIG_IQ_F32 && sigtype != SIG_IQ_S16)
      return fail(NFCB200_ERR_UNSUPPORTED, "the spectrum needs IQ samples (FourierProcessTask.cpp:234 skips other buffers)");
   uint64_t nf = 0;
   uint32_t dec = 0;
   int rc = nfcb200_spectrum_shape(n_samples, sample_rate, hop, &nf, &dec);
   if (rc)
      return rc;
   const uint32_t bs = sig_bytes(sigtype);
   if (samples_on_device && ((uintptr_t) samples % bs))
      return fail(NFCB200_ERR_INVALID, "device samples not aligned to %u bytes", bs);
   if (nf > (~0ull / SPEC_LEN) / n_streams)
      return fail(NFCB200_ERR_UNSUPPORTED, "%llu frames per stream overflow the output size", (unsigned long long) nf);
   if (n_frames)
      *n_frames = nf;
   const uint64_t total = (uint64_t) n_streams * nf;
   if (total * SPEC_LEN > cap)
      return fail(NFCB200_ERR_CAPACITY, "%llu spectrum floats needed but room for %llu only", (unsigned long long) (total * SPEC_LEN),
                  (unsigned long long) cap);
   if (total == 0)
      return 0;

   CUDA_TRY(cudaSetDevice(h->device));
   cudaStream_t st = h->stream;

   if (!h->specTablesReady)
   {
      SpecCx tw[SPEC_LEN];
      float win[SPEC_LEN];
      spectrum_tables(tw, win);
      rc = h->specTables.reserve(sizeof(tw) + sizeof(win));
      if (rc)
         return rc;
      CUDA_TRY(cudaMemcpy(h->specTables.ptr, tw, sizeof(tw), cudaMemcpyHostToDevice));
      CUDA_TRY(cudaMemcpy(h->specTables.as<unsigned char>() + sizeof(tw), win, sizeof(win), cudaMemcpyHostToDevice));
      h->specTablesReady = true;
   }

   SpecLaunch L = {};
   L.n_samples = n_samples;
   L.hop = hop;
   L.n_frames = nf;
   L.decimation = dec;
   L.tw = h->specTables.as<SpecCx>();
   L.win = (const float *) (h->specTables.as<SpecCx>() + SPEC_LEN);
   const bool s16 = sigtype == SIG_IQ_S16;

   // host input is staged a group of whole streams at a time (about 1 GB); host output a group of frames at a time (256 MB)
   const uint64_t streamBytes = n_samples * bs;
   const uint32_t chunkStreams = samples_on_device ? n_streams : (uint32_t) std::max<uint64_t>(1, std::min<uint64_t>(n_streams, (1ull << 30) / streamBytes));
   const uint64_t chunkFrames = 1ull << 16;
   if (!samples_on_device && (rc = h->specIn.reserve((uint64_t) chunkStreams * streamBytes)))
      return rc;
   if (!out_on_device && (rc = h->specOut.reserve(std::min(total, chunkFrames) * SPEC_LEN * sizeof(float))))
      return rc;

   for (uint32_t s0 = 0; s0 < n_streams; s0 += chunkStreams)
   {
      const uint32_t sc = std::min(chunkStreams, n_streams - s0);
      if (samples_on_device)
         L.samples = (const unsigned char *) samples + (uint64_t) s0 * streamBytes;
      else
      {
         CUDA_TRY(cudaMemcpyAsync(h->specIn.ptr, (const unsigned char *) samples + (uint64_t) s0 * streamBytes, (uint64_t) sc * streamBytes,
                                  cudaMemcpyHostToDevice, st));
         L.samples = h->specIn.ptr;
      }
      L.s0 = s0;
      const uint64_t g1 = (uint64_t) (s0 + sc) * nf;
      for (uint64_t g0 = (uint64_t) s0 * nf; g0 < g1;)
      {
         L.g0 = g0;
         L.count = out_on_device ? g1 - g0 : std::min(chunkFrames, g1 - g0);
         L.out = out_on_device ? out + g0 * SPEC_LEN : h->specOut.as<float>();
         launch_spectrum(h, s16, L, st);
         CUDA_TRY(cudaGetLastError());
         if (!out_on_device)
            CUDA_TRY(cudaMemcpyAsync(out + g0 * SPEC_LEN, h->specOut.ptr, L.count * SPEC_LEN * sizeof(float), cudaMemcpyDeviceToHost, st));
         g0 += L.count;
      }
   }
   CUDA_TRY(cudaStreamSynchronize(st));
   return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// ISO 7816 contact smart-card traffic from 4-channel logic captures (lab::IsoDecoder, iso_decode.cuh)
// ---------------------------------------------------------------------------------------------------------------------
int nfcb200_iso7816_decode_batch(nfcb200_handle *h, const void *samples, int samples_on_device, int sigtype, uint32_t n_streams, uint64_t n_samples,
                                 uint32_t sample_rate, nfcb200_frame *out, uint64_t cap, uint64_t *n_out)
{
   if (!h)
      return fail(NFCB200_ERR_INVALID, "null handle");
   if (n_out)
      *n_out = 0;
   if (sigtype != NFCB200_SIG_LOGIC_F32 && sigtype != NFCB200_SIG_LOGIC_S16)
      return fail(NFCB200_ERR_INVALID, "signal type %d is not a 4-channel logic format", sigtype);
   if (sample_rate == 0)
      return fail(NFCB200_ERR_INVALID, "sample rate of 0");
   if (!samples || n_streams == 0 || n_samples == 0)
      return fail(NFCB200_ERR_INVALID, "empty batch");
   if (cap && !out)
      return fail(NFCB200_ERR_INVALID, "null frame buffer");
   if (n_samples >= 0xFFFFFFFFull)
      return fail(NFCB200_ERR_UNSUPPORTED, "streams of 2^32 - 1 samples or more exceed the 32-bit sample clock of the reference (IsoTech.h:221)");
   const bool s16 = sigtype == NFCB200_SIG_LOGIC_S16;
   const uint64_t bs = s16 ? 8 : 16;
   if (samples_on_device && ((uintptr_t) samples % bs))
      return fail(NFCB200_ERR_INVALID, "device samples not aligned to %u bytes", (unsigned) bs);

   CUDA_TRY(cudaSetDevice(h->device));
   cudaStream_t st = h->stream;
   int rc;

   // host input is staged a group of whole streams at a time (about 1 GB); a group's streams are the edge pass's grid.y
   const uint64_t streamBytes = n_samples * bs;
   const uint64_t maxGroup = samples_on_device ? n_streams : std::max<uint64_t>(1, (1ull << 30) / streamBytes);
   const uint32_t chunkStreams = (uint32_t) std::min<uint64_t>(std::min<uint64_t>(n_streams, maxGroup), 65535);
   const uint32_t nTiles = (uint32_t) ((n_samples + ISO_TILE - 1) / ISO_TILE);
   const uint64_t chunkTiles = (uint64_t) chunkStreams * nTiles;
   if (!samples_on_device && (rc = h->isoIn.reserve((uint64_t) chunkStreams * streamBytes)))
      return rc;
   if ((rc = h->isoClkCount.reserve(chunkTiles * 4)) || (rc = h->isoLineCount.reserve(chunkTiles * 4)) || (rc = h->isoCtr.reserve(8)) ||
       (rc = h->isoStreamCount.reserve((uint64_t) chunkStreams * 4)) || (rc = h->isoFirst.reserve((uint64_t) chunkStreams * 8)))
      return rc;
   uint32_t poolCap = (uint32_t) std::max<uint64_t>(1024, h->isoPool.cap / sizeof(nfcb200_frame));
   if ((rc = h->isoPool.reserve((uint64_t) poolCap * sizeof(nfcb200_frame))))
      return rc;

   uint64_t nf = 0; // frames of the chunks so far
   std::vector<uint32_t> streamCount(chunkStreams);
   std::vector<uint64_t> first(chunkStreams);
   for (uint32_t s0 = 0; s0 < n_streams; s0 += chunkStreams)
   {
      const uint32_t sc = std::min(chunkStreams, n_streams - s0);
      IsoEdgesArgs E = {};
      if (samples_on_device)
         E.samples = (const unsigned char *) samples + (uint64_t) s0 * streamBytes;
      else
      {
         CUDA_TRY(cudaMemcpyAsync(h->isoIn.ptr, (const unsigned char *) samples + (uint64_t) s0 * streamBytes, (uint64_t) sc * streamBytes,
                                  cudaMemcpyHostToDevice, st));
         E.samples = h->isoIn.ptr;
      }
      E.n_samples = n_samples;
      E.n_tiles = nTiles;
      E.line_count = h->isoLineCount.as<uint32_t>();
      E.clk_count = h->isoClkCount.as<uint32_t>();
      E.overflow = h->isoCtr.as<uint32_t>() + 1;
      // the dense pass, again with room for a line event and a CLK falling edge at every sample when a tile overflows
      // the first try's slots
      for (E.line_cap = ISO_LINE_CAP, E.clk_cap = ISO_CLK_CAP;; E.line_cap = E.clk_cap = ISO_TILE)
      {
         if ((rc = h->isoLine.reserve((uint64_t) sc * nTiles * E.line_cap * 4)) ||
             (rc = h->isoClk.reserve((uint64_t) sc * nTiles * E.clk_cap * sizeof(uint16_t))))
            return rc;
         E.line = h->isoLine.as<uint32_t>();
         E.clk = h->isoClk.as<uint16_t>();
         CUDA_TRY(cudaMemsetAsync(E.overflow, 0, 4, st));
         const dim3 grid(nTiles, sc);
         if (s16)
            iso_edges_kernel<true><<<grid, ISO_THREADS, 0, st>>>(E);
         else
            iso_edges_kernel<false><<<grid, ISO_THREADS, 0, st>>>(E);
         CUDA_TRY(cudaGetLastError());
         uint32_t overflow = 0;
         CUDA_TRY(cudaMemcpyAsync(&overflow, E.overflow, 4, cudaMemcpyDeviceToHost, st));
         CUDA_TRY(cudaStreamSynchronize(st));
         if (!overflow || E.line_cap == ISO_TILE)
            break;
      }
      // the walk, again with a larger pool when the frames did not fit
      IsoWalkArgs W = {};
      W.n_streams = sc;
      W.stream0 = s0;
      W.n_samples = (uint32_t) n_samples;
      W.n_tiles = nTiles;
      W.line_cap = E.line_cap;
      W.clk_cap = E.clk_cap;
      W.sample_rate = sample_rate;
      W.stream_time = h->cfg.stream_time;
      W.line = E.line;
      W.line_count = E.line_count;
      W.clk = E.clk;
      W.clk_count = E.clk_count;
      W.pool_count = h->isoCtr.as<uint32_t>();
      W.stream_count = h->isoStreamCount.as<uint32_t>();
      uint32_t count = 0;
      while (true)
      {
         W.pool = h->isoPool.as<nfcb200_frame>();
         W.pool_cap = poolCap;
         CUDA_TRY(cudaMemsetAsync(W.pool_count, 0, 4, st));
         iso_walk_kernel<<<sc, 32, 0, st>>>(W);
         CUDA_TRY(cudaGetLastError());
         CUDA_TRY(cudaMemcpyAsync(&count, W.pool_count, 4, cudaMemcpyDeviceToHost, st));
         CUDA_TRY(cudaStreamSynchronize(st));
         if (count <= poolCap)
            break;
         poolCap = count;
         if ((rc = h->isoPool.reserve((uint64_t) poolCap * sizeof(nfcb200_frame))))
            return rc;
      }
      // (stream, rank in the stream): the order the reference returns each capture's frames in
      if (count && nf < cap)
      {
         CUDA_TRY(cudaMemcpy(streamCount.data(), W.stream_count, (uint64_t) sc * 4, cudaMemcpyDeviceToHost));
         uint64_t at = 0;
         for (uint32_t i = 0; i < sc; i++)
         {
            first[i] = at;
            at += streamCount[i];
         }
         if ((rc = h->isoOrdered.reserve((uint64_t) count * sizeof(nfcb200_frame))))
            return rc;
         CUDA_TRY(cudaMemcpyAsync(h->isoFirst.ptr, first.data(), (uint64_t) sc * 8, cudaMemcpyHostToDevice, st));
         const uint32_t blocks = (uint32_t) std::min<uint64_t>((count + 7) / 8, (uint64_t) h->smCount * 16);
         iso_gather_kernel<<<blocks, 256, 0, st>>>(W.pool, count, h->isoFirst.as<uint64_t>(), s0, h->isoOrdered.as<nfcb200_frame>());
         CUDA_TRY(cudaGetLastError());
         CUDA_TRY(cudaMemcpyAsync(out + nf, h->isoOrdered.ptr, std::min<uint64_t>(count, cap - nf) * sizeof(nfcb200_frame), cudaMemcpyDeviceToHost, st));
         CUDA_TRY(cudaStreamSynchronize(st));
      }
      nf += count;
   }

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
   if (!blob || size == 0)
   {
      h->haveCarryIn = false;
      return 0;
   }
   if (size != sizeof(Carry))
      return fail(NFCB200_ERR_INVALID, "carry blob of %llu bytes, expected %zu", (unsigned long long) size, sizeof(Carry));
   memcpy(&h->carryIn, blob, sizeof(Carry));
   carry_canon(h->carryIn);
   if (h->carryIn.edgeTime)
      h->carryIn.edgeTime = h->carryIn.edgeTime > clock_shift ? h->carryIn.edgeTime - clock_shift : 1;
   h->haveCarryIn = true;
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
   if (h->lastStreams != 1)
      return fail(NFCB200_ERR_INVALID, "the carry query needs a single-stream decode before it");
   CUDA_TRY(cudaSetDevice(h->device));
   cudaStream_t st = h->stream;
   Carry *dOut = h->carryDev.as<Carry>() + 1;
   u32 *dBegin = (u32 *) (h->carryDev.as<Carry>() + 2);
   carry_before_kernel<<<1, 32, 0, st>>>(h->lanes.as<LaneRec>(), h->lastLanes, h->lastCarryInUsed ? h->carryDev.as<Carry>() : nullptr,
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
      *records = h->packed.ptr;
   if (n_records)
      *n_records = h->packedCount;
   if (ext)
      *ext = h->packedExt.ptr;
   if (n_ext_chunks)
      *n_ext_chunks = h->packedExtCount;
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
   const FrameRec *recs = (const FrameRec *) records;
   const unsigned workers = (unsigned) std::max<uint64_t>(1, std::min<uint64_t>(host_workers(), n_records / 4096));
   auto work = [&](uint64_t lo, uint64_t hi) {
      for (uint64_t i = lo; i < hi; i++)
         emit_frame(h, recs[i], (const unsigned char *) ext, (size_t) n_ext_chunks * 128, recs[i].lane + stream_offset, sample_rate, out[i]);
   };
   if (workers <= 1 || n_records < 8192)
      work(0, n_records);
   else
   {
      std::vector<std::thread> pool;
      const uint64_t step = (n_records + workers - 1) / workers;
      for (unsigned w = 0; w < workers; w++)
         pool.emplace_back(work, std::min(n_records, w * step), std::min(n_records, (w + 1) * step));
      for (auto &t: pool)
         t.join();
   }
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

   auto work = [&](uint64_t lo, uint64_t hi) {
      for (uint64_t i = lo; i < hi; i++)
      {
         memcpy(head + i * headBytes, &frames[i], headBytes);
         uint32_t stream = frames[i].stream + stream_offset;
         memcpy(head + i * headBytes, &stream, 4);
         memcpy(pay + offs[i], frames[i].data, offs[i + 1] - offs[i]);
      }
   };
   const unsigned workers = (unsigned) std::max<uint64_t>(1, std::min<uint64_t>(host_workers(), n / 8192));
   if (workers <= 1)
      work(0, n);
   else
   {
      std::vector<std::thread> pool;
      const uint64_t step = (n + workers - 1) / workers;
      for (unsigned w = 0; w < workers; w++)
         pool.emplace_back(work, std::min(n, w * step), std::min(n, (w + 1) * step));
      for (auto &t: pool)
         t.join();
   }
   return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// streaming
// ---------------------------------------------------------------------------------------------------------------------
int nfcb200_stream_reset(nfcb200_handle *h)
{
   if (!h)
      return fail(NFCB200_ERR_INVALID, "null handle");
   h->sInit = false;
   h->sBase = 0;
   h->sCount = 0;
   h->sEmitted = 0;
   h->sHostTail.clear();
   h->sPending.clear();
   return 0;
}

int nfcb200_stream_pending(nfcb200_handle *h, nfcb200_frame *out, uint64_t cap, uint64_t *n_out, uint64_t *n_left)
{
   if (!h)
      return fail(NFCB200_ERR_INVALID, "null handle");
   const uint64_t deliver = std::min<uint64_t>(h->sPending.size(), out ? cap : 0);
   for (uint64_t i = 0; i < deliver; i++)
      out[i] = h->sPending[i];
   h->sPending.erase(h->sPending.begin(), h->sPending.begin() + (size_t) deliver);
   if (n_out)
      *n_out = deliver;
   if (n_left)
      *n_left = h->sPending.size();
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

   const bool flush = n == 0;

   if (flush && !h->sInit)
   {
      // nextFrames({}) on a decoder that never saw a sample: one carrier-off frame at clock -1 (NfcDecoder.cpp:449-463)
      if (cap < 1)
         return fail(NFCB200_ERR_CAPACITY, "room for the flush frame needed");
      memset(&out[0], 0, sizeof(nfcb200_frame));
      out[0].tech_type = TT_Any;
      out[0].frame_type = FT_CarrierOff;
      out[0].frame_phase = PH_Carrier;
      out[0].sample_start = out[0].sample_end = 0xFFFFFFFFull;
      if (n_out)
         *n_out = 1;
      return 0;
   }

   // a sample-rate (or format) change re-initialises the decoder (NfcDecoder.cpp:383-388)
   if (!flush && (!h->sInit || h->sRate != sample_rate || h->sSig != sigtype))
   {
      nfcb200_stream_reset(h);
      int rc = 0;
      if (h->paramsRate != sample_rate)
         rc = setup_params(h, sample_rate);
      if (rc)
         return rc;

      rc = h->sState.reserve(sizeof(StreamState));
      rc = rc ? rc : h->sScratch.reserve(NFCB200_SCRATCH_FLOATS * sizeof(float));
      rc = rc ? rc : h->sSbuf.reserve(512);
      rc = rc ? rc : h->counters.reserve(sizeof(Counters));
      if (rc)
         return rc;

      StreamState init;
      memset(&init, 0, sizeof(init));
      carry_init(init.carry, h->P);
      carry_canon(init.carry);
      CUDA_TRY(cudaMemcpyAsync(h->sState.ptr, &init, sizeof(init), cudaMemcpyHostToDevice, st));
      CUDA_TRY(cudaMemsetAsync(h->sScratch.ptr, 0, NFCB200_SCRATCH_FLOATS * sizeof(float), st));
      CUDA_TRY(cudaStreamSynchronize(st));

      h->sRate = sample_rate;
      h->sSig = sigtype;
      h->sInit = true;
   }
   else if (h->paramsRate != h->sRate)
   {
      int rc = setup_params(h, h->sRate);
      if (rc)
         return rc;
   }

   const u32 bs = sig_bytes(h->sSig);

   // The streaming lane keeps absolute sample positions in 32 bits like the reference's signalClock (NfcTech.h:338).  The
   // reference wraps silently after 2^32 samples (7 minutes at 10 MS/s); here the position space must not wrap (retention and
   // the flag window are indexed by it), so the stream refuses further samples with an explicit error instead of stalling.
   if ((uint64_t) h->sBase + h->sCount + n >= 0xFFFF0000ull)
      return fail(NFCB200_ERR_UNSUPPORTED, "stream position would pass 2^32 samples: call nfcb200_stream_reset (the reference's 32-bit sample clock wraps here)");

   // retained host-side tail + new samples -> device buffer covering absolute samples [sBase, sBase + sCount + n)
   const u32 newCount = h->sCount + (u32) n;
   {
      int rc = h->sSamples.reserve((size_t) newCount * bs + 64);
      if (rc)
         return rc;
   }
   if (h->sCount)
      CUDA_TRY(cudaMemcpyAsync(h->sSamples.ptr, h->sHostTail.data(), (size_t) h->sCount * bs, cudaMemcpyHostToDevice, st));
   if (n)
      CUDA_TRY(cudaMemcpyAsync((unsigned char *) h->sSamples.ptr + (size_t) h->sCount * bs, samples, (size_t) n * bs, cudaMemcpyHostToDevice, st));

   // host copy of the buffer for the next retention step
   {
      std::vector<unsigned char> merged((size_t) newCount * bs);
      if (h->sCount)
         memcpy(merged.data(), h->sHostTail.data(), (size_t) h->sCount * bs);
      if (n)
         memcpy(merged.data() + (size_t) h->sCount * bs, samples, (size_t) n * bs);
      h->sHostTail.swap(merged);
   }
   h->sCount = newCount;

   // the buffer always starts on a block boundary, so buffer block i is absolute block sBase / 256 + i
   const u32 n_blocks = (newCount + NFCB200_BLOCK - 1) / NFCB200_BLOCK;
   const u32 tiles = (newCount + SCR_TILE - 1) / SCR_TILE;

   if (newCount)
   {
      int rc = h->sFlags.reserve(n_blocks);
      rc = rc ? rc : h->sBsum.reserve((size_t) n_blocks * sizeof(float));
      rc = rc ? rc : h->sCounts.reserve(sizeof(u32) * 2);
      if (rc)
         return rc;

      ScreenConfig sc;
      memset(&sc, 0, sizeof(sc));
      sc.samples = h->sSamples.ptr;
      sc.n_samples = newCount;
      sc.n_streams = 1;
      sc.sigtype = h->sSig;
      sc.n_blocks = n_blocks;
      sc.tiles_per_stream = tiles;
      sc.flags = h->sFlags.as<uint8_t>();
      sc.bsum = h->sBsum.as<float>();
      fill_screen_config(h, sc);
      if ((((uintptr_t) sc.samples) & 15) || (((uint64_t) newCount * bs) & 15))
         sc.use_tma = 0;

      launch_screen(h, sc, tiles, st);
      CUDA_TRY(cudaGetLastError());

      SegmentConfig sg;
      memset(&sg, 0, sizeof(sg));
      sg.flags = h->sFlags.as<uint8_t>();
      sg.bsum = h->sBsum.as<float>();
      sg.n_streams = 1;
      sg.n_blocks = n_blocks;
      sg.n_samples = newCount;
      sg.counts = h->sCounts.as<u32>();
      sg.low = h->P.lowThr;
      sg.high = h->P.highThr;
      sg.meanW = powf(h->P.meanW0, (float) NFCB200_BLOCK);
      // note: the stream-start margin of blocks_activate applies to buffer block 0; at the true stream start that is
      // exactly the reference start, later it only makes a few retained blocks active (harmless)
      sg.segTotal = &h->counters.as<Counters>()->segTotal;
      const u32 bgrid = (n_blocks + 255) / 256;
      segment_flags_kernel<<<bgrid, 256, 0, st>>>(sg);
      segment_activate_kernel<<<bgrid, 256, 0, st>>>(sg);
      CUDA_TRY(cudaGetLastError());
   }

   // frame pool for this push
   const u32 poolCap = 1u << 14, extCap = 1u << 12;
   {
      int rc = h->pool.reserve((size_t) poolCap * sizeof(FrameRec));
      rc = rc ? rc : h->ext.reserve((size_t) extCap * 128);
      if (rc)
         return rc;
   }
   Counters *dC = h->counters.as<Counters>();
   CUDA_TRY(cudaMemsetAsync(dC, 0, sizeof(Counters), st));

   StreamConfig cfg;
   memset(&cfg, 0, sizeof(cfg));
   cfg.samples = h->sSamples.ptr;
   cfg.base = h->sBase;
   cfg.count = newCount;
   cfg.sigtype = h->sSig;
   cfg.flags = h->sFlags.as<uint8_t>();
   cfg.flagBase = h->sBase / NFCB200_BLOCK;
   cfg.flagCount = n_blocks;
   cfg.limit = h->sBase + newCount;
   cfg.final = flush ? 1 : 0;
   cfg.state = h->sState.as<StreamState>();
   cfg.scratch = h->sScratch.as<float>();
   cfg.sbuf = h->sSbuf.as<uint8_t>();
   cfg.pool.recs = h->pool.as<FrameRec>();
   cfg.pool.cap = poolCap;
   cfg.pool.count = &dC->poolCount;
   cfg.pool.ext = h->ext.as<u8>();
   cfg.pool.extCap = extCap;
   cfg.pool.extCount = &dC->extCount;

   stream_kernel<<<1, 32, 0, st>>>(cfg, h->P);
   CUDA_TRY(cudaGetLastError());

   Counters hc;
   StreamState hs;
   CUDA_TRY(cudaMemcpyAsync(&hc, dC, sizeof(Counters), cudaMemcpyDeviceToHost, st));
   CUDA_TRY(cudaMemcpyAsync(&hs, h->sState.ptr, sizeof(StreamState), cudaMemcpyDeviceToHost, st));
   CUDA_TRY(cudaStreamSynchronize(st));

   if (hc.poolCount > poolCap || hc.extCount > extCap)
      return fail(NFCB200_ERR_CAPACITY, "stream frame pool exhausted");

   std::vector<FrameRec> recs(hc.poolCount);
   std::vector<unsigned char> ext((size_t) hc.extCount * 128);
   if (hc.poolCount)
      CUDA_TRY(cudaMemcpy(recs.data(), h->pool.ptr, (size_t) hc.poolCount * sizeof(FrameRec), cudaMemcpyDeviceToHost));
   if (hc.extCount)
      CUDA_TRY(cudaMemcpy(ext.data(), h->ext.ptr, ext.size(), cudaMemcpyDeviceToHost));

   std::sort(recs.begin(), recs.end(), [](const FrameRec &a, const FrameRec &b) { return a.seq < b.seq; });

   // frames go through a pending list: what does not fit the caller's buffer is delivered by the next call, not lost
   for (const FrameRec &r: recs)
   {
      h->sPending.emplace_back();
      emit_frame(h, r, ext.data(), ext.size(), 0, h->sRate, h->sPending.back());
   }

   if (flush)
   {
      // nextFrames({}): one carrier frame at the current clock (NfcDecoder.cpp:449-463)
      u32 clock = hs.pos - 1;
      bool on = hs.running ? hs.L.c.carrierOn != 0 : hs.carry.carrierOn != 0;
      h->sPending.emplace_back();
      nfcb200_frame &o = h->sPending.back();
      memset(&o, 0, sizeof(o));
      o.tech_type = TT_Any;
      o.frame_type = on ? FT_CarrierOn : FT_CarrierOff;
      o.frame_phase = PH_Carrier;
      o.sample_start = o.sample_end = clock;
      o.sample_rate = h->sRate;
      o.time_start = o.time_end = (double) clock / (double) h->sRate;
      o.date_time = (double) h->P.streamTime + o.time_start;
   }

   const uint64_t nf = h->sPending.size();
   const uint64_t deliver = std::min<uint64_t>(nf, cap);
   for (uint64_t i = 0; i < deliver; i++)
      out[i] = h->sPending[i];
   h->sPending.erase(h->sPending.begin(), h->sPending.begin() + (size_t) deliver);

   // retention: keep what the parked / running lane can still need.  A running lane only reads forward (its history is in
   // its rings); a parked lane may cold start HALO samples before a later active block or be resumed at pos.
   {
      u32 keepFrom = hs.pos > NFCB200_HALO + 2 * NFCB200_BLOCK ? hs.pos - NFCB200_HALO - 2 * NFCB200_BLOCK : 0;
      if (hs.running)
         keepFrom = hs.pos > SCR_HALO + NFCB200_BLOCK ? hs.pos - SCR_HALO - NFCB200_BLOCK : 0; // screening history only
      keepFrom &= ~(u32) (NFCB200_BLOCK - 1); // block aligned
      if (keepFrom < h->sBase)
         keepFrom = h->sBase;
      u32 drop = keepFrom - h->sBase;
      if (drop)
      {
         h->sHostTail.erase(h->sHostTail.begin(), h->sHostTail.begin() + (size_t) drop * bs);
         h->sBase += drop;
         h->sCount -= drop;
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
