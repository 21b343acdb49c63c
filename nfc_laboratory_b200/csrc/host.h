/*
 * host.h -- host-side plumbing shared by the translation units of libnfcb200.so (not part of the C ABI): errors, buffers
 * that own their memory, the host worker threads, staging of host input, and the handle.
 */
#ifndef NFCB200_HOST_H
#define NFCB200_HOST_H

#include <cuda_runtime.h>
#include <sched.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <type_traits>
#include <vector>

#include "../../include/nfcb200.h"
#include "nfc_params.h"

namespace nfcb200 {

// errors: the message is kept per thread for nfcb200_last_error
int fail(int code, const char *fmt, ...);

#define CUDA_TRY(expr)                                                                                              \
   do                                                                                                               \
   {                                                                                                                \
      cudaError_t e_ = (expr);                                                                                      \
      if (e_ != cudaSuccess)                                                                                        \
         return fail(NFCB200_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); \
   }                                                                                                                \
   while (0)

// buffer that only grows, freed by its owner: device memory, or pinned host memory (frame records travel device -> host
// at link speed, not through a pageable bounce)
template <bool Pinned>
struct Buf
{
   void *ptr = nullptr;
   size_t cap = 0;

   Buf() = default;
   Buf(const Buf &) = delete;
   Buf &operator=(const Buf &) = delete;
   ~Buf() { release(); }

   int reserve(size_t bytes)
   {
      if (bytes <= cap)
         return 0;
      release();
      return grow(Pinned ? bytes + bytes / 4 + 4096 : bytes + bytes / 8 + 256, 0, nullptr);
   }

   // grow, preserving the first `keep` bytes (the packed frames of the earlier chunks of one call)
   int reserve_keep(size_t bytes, size_t keep, cudaStream_t st)
   {
      static_assert(!Pinned, "reserve_keep copies device memory");
      return bytes <= cap ? 0 : grow(bytes + bytes / 2 + 256, keep, st);
   }

   template <class T>
   T *as() const
   {
      return (T *) ptr;
   }

private:
   int grow(size_t want, size_t keep, cudaStream_t st)
   {
      void *np = nullptr;
      cudaError_t e = Pinned ? cudaHostAlloc(&np, want, cudaHostAllocDefault) : cudaMalloc(&np, want);
      if (e != cudaSuccess)
         return fail(NFCB200_ERR_CUDA, "%s(%zu) failed: %s", Pinned ? "cudaHostAlloc" : "cudaMalloc", want, cudaGetErrorString(e));
      if (ptr && keep)
      {
         cudaMemcpyAsync(np, ptr, keep, cudaMemcpyDeviceToDevice, st);
         cudaStreamSynchronize(st);
      }
      release();
      ptr = np;
      cap = want;
      return 0;
   }

   void release()
   {
      if (ptr)
         Pinned ? cudaFreeHost(ptr) : cudaFree(ptr);
      ptr = nullptr;
      cap = 0;
   }
};

using DevBuf = Buf<false>;
using HostBuf = Buf<true>;

static_assert(!std::is_copy_constructible<DevBuf>::value && !std::is_copy_assignable<DevBuf>::value &&
                 !std::is_copy_constructible<HostBuf>::value && !std::is_copy_assignable<HostBuf>::value,
              "a buffer owns its memory: a copy would free it twice");

// Host threads this process may use for the conversion of frame records: the CPUs it is allowed to run on (affinity, clipped
// by a cgroup CPU quota) divided by the processes that share them (one per GPU under torchrun: LOCAL_WORLD_SIZE).  With 8
// ranks on a 16-CPU quota, 8 x 16 conversion threads exhausted the quota and the kernel throttled the whole job.
inline unsigned host_workers()
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

// fn(lo, hi) over the slices of [0, count): one per host worker, none smaller than `grain` items
template <class F>
void parallel_for(uint64_t count, uint64_t grain, const F &fn)
{
   const unsigned workers = (unsigned) std::max<uint64_t>(1, std::min<uint64_t>(host_workers(), count / grain));
   if (workers <= 1)
   {
      fn(0, count);
      return;
   }
   std::vector<std::thread> pool;
   const uint64_t step = (count + workers - 1) / workers;
   for (unsigned w = 0; w < workers; w++)
      pool.emplace_back(fn, std::min(count, w * step), std::min(count, (w + 1) * step));
   for (auto &t: pool)
      t.join();
}

// fn(s0, count, deviceSamples) for the input of a batch call, a group of whole streams at a time, at most `limit`: a
// device batch is read where it lies, all streams in one group; a host batch is copied to `staging` about 1 GB at a time
template <class F>
int for_each_stream_group(const void *samples, bool onDevice, uint32_t n_streams, uint64_t streamBytes, uint32_t limit, DevBuf &staging,
                          cudaStream_t st, const F &fn)
{
   const uint64_t fit = onDevice ? n_streams : std::max<uint64_t>(1, std::min<uint64_t>(n_streams, (1ull << 30) / streamBytes));
   const uint32_t group = (uint32_t) std::min<uint64_t>(fit, limit);
   for (uint32_t s0 = 0; s0 < n_streams; s0 += group)
   {
      const uint32_t count = std::min(group, n_streams - s0);
      const void *src = (const unsigned char *) samples + (uint64_t) s0 * streamBytes;
      if (!onDevice)
      {
         if (int rc = staging.reserve((uint64_t) group * streamBytes))
            return rc;
         CUDA_TRY(cudaMemcpyAsync(staging.ptr, src, (uint64_t) count * streamBytes, cudaMemcpyHostToDevice, st));
         src = staging.ptr;
      }
      if (int rc = fn(s0, count, src))
         return rc;
   }
   return 0;
}

// device events of an NFC batch decode: the call, a chunk's wait for its host input, then the phases of a chunk
enum { EV_CALL, EV_END, EV_COPY_WAIT, EV_COPIED, EV_SCREEN, EV_SCREENED, EV_FRONT, EV_LANES, EV_GATHER, EV_GATHERED, EV_COUNT };

} // namespace nfcb200

// the handle: what every entry point shares, then the state each group of entry points owns
struct nfcb200_handle
{
   nfcb200_config cfg;
   nfcb200::Params P;
   nfcb200::u32 paramsRate = 0;
   int device = 0;
   int smCount = 132;
   cudaStream_t stream = nullptr;

   // nfcb200_decode_batch, and the entry points that read what it left: statistics, block flags, carry, device frames
   struct NfcBatch
   {
      int wlanesPerSm = 7; // resident warp lanes per SM (shared memory: sizeof(WLaneSmem) each)
      bool stragglerAlways = false;
      nfcb200::u32 stragglerMargin = 0; // thread lanes: samples past its queued length after which a lane that holds the launch
                                        // gives up and is decoded again by a warp lane (0: never; development knob NFCB200_STRAGGLER)
      int laneBlocks = 4;               // resident thread-lane blocks per SM (lanes_kernel __launch_bounds__)
      int shortHalo = 1;                // NFCB200_HALO_SHORT=0 forces the long warm-up for every segment (measurement knob)

      cudaEvent_t ev[nfcb200::EV_COUNT] = {};
      cudaStream_t copyStream = nullptr; // host input: the copy of the next chunk overlaps the decode of this one
      cudaEvent_t copied[2] = {};
      nfcb200::DevBuf samples;           // host input staging, two chunks

      nfcb200::DevBuf flags, bsum, counts, offsets, segCounts, segOffsets, segs, feats, lanes, queue, scratch, sbuf, pool, ext, meta, counters;
      nfcb200::HostBuf hRecs, hExt;                    // gather staging
      nfcb200::DevBuf packed, packedExt, packCtr;      // frames of the current call, ordered and packed on the device (all chunks)
      uint64_t packedCount = 0;                        // records in `packed`
      nfcb200::u32 packedExtCount = 0;                 // 128-byte chunks in `packedExt`
      nfcb200_stats stats = {};

      nfcb200::DevBuf carryDev;       // injected carry (nfcb200_set_carry) / carry query result
      std::vector<unsigned char> carryIn; // host copy of the injected carry (a Carry, nfc_core.h); empty: none
      bool lastCarryInUsed = false;   // the last decode started from the injected carry
      nfcb200::u32 lastLanes = 0;     // lanes of the last single-stream decode (nfcb200_carry_before)
      nfcb200::u32 lastStreams = 0, lastBlocks = 0; // last batch geometry (for the flag tap)
   } batch;

   // nfcb200_stream_push: one live capture
   struct NfcStream
   {
      nfcb200::DevBuf state, scratch, sbuf, samples, flags, bsum, pool, ext, counters;
      nfcb200::DevBuf saved;                // state, scratch and sbuf as the current push found them
      nfcb200::u32 poolCap = 1u << 14;      // frame pool: records, 128-byte extension chunks (grown to what a push needed)
      nfcb200::u32 extCap = 1u << 12;
      std::vector<unsigned char> hostTail;  // samples retained on the host side of the stream buffer
      nfcb200::u32 base = 0;                // absolute index of the first retained sample
      nfcb200::u32 count = 0;               // retained samples
      nfcb200::u32 rate = 0;
      int sig = 0;
      bool init = false;
      std::vector<nfcb200_frame> pending;   // decoded but not yet delivered (the caller's buffer was too small)
   } strm;

   // nfcb200_spectrum: its own buffers, so that a spectrum call leaves every decode state above as it was
   struct Spectrum
   {
      nfcb200::DevBuf tables, in, out; // twiddles + window (uploaded once), staged host input, staged host output
      bool tablesReady = false;
   } spec;

   // nfcb200_adaptive_radio / nfcb200_adaptive_logic: buffers of their own too
   struct Adaptive
   {
      nfcb200::DevBuf in, count, first, out; // staged host input, points per list, their places, points of one window
      nfcb200::HostBuf hCount;               // points per list on the host
   } adapt;

   // the ISO 7816 dense pass's per-tile event slots and counts (iso_decode.cuh)
   struct IsoEvents
   {
      nfcb200::DevBuf line, lineCount, clk, clkCount;
   };

   // nfcb200_iso7816_decode_batch: its own buffers too
   struct Iso
   {
      IsoEvents ev;
      nfcb200::DevBuf in, pool, ctr, streamCount, first, ordered;
   } iso;

   // nfcb200_iso7816_stream_push: one live logic capture, beside (not instead of) the NFC stream
   struct IsoStream
   {
      IsoEvents ev;
      nfcb200::DevBuf in, pool, ctr, streamCount, state; // state: two iso7816::IsoStreamState, the current one is `cur`
      int cur = 0;
      bool init = false;                 // a buffer was pushed since the last reset
      nfcb200::u32 rate = 0;             // sample rate of the last buffer
      nfcb200::u32 clock = 0;            // samples since the decoder last (re)started: the next buffer's first sample
      float last[4] = {0, 0, 0, 0};      // the last sample pushed (IsoDecoderStatus::sampleLast), 0 before the first
      std::vector<nfcb200_frame> pending; // decoded but not yet delivered
   } isoStream;
};

#endif
