/*
 * nfc_screen.cuh -- K1: the dense, HBM-bound pass over every sample of every capture stream.
 *
 * Fuses, per tile of one stream, what the reference does one sample at a time on the CPU for every idle sample
 * (85 % of its run time, SURVEY.md 3.1):
 *   IQ -> magnitude                 sqrtf(I*I + Q*Q)                     RadioDeviceTask.cpp:627-637
 *   DC-removal IIR edge signal      w = x - x[-1] + 0.9 w[-1]            NfcTech.cpp:56-62      (NFC-B detector input)
 *   half-symbol moving sums         C[t] = sum x[t-p2+1 .. t]            NfcA.cpp:246-250 (A x3 rates, F x2 share them)
 *   sliding correlators             S0 - S1 = C[t] - 2 C[t-(p1-p2)] + C[t-1]   NfcA.cpp:253-255, NfcF.cpp:247-249
 *   NFC-V pulse correlator          C[t-(p1-p2)] - C[t]                  NfcV.cpp:274
 * and tests them against the detectors' trigger thresholds with a safety margin.  The moving sums are differences of
 * a mean-removed block prefix sum (warp-shuffle scan), the IIR is an affine warp scan.  The kernel writes 5 bytes per
 * 256-sample block (trigger flag + block sum) and never materialises magnitude or features in HBM: algorithmic traffic
 * is one read of the input (8 B / sample for float2 IQ).
 *
 * Input tiles are staged into shared memory by the TMA engine (cp.async.bulk, 1-D) under an mbarrier, double
 * buffered, one persistent CTA per SM slot.
 *
 * The screen is CONSERVATIVE, not exact: any sample on which a reference detector could leave its idle state lies in
 * a flagged block (margins: thresholds x 0.9 against the block envelope, +-blocks dilation in nfc_chain.h).  The exact
 * decisions are taken by the lanes (nfc_decode.cuh) on the flagged regions only.
 */
#ifndef NFCB200_SCREEN_CUH
#define NFCB200_SCREEN_CUH

#include <cuda_runtime.h>
#include <stdint.h>

#include "nfc_chain.h"

namespace nfcb200 {

// sample formats accepted at the boundary (hw/SignalType.h:27-36 for 1 and 2; 3 and 4 are WAV ingest, RecordDevice.cpp:281-311)
enum { SIG_IQ_F32 = 1, SIG_MAG_F32 = 2, SIG_MAG_S16 = 3, SIG_IQ_S16 = 4 };

__host__ __device__ constexpr inline uint32_t sig_bytes(int sigtype)
{
   return sigtype == SIG_IQ_F32 ? 8 : sigtype == SIG_MAG_F32 ? 4 : sigtype == SIG_MAG_S16 ? 2 : 4;
}

// exact magnitude of one sample (reference operation order, no FMA: the unit is compiled with -fmad=false)
__device__ __forceinline__ float sample_from_raw(const void *tile, int sigtype, uint32_t i)
{
   switch (sigtype)
   {
      case SIG_IQ_F32:
      {
         float2 v = ((const float2 *) tile)[i];
         return sqrtf(v.x * v.x + v.y * v.y);
      }
      case SIG_MAG_F32:
         return ((const float *) tile)[i];
      case SIG_MAG_S16:
         return (float) ((const short *) tile)[i] / 32768.0f;
      default:
      {
         short2 v = ((const short2 *) tile)[i];
         float I = (float) v.x / 32768.0f, Q = (float) v.y / 32768.0f;
         return sqrtf(I * I + Q * Q);
      }
   }
}

// magnitude for SCREENING only: one fused multiply-add and the approximate square root (MUFU) instead of the IEEE
// sequence; the exact decoder lanes recompute the magnitude with sample_from_raw / load_sample
__device__ __forceinline__ float approx_sqrt(float p)
{
   float r;
   asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(p));
   return r;
}

template <int SIG>
__device__ __forceinline__ float screen_mag(const void *tile, uint32_t i)
{
   if (SIG == SIG_IQ_F32)
   {
      float2 v = ((const float2 *) tile)[i];
      return approx_sqrt(__fmaf_rn(v.y, v.y, v.x * v.x));
   }
   else if (SIG == SIG_MAG_F32)
   {
      return ((const float *) tile)[i];
   }
   else if (SIG == SIG_MAG_S16)
   {
      return (float) ((const short *) tile)[i] * (1.0f / 32768.0f);
   }
   else
   {
      short2 v = ((const short2 *) tile)[i];
      float I = (float) v.x * (1.0f / 32768.0f), Q = (float) v.y * (1.0f / 32768.0f);
      return approx_sqrt(__fmaf_rn(Q, Q, I * I));
   }
}

#define SCR_THREADS 256
#define SCR_WARPS (SCR_THREADS / 32)
#define SCR_PER_THREAD 17
#define SCR_SPAN (SCR_THREADS * SCR_PER_THREAD)   /* 4352 samples staged per tile            */
#define SCR_HALO 512                               /* history before the tile's own samples   */
#define SCR_TILE (SCR_SPAN - SCR_HALO)             /* 3840 = 15 blocks of 256 own samples     */
#define SCR_TILE_BLOCKS (SCR_TILE / NFCB200_BLOCK)
#define SCR_WARP_SPAN (32 * SCR_PER_THREAD)        /* 544 consecutive samples per warp        */

struct ScreenConfig
{
   const void *samples;    // [n_streams][n_samples] of sigtype
   uint64_t n_samples;     // per stream
   uint32_t n_streams;
   int sigtype;
   uint32_t n_blocks;      // blocks per stream
   uint32_t tiles_per_stream;
   uint8_t *flags;         // [n_streams][n_blocks]
   float *bsum;            // [n_streams][n_blocks] block sums of x
   // correlator geometry (samples): A/F rates 106, 212, 424 and NFC-V
   uint32_t p1[3], p2[3];
   uint32_t vp1, vp2;
   float thrA[3];          // |C[t] - C[t-q]| > thrA[r] * envelope flags rate r (see the derivation in the kernel)
   float thrV;             // same for the NFC-V pulse correlator
   float kB;               // |w| > kB * envelope flags an NFC-B edge
   float quiet;            // a warp span whose sample range is <= quiet * (its minimum) cannot trigger any test
   int use_tma;
};

// ---- mbarrier / TMA bulk copy (PTX; SASS: SYNCS.*, UBLKCP) ---------------------------------------------------------

__device__ __forceinline__ uint32_t smem_u32(const void *p)
{
   return (uint32_t) __cvta_generic_to_shared(p);
}

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
   asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}

__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
   asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}

__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
   asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "NFCB200_WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra NFCB200_DONE_%=;\n"
      "bra NFCB200_WAIT_%=;\n"
      "NFCB200_DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}

__device__ __forceinline__ void tma_load_1d(void *dst, const void *src, uint32_t bytes, uint64_t *bar)
{
   asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes),
                "r"(smem_u32(bar))
                : "memory");
}

// warp-wide min / max of a float through the integer reduction unit (redux.sync): order-preserving key
__device__ __forceinline__ uint32_t float_key(float f)
{
   uint32_t u = __float_as_uint(f);
   return u ^ ((uint32_t) ((int32_t) u >> 31) | 0x80000000u);
}

__device__ __forceinline__ float key_float(uint32_t k)
{
   uint32_t u = (k & 0x80000000u) ? (k ^ 0x80000000u) : ~k;
   return __uint_as_float(u);
}

// ---- the kernel --------------------------------------------------------------------------------------------------------

struct ScreenSmem
{
   // raw staging, two stages, 16-byte aligned; sized for the widest format (float2)
   unsigned char raw[2][SCR_SPAN * 8];
   float P[2][SCR_SPAN + 1];    // inclusive prefix sum of the staged magnitudes, P[.][0] = 0 (two buffers: DB variant)
   float warpAgg[SCR_WARPS];    // sum of every warp's 544 samples
   float warpW[SCR_WARPS];      // IIR state at the end of every warp's span
   float warpMin[SCR_WARPS], warpMax[SCR_WARPS];
   uint32_t blockHit[2][SCR_TILE_BLOCKS + 1];
   uint64_t bar[2];
};

struct ScreenTaps
{
   int p20, q0, p21, q1, p22, q2, pv, qv;
   float t0, t1, t2, tv, tb;
};

// 0.9^(i+1): what is left after i + 1 samples of the IIR state that entered a thread's chunk
__device__ __forceinline__ constexpr float iir_decay(int i)
{
   constexpr float d[SCR_PER_THREAD] = {0.9f,          0.81f,         0.729f,        0.6561f,       0.59049f,      0.531441f,
                                        0.4782969f,    0.43046721f,   0.387420489f,  0.3486784401f, 0.3138105961f, 0.2824295365f,
                                        0.2541865828f, 0.2287679245f, 0.2058911321f, 0.1853020189f, 0.166771817f};
   return d[i];
}

#define SCR_IIR_CHUNK 0.166771817f /* 0.9^17: decay of the IIR state over one thread chunk */

// envelope reference of tile block b: min(mean of the block, mean of the previous block) -- in idle both equal the
// reference's envelope EMA to within the noise; during a pause the smaller one only makes the tests stricter
__device__ __forceinline__ float block_env(const float *P, int b)
{
   const int bslot = SCR_HALO + (b << 8);
   const float p0 = P[bslot - NFCB200_BLOCK], p1 = P[bslot], p2 = P[bslot + NFCB200_BLOCK];
   const float env = fminf(p2 - p1, p1 - p0) * (1.0f / NFCB200_BLOCK);
   return env < 0 ? 0 : env;
}

/*
 * Trigger tests of one thread's 17 consecutive own samples, branch-free.
 * Evaluation density: 424k window every sample, 212k at chunk offsets 0, 2, .., 16, 106k at 0, 4, .., 16, NFC-V at 0, 8,
 * 16 (the gap to the next chunk's offset 0 is one sample) -- the thresholds were lowered on the host by the change
 * |C[t] - C[t - q]| can undergo between evaluations (2 xmax per sample).  Chunk-relative phases keep every warp uniform.
 * The chunk spans at most two screening blocks: their envelope-scaled thresholds are formed once and selected per sample.
 */
__device__ __forceinline__ void screen_tests(const float *Pbase, uint32_t *blockHit, const ScreenTaps &tp, int first, float wCarry,
                                             const float (&wl)[SCR_PER_THREAD])
{
   const int blkA = (first - SCR_HALO) >> 8;
   const int blkB = (first + SCR_PER_THREAD - 1 - SCR_HALO) >> 8;
   const int split = SCR_HALO + (blkB << 8) - first; // samples i < split belong to blkA (split >= 17 when blkA == blkB)
   const float envA = block_env(Pbase, blkA), envB = blkB == blkA ? envA : block_env(Pbase, blkB);

   const float bA = tp.tb * envA, bB = tp.tb * envB;
   const float a2A = tp.t2 * envA, a2B = tp.t2 * envB;
   const float a1A = tp.t1 * envA, a1B = tp.t1 * envB;
   const float a0A = tp.t0 * envA, a0B = tp.t0 * envB;
   const float avA = tp.tv * envA, avB = tp.tv * envB;

   const float *P = Pbase + first + 1; // P[i] = inclusive prefix at the chunk's i-th sample

   bool hitA = false, hitB = false;

#pragma unroll
   for (int i = 0; i < SCR_PER_THREAD; i++)
   {
      const bool inA = i < split;
      const float Pt = P[i];

      bool hit = fabsf(__fmaf_rn(iir_decay(i), wCarry, wl[i])) > (inA ? bA : bB);

      hit |= fabsf((Pt - P[i - tp.p22]) - (P[i - tp.q2] - P[i - tp.q2 - tp.p22])) > (inA ? a2A : a2B);

      if ((i & 1) == 0)
         hit |= fabsf((Pt - P[i - tp.p21]) - (P[i - tp.q1] - P[i - tp.q1 - tp.p21])) > (inA ? a1A : a1B);

      if ((i & 3) == 0)
         hit |= fabsf((Pt - P[i - tp.p20]) - (P[i - tp.q0] - P[i - tp.q0 - tp.p20])) > (inA ? a0A : a0B);

      if ((i & 7) == 0)
         hit |= fabsf((Pt - P[i - tp.pv]) - (P[i - tp.qv] - P[i - tp.qv - tp.pv])) > (inA ? avA : avB);

      hitA |= hit && inA;
      hitB |= hit && !inA;
   }

   if (hitA)
      blockHit[blkA] = 1; // benign race: all writers store 1
   if (hitB)
      blockHit[blkB] = 1;
}

// work item -> (stream, tile); staged range in samples [lo, hi) clipped to the stream, `base` = index of smem slot 0
struct TileGeom
{
   uint32_t stream, tile;
   int64_t base;  // sample index of staged slot 0 (may be negative for tile 0)
   int64_t lo, hi; // valid samples [lo, hi)
};

__device__ __forceinline__ TileGeom tile_geom(const ScreenConfig &c, uint32_t stream, uint32_t tile)
{
   TileGeom g;
   g.stream = stream;
   g.tile = tile;
   g.base = (int64_t) g.tile * SCR_TILE - SCR_HALO;
   g.lo = g.base < 0 ? 0 : g.base;
   g.hi = g.base + SCR_SPAN;
   if (g.hi > (int64_t) c.n_samples)
      g.hi = (int64_t) c.n_samples;
   return g;
}

template <int SIG>
__device__ __forceinline__ void tile_issue(const ScreenConfig &c, ScreenSmem &s, int stage, uint32_t stream, uint32_t tile)
{
   // one elected thread arms the barrier and launches the bulk copy of the valid part of the tile
   TileGeom g = tile_geom(c, stream, tile);
   constexpr uint32_t bs = sig_bytes(SIG);
   const unsigned char *src = (const unsigned char *) c.samples + ((uint64_t) g.stream * c.n_samples + (uint64_t) g.lo) * bs;
   uint32_t bytes = (uint32_t) (g.hi - g.lo) * bs;
   uint32_t dstoff = (uint32_t) (g.lo - g.base) * bs;
   // cp.async.bulk needs 16-byte aligned addresses and sizes: the head is aligned by construction (tile and halo are
   // multiples of 8 samples, stream pitch checked on the host); a ragged tail is finished with plain loads below
   uint32_t bulk = bytes & ~15u;
   mbar_expect_tx(&s.bar[stage], bulk);
   if (bulk)
      tma_load_1d(s.raw[stage] + dstoff, src, bulk, &s.bar[stage]);
}

/*
 * One persistent CTA walks the work items (stream, tile) blockIdx.x, blockIdx.x + gridDim.x, ...  Per tile:
 *   phase 1  every thread: 17 magnitudes from the staged raw tile, thread-local prefix sum / IIR / min / max, warp scans
 *   phase 2  cross-warp carries, prefix sums to shared memory, the warp's QUIET test
 *   phase 3  warps that are not quiet: envelope per block, the sliding correlator and edge tests (shared-memory taps)
 *   phase 4  15 threads write the tile's block flags and block sums
 * Quiet test: every quantity phase 3 compares is bounded by the range of the samples it covers --
 *   |C[t] - C[t-q]| <= p2 (max - min),   |w| <= max - min (w = x minus a weighted average of its past) --
 * and every threshold is a multiple of a block mean >= min.  All taps of a warp's samples (<= 283 back), the means of
 * their blocks (<= 511 back, <= 255 ahead) and the IIR memory (0.9^544 = 1e-25) lie within the warp's own span, the
 * previous and the next one, so with hi / lo taken over those three spans no test can fire when hi - lo <= quiet * lo
 * (quiet = 0.999 min(kB, thrA[r] / p2[r], thrV / vp2), host side).  On an idle carrier that is every warp.
 */
// phase 4: block flags and block sums of one tile (15 threads)
__device__ __forceinline__ void screen_write_blocks(const ScreenConfig &c, const TileGeom &g, const float *P, uint32_t *blockHit, int tid)
{
   if (tid < SCR_TILE_BLOCKS)
   {
      const uint32_t b = g.tile * SCR_TILE_BLOCKS + tid;
      const uint32_t hit = blockHit[tid];
      blockHit[tid] = 0; // the next tests into this buffer are at least two barriers away
      if (b < c.n_blocks)
      {
         const int bslot = SCR_HALO + (tid << 8);
         c.flags[(uint64_t) g.stream * c.n_blocks + b] = hit ? SCR_TRIGGER : 0;
         // block sum of x over the samples that exist (the replicated tail contributes nothing real: the last block
         // of a stream is always active through the trailing margin, so its sum is only used for the envelope)
         c.bsum[(uint64_t) g.stream * c.n_blocks + b] = P[bslot + NFCB200_BLOCK] - P[bslot];
      }
   }
}

/*
 * DB = true: the prefix sums and block hits are double buffered, so the barrier between the tests of a tile (phase 3) and
 * its block output (phase 4) disappears -- phase 4 of tile i runs after the first barrier of tile i + 1, which every
 * thread reaches only after its phase 3 of tile i.  Warps that are quiet start the next tile while the warps inside a
 * frame are still testing (that barrier was 23 % of the kernel's stall samples).
 */
template <int SIG, bool DB>
__global__ void __launch_bounds__(SCR_THREADS, 2) screen_kernel(ScreenConfig c, uint32_t n_items)
{
   extern __shared__ __align__(128) unsigned char smem_raw[];
   ScreenSmem &s = *reinterpret_cast<ScreenSmem *>(smem_raw);

   const int tid = threadIdx.x;
   const int lane = tid & 31;
   const int warp = tid >> 5;
   constexpr uint32_t bs = sig_bytes(SIG);

   if (c.use_tma && tid == 0)
   {
      mbar_init(&s.bar[0], 1);
      mbar_init(&s.bar[1], 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
   }
   if (tid <= SCR_TILE_BLOCKS)
   {
      s.blockHit[0][tid] = 0;
      s.blockHit[1][tid] = 0;
   }
   __syncthreads();

   // (stream, tile) of the current item, advanced without divisions
   const uint32_t tps = c.tiles_per_stream;
   const uint32_t stepS = gridDim.x / tps, stepT = gridDim.x % tps;
   uint32_t stream = blockIdx.x / tps, tile = blockIdx.x % tps;

   uint32_t item = blockIdx.x;
   uint32_t phaseBits = 0; // bit s: parity the barrier of stage s completes next
   int stage = 0;

   if (c.use_tma && tid == 0 && item < n_items)
      tile_issue<SIG>(c, s, 0, stream, tile);

   ScreenTaps tp;
   tp.p20 = (int) c.p2[0];
   tp.q0 = (int) (c.p1[0] - c.p2[0]);
   tp.p21 = (int) c.p2[1];
   tp.q1 = (int) (c.p1[1] - c.p2[1]);
   tp.p22 = (int) c.p2[2];
   tp.q2 = (int) (c.p1[2] - c.p2[2]);
   tp.pv = (int) c.vp2;
   tp.qv = (int) (c.vp1 - c.vp2);
   tp.t0 = c.thrA[0];
   tp.t1 = c.thrA[1];
   tp.t2 = c.thrA[2];
   tp.tv = c.thrV;
   tp.tb = c.kB;

   TileGeom prevG = tile_geom(c, stream, tile); // DB: the tile whose block output is still pending
   bool havePrev = false;

   for (; item < n_items; item += gridDim.x, stage ^= 1)
   {
      const TileGeom g = tile_geom(c, stream, tile);
      float *P = s.P[DB ? stage : 0];
      uint32_t *blockHit = s.blockHit[DB ? stage : 0];

      // next item
      uint32_t nstream = stream + stepS, ntile = tile + stepT;
      if (ntile >= tps)
      {
         ntile -= tps;
         nstream++;
      }

      const uint32_t bytes = (uint32_t) (g.hi - g.lo) * bs;
      const uint32_t bulk = bytes & ~15u;

      if (c.use_tma)
      {
         // prefetch the next tile into the other stage (every thread finished reading it: it passed the last barrier of
         // the previous iteration after its phase 1), then wait for this one
         if (tid == 0 && item + gridDim.x < n_items)
            tile_issue<SIG>(c, s, stage ^ 1, nstream, ntile);

         mbar_wait(&s.bar[stage], (phaseBits >> stage) & 1u);
         phaseBits ^= 1u << stage;

         // ragged tail (< 16 bytes) of the last tile of a stream
         if (bytes != bulk)
         {
            if (tid < (int) (bytes - bulk))
            {
               const unsigned char *src = (const unsigned char *) c.samples + ((uint64_t) g.stream * c.n_samples + (uint64_t) g.lo) * bs;
               s.raw[stage][(uint32_t) (g.lo - g.base) * bs + bulk + tid] = src[bulk + tid];
            }
            __syncthreads();
         }
      }
      else
      {
         // plain coalesced 16-byte loads (debug knob; same staging layout).  This path also serves batches whose stream
         // pitch is not a multiple of 16 bytes, where a stream after the first starts unaligned: bytes one at a time
         const unsigned char *src = (const unsigned char *) c.samples + ((uint64_t) g.stream * c.n_samples + (uint64_t) g.lo) * bs;
         unsigned char *dst = s.raw[stage] + (uint32_t) (g.lo - g.base) * bs;
         uint32_t vec = (((uintptr_t) src | (uintptr_t) dst) & 15) ? 0 : bytes >> 4;
         for (uint32_t i = tid; i < vec; i += SCR_THREADS)
            ((uint4 *) dst)[i] = __ldg(((const uint4 *) src) + i);
         for (uint32_t i = (vec << 4) + tid; i < bytes; i += SCR_THREADS)
            dst[i] = src[i];
         __syncthreads();
      }

      // ---- phase 1: per-thread chunk: magnitude, local prefix, local IIR, range -------------------------------------
      const int validLo = (int) (g.lo - g.base); // slots below hold no data (stream start): replicate the first sample
      const int validHi = (int) (g.hi - g.base); // slots at / above hold no data (stream end): replicate the last sample
      const void *raw = s.raw[stage];
      const bool whole = validLo == 0 && validHi == SCR_SPAN;

      float xs[SCR_PER_THREAD];
      const int first = tid * SCR_PER_THREAD;
      float prevx; // x[first - 1] (the chunk's own first sample at the very start of the tile: w starts from zero)

      if (whole)
      {
#pragma unroll
         for (int i = 0; i < SCR_PER_THREAD; i++)
            xs[i] = screen_mag<SIG>(raw, (uint32_t) (first + i));
         prevx = screen_mag<SIG>(raw, (uint32_t) (first ? first - 1 : 0));
      }
      else
      {
#pragma unroll
         for (int i = 0; i < SCR_PER_THREAD; i++)
         {
            int slot = first + i;
            slot = slot < validLo ? validLo : (slot >= validHi ? validHi - 1 : slot);
            xs[i] = screen_mag<SIG>(raw, (uint32_t) slot);
         }
         int slot = first ? first - 1 : 0;
         slot = slot < validLo ? validLo : (slot >= validHi ? validHi - 1 : slot);
         prevx = screen_mag<SIG>(raw, (uint32_t) slot);
      }

      // thread-local inclusive prefix, IIR from a zero state, minimum and maximum
      float loc[SCR_PER_THREAD], wl[SCR_PER_THREAD];
      float run = 0, w = 0, mn = xs[0], mx = xs[0];
#pragma unroll
      for (int i = 0; i < SCR_PER_THREAD; i++)
      {
         run += xs[i];
         loc[i] = run;
         w = __fmaf_rn(w, 0.9f, xs[i] - prevx); // w[n] = 0.9 w[n-1] + (x[n] - x[n-1])
         prevx = xs[i];
         wl[i] = w;
         mn = fminf(mn, xs[i]);
         mx = fmaxf(mx, xs[i]);
      }

      // warp scans over the 32 chunks: additive for the prefix; affine with the constant factor 0.9^17 for the IIR
      float incl = run, sW = w, fac = SCR_IIR_CHUNK;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1)
      {
         const float o = __shfl_up_sync(0xffffffffu, incl, d);
         const float ow = __shfl_up_sync(0xffffffffu, sW, d);
         if (lane >= d)
         {
            incl += o;
            sW = __fmaf_rn(fac, ow, sW);
         }
         fac *= fac;
      }

      const float wmn = key_float(__reduce_min_sync(0xffffffffu, float_key(mn)));
      const float wmx = key_float(__reduce_max_sync(0xffffffffu, float_key(mx)));

      if (lane == 31)
      {
         s.warpAgg[warp] = incl;
         s.warpW[warp] = sW; // the state that entered the warp has decayed by 0.9^544 = 1e-25: dropped
         s.warpMin[warp] = wmn;
         s.warpMax[warp] = wmx;
      }

      __syncthreads();

      if (DB && havePrev)
         screen_write_blocks(c, prevG, s.P[stage ^ 1], s.blockHit[stage ^ 1], tid); // every warp is past its tests of that tile

      // ---- phase 2: carries across warps, prefix to shared memory, quiet test ---------------------------------------
      float prefBase = 0;
#pragma unroll
      for (int v = 0; v < SCR_WARPS - 1; v++)
         prefBase += v < warp ? s.warpAgg[v] : 0.0f;

      const float exclPref = prefBase + (incl - run);

#pragma unroll
      for (int i = 0; i < SCR_PER_THREAD; i++)
         P[first + i + 1] = exclPref + loc[i];
      if (tid == 0)
         P[0] = 0;

      // IIR state entering this thread's chunk: the warp scan's value of the previous lane plus what is left of the state
      // that entered the warp, 0.9^(17 lane) (exp2 of lane * log2(0.9^17); approximate like everything in this screen)
      const float eW = __shfl_up_sync(0xffffffffu, sW, 1);
      const float wWarp = warp ? s.warpW[warp - 1] : 0.0f;
      const float wCarry = __fmaf_rn(exp2f((float) lane * -2.5840526f), wWarp, lane ? eW : 0.0f);

      // range over the previous, this and the next warp's span (the block of this warp's last samples reaches up to 255
      // samples into the next span; the last warp ends on a block boundary)
      const int wp = warp ? warp - 1 : 0, wn = warp < SCR_WARPS - 1 ? warp + 1 : warp;
      const float lo = fminf(wmn, fminf(s.warpMin[wp], s.warpMin[wn]));
      const float hi = fmaxf(wmx, fmaxf(s.warpMax[wp], s.warpMax[wn]));
      const bool quiet = (hi - lo) <= c.quiet * lo;

      __syncthreads();

      // ---- phase 3: correlators and trigger tests on the tile's own samples ------------------------------------------
      // With C[t] = P[t] - P[t - p2] (half-symbol moving sum) the reference's correlator is
      //    S0 - S1 = (C[t] - C[t - q]) - (C[t - q] - C[t - 1]) = 2 (C[t] - C[t - q]) - (x[t] - x[t - p2])
      // so  |S0 - S1| <= 2 |C[t] - C[t - q]| + xmax, and a detector needing |S0 - S1| / p2 > T env cannot trigger while
      //    |C[t] - C[t - q]| <= thr env,   thr = min(0.9 T p2, T p2 - 1.25) / 2          (xmax <= 1.25 env)
      // One difference of two moving sums (3 shared-memory taps) per rate and sample.  The long windows change slowly
      // (by at most 2 xmax per sample), so the 212k correlator is evaluated on every 2nd sample, the 106k one on every
      // 4th and the NFC-V one on every 8th, with the thresholds lowered by the possible change in between.
      if (!quiet)
      {
         const int ownEnd = (int) ((int64_t) c.n_samples - g.base); // first slot past the stream
         const int lastSlot = first + SCR_PER_THREAD - 1;

         if (first >= SCR_HALO && lastSlot < ownEnd)
         {
            // whole chunk inside the tile's own samples: branch-free tests
            screen_tests(P, blockHit, tp, first, wCarry, wl);
         }
         else if (lastSlot >= SCR_HALO && first < ownEnd)
         {
            // chunk straddling the halo boundary or the end of the stream: same tests, checked per sample, no decimation
#pragma unroll
            for (int i = 0; i < SCR_PER_THREAD; i++)
            {
               const int slot = first + i;
               if (slot < SCR_HALO || slot >= ownEnd)
                  continue;
               const int blk = (slot - SCR_HALO) >> 8;
               const float env = block_env(P, blk);
               const int t = slot + 1;
               const float Pt = P[t];
               bool hit = fabsf(__fmaf_rn(iir_decay(i), wCarry, wl[i])) > tp.tb * env;
               hit |= fabsf((Pt - P[t - tp.p20]) - (P[t - tp.q0] - P[t - tp.q0 - tp.p20])) > tp.t0 * env;
               hit |= fabsf((Pt - P[t - tp.p21]) - (P[t - tp.q1] - P[t - tp.q1 - tp.p21])) > tp.t1 * env;
               hit |= fabsf((Pt - P[t - tp.p22]) - (P[t - tp.q2] - P[t - tp.q2 - tp.p22])) > tp.t2 * env;
               hit |= fabsf((Pt - P[t - tp.pv]) - (P[t - tp.qv] - P[t - tp.qv - tp.pv])) > tp.tv * env;
               if (hit)
                  blockHit[blk] = 1;
            }
         }
      }

      if (!DB)
      {
         __syncthreads();

         // ---- phase 4: block flags and block sums of the tile ---------------------------------------------------------
         screen_write_blocks(c, g, P, blockHit, tid);
      }
      else
      {
         prevG = g;
         havePrev = true;
      }

      stream = nstream;
      tile = ntile;
      // no barrier here: P, blockHit and the warp aggregates are rewritten in phase 2 / after the first barrier of the
      // next iteration, which every thread reaches only after this phase 4
   }

   if (DB && havePrev)
   {
      __syncthreads();
      screen_write_blocks(c, prevG, s.P[stage ^ 1], s.blockHit[stage ^ 1], tid); // `stage` was flipped once more by the loop
   }
}

}

#endif
