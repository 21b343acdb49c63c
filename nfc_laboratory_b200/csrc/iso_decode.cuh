/*
 * iso_decode.cuh -- ISO 7816 contact smart-card decoding of 4-channel logic captures on the device (iso_core.h).
 *
 *   iso_edges_kernel<S16>  the dense pass: one CTA per tile of ISO_TILE samples of one stream.  Every sample is read once
 *                          (one 16-byte load per float sample, one 8-byte load per int16 sample), its flags are computed
 *                          against the previous sample, and the tile writes, in sample order, its line events (IO / RST /
 *                          VCC edges: 12-bit offset | flags << 12) and the 12-bit offsets of its CLK falling edges into
 *                          per-tile slots.  Events beyond a tile's slots (`line_cap`, `clk_cap`) are counted but not
 *                          written, and the call runs the pass again with room for one of each at every sample: a
 *                          two-level clock has at most ISO_TILE / 2 falling edges per tile, but a clock with more levels
 *                          (noise, a staircase, a ramp) can fall on every sample.
 *   iso_edges_u8x4_kernel  the same pass over 8-bit samples at stride 4 (one 32-bit word per sample, 16-byte loads).
 *   iso_edges_staged_kernel<T>  the same pass at any stride 4-8 and alignment: each sub-tile of iso_sub<T>() samples is copied
 *                          to shared memory with 16-byte loads, then channels 0-3 are picked there.
 *   iso_walk_kernel        one warp per stream runs iso_walk() over the tiles' events in order (the lanes evaluate 32
 *                          clock measurements at a time) and appends its frames to a pool with the stream index and the
 *                          frame's rank in its stream, and the stream's frame count.  A stream pushed buffer by buffer
 *                          (nfcb200_iso7816_stream_push) resumes from the decoder state the previous buffer left.
 *   iso_gather_kernel      moves every pooled frame to its place in (stream, rank) order: the host's scan of the
 *                          streams' counts gives each stream's first place.
 */
#ifndef NFCB200_ISO_DECODE_CUH
#define NFCB200_ISO_DECODE_CUH

#include <stdint.h>

#include "../../include/nfcb200.h"
#include "iso_core.h"

namespace nfcb200 {

constexpr uint32_t ISO_TILE = 4096;             // samples per tile (12-bit offsets)
constexpr uint32_t ISO_THREADS = 256;
constexpr uint32_t ISO_PER_THREAD = ISO_TILE / ISO_THREADS;
constexpr uint32_t ISO_CLK_CAP = ISO_TILE / 2;  // CLK falling edges per tile on the first try (a two-level clock fits)
constexpr uint32_t ISO_LINE_CAP = 256;          // line events per tile on the first try

struct IsoEdgesArgs
{
   const void *samples;  // [n_streams][n_samples][4]
   uint64_t n_samples;
   uint32_t n_tiles;     // tiles per stream
   uint32_t line_cap, clk_cap;
   uint32_t *line;       // [stream][tile][line_cap]
   uint32_t *line_count; // [stream][tile]
   uint16_t *clk;        // [stream][tile][clk_cap]
   uint32_t *clk_count;  // [stream][tile]
   uint32_t *overflow;   // set when a tile has more line events than line_cap or more CLK falling edges than clk_cap
   float4 last;          // the sample before each stream's first: 0 in a batch (DESIGN.md section 13), the previous
                         // buffer's last sample in a pushed stream
};

template <bool S16>
__device__ __forceinline__ void iso_load(const void *base, uint64_t i, float d[4])
{
   if (S16)
   {
      const uint2 v = __ldg((const uint2 *) base + i);
      d[0] = (int16_t) (v.x & 0xFFFF) / 32768.f;
      d[1] = (int16_t) (v.x >> 16) / 32768.f;
      d[2] = (int16_t) (v.y & 0xFFFF) / 32768.f;
      d[3] = (int16_t) (v.y >> 16) / 32768.f;
   }
   else
   {
      const float4 v = __ldg((const float4 *) base + i);
      d[0] = v.x;
      d[1] = v.y;
      d[2] = v.z;
      d[3] = v.w;
   }
}

// A tile's flags as its threads hold them: fl[j * K + k] is sample j * ISO_THREADS * K + threadIdx.x * K + k of the tile, so
// the samples run in (j, warp, lane, k) order.  iso_tile_count() is called once per j as the flags come, iso_tile_scan()
// once, iso_tile_write() then puts every event in its slot in sample order.
template <uint32_t K>
struct IsoTileSlots
{
   static constexpr uint32_t J = ISO_PER_THREAD / K, W = ISO_THREADS / 32;
   uint32_t warpLine[J][W], warpClk[J][W]; // events of each (j, warp)
   uint32_t offLine[J][W], offClk[J][W];   // their first slot
   uint32_t total[2];
};

template <uint32_t K>
__device__ __forceinline__ void iso_tile_count(IsoTileSlots<K> &sh, const uint32_t *fl, uint32_t j)
{
   using namespace iso7816;
   const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
   uint32_t nl = 0, nc = 0;
#pragma unroll
   for (uint32_t k = 0; k < K; k++)
   {
      nl += __popc(__ballot_sync(~0u, (fl[j * K + k] & F_LINE) != 0));
      nc += __popc(__ballot_sync(~0u, (fl[j * K + k] & F_CLK_FALL) != 0));
   }
   if (lane == 0)
   {
      sh.warpLine[j][warp] = nl;
      sh.warpClk[j][warp] = nc;
   }
}

// exclusive scan of the per-(j, warp) counts in sample order, by warp 0 (between two barriers)
template <uint32_t K>
__device__ __forceinline__ void iso_tile_scan(IsoTileSlots<K> &sh)
{
   const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
   if (warp == 0)
   {
      constexpr uint32_t N = IsoTileSlots<K>::J * IsoTileSlots<K>::W, PER = N / 32;
      uint32_t *wl = &sh.warpLine[0][0], *wc = &sh.warpClk[0][0];
      uint32_t sl = 0, sc = 0;
      for (uint32_t k = 0; k < PER; k++)
      {
         sl += wl[lane * PER + k];
         sc += wc[lane * PER + k];
      }
      uint32_t il = sl, ic = sc;
      for (uint32_t o = 1; o < 32; o <<= 1)
      {
         const uint32_t vl = __shfl_up_sync(~0u, il, o), vc = __shfl_up_sync(~0u, ic, o);
         if (lane >= o)
         {
            il += vl;
            ic += vc;
         }
      }
      uint32_t el = il - sl, ec = ic - sc;
      for (uint32_t k = 0; k < PER; k++)
      {
         const uint32_t cl = wl[lane * PER + k], cc = wc[lane * PER + k];
         (&sh.offLine[0][0])[lane * PER + k] = el;
         (&sh.offClk[0][0])[lane * PER + k] = ec;
         el += cl;
         ec += cc;
      }
      if (lane == 31)
      {
         sh.total[0] = il;
         sh.total[1] = ic;
      }
   }
}

template <uint32_t K>
__device__ __forceinline__ void iso_tile_write(const IsoEdgesArgs &a, const IsoTileSlots<K> &sh, const uint32_t *fl)
{
   using namespace iso7816;
   const uint32_t tile = blockIdx.x, stream = blockIdx.y;
   const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
   const uint64_t slot = (uint64_t) stream * a.n_tiles + tile;
   uint32_t *line = a.line + slot * a.line_cap;
   uint16_t *clk = a.clk + slot * a.clk_cap;
   const uint32_t below = (1u << lane) - 1;
#pragma unroll
   for (uint32_t j = 0; j < IsoTileSlots<K>::J; j++)
   {
      uint32_t bl[K], bc[K], kl = sh.offLine[j][warp], kc = sh.offClk[j][warp];
#pragma unroll
      for (uint32_t k = 0; k < K; k++)
      {
         bl[k] = __ballot_sync(~0u, (fl[j * K + k] & F_LINE) != 0);
         bc[k] = __ballot_sync(~0u, (fl[j * K + k] & F_CLK_FALL) != 0);
      }
#pragma unroll
      for (uint32_t k = 0; k < K; k++) // the events of the lanes below, then this lane's own earlier samples
      {
         kl += __popc(bl[k] & below);
         kc += __popc(bc[k] & below);
      }
#pragma unroll
      for (uint32_t k = 0; k < K; k++)
      {
         const uint32_t f = fl[j * K + k], off = (j * ISO_THREADS + threadIdx.x) * K + k;
         if (f & F_LINE)
         {
            if (kl < a.line_cap)
               line[kl] = off | (f & ~F_CLK_FALL) << 12;
            kl++;
         }
         if (f & F_CLK_FALL)
         {
            if (kc < a.clk_cap)
               clk[kc] = (uint16_t) off;
            kc++;
         }
      }
   }
   if (threadIdx.x == 0)
   {
      a.line_count[slot] = sh.total[0];
      a.clk_count[slot] = sh.total[1];
      if (sh.total[0] > a.line_cap || sh.total[1] > a.clk_cap)
         atomicOr(a.overflow, 1u);
   }
}

// float32 / int16 at stride 4, the stream aligned to the sample (16 / 8 bytes): one vector load per sample.  It keeps its
// own copy of the tile's count, scan and write (those of IsoTileSlots with K = 1), so its code stays as it was measured.
template <bool S16>
__global__ void __launch_bounds__(ISO_THREADS) iso_edges_kernel(const IsoEdgesArgs a)
{
   using namespace iso7816;
   __shared__ uint32_t warpLine[ISO_PER_THREAD][ISO_THREADS / 32], warpClk[ISO_PER_THREAD][ISO_THREADS / 32];

   const uint32_t tile = blockIdx.x, stream = blockIdx.y;
   const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
   const uint64_t t0 = (uint64_t) tile * ISO_TILE;
   const void *base = S16 ? (const void *) ((const uint2 *) a.samples + (uint64_t) stream * a.n_samples)
                          : (const void *) ((const float4 *) a.samples + (uint64_t) stream * a.n_samples);

   uint32_t fl[ISO_PER_THREAD];
#pragma unroll
   for (uint32_t j = 0; j < ISO_PER_THREAD; j++)
   {
      const uint64_t i = t0 + j * ISO_THREADS + threadIdx.x;
      float d[4] = {0, 0, 0, 0}, l[4] = {a.last.x, a.last.y, a.last.z, a.last.w};
      if (i < a.n_samples)
      {
         iso_load<S16>(base, i, d);
         if (i > 0)
            iso_load<S16>(base, i - 1, l);
      }
      fl[j] = i < a.n_samples ? sample_flags(d, l) : 0u;
      const uint32_t bl = __ballot_sync(~0u, (fl[j] & F_LINE) != 0), bc = __ballot_sync(~0u, (fl[j] & F_CLK_FALL) != 0);
      if (lane == 0)
      {
         warpLine[j][warp] = __popc(bl);
         warpClk[j][warp] = __popc(bc);
      }
   }
   __syncthreads();
   // exclusive scan of the per-(j, warp) counts in sample order, by warp 0
   __shared__ uint32_t offLine[ISO_PER_THREAD][ISO_THREADS / 32], offClk[ISO_PER_THREAD][ISO_THREADS / 32], total[2];
   if (warp == 0)
   {
      constexpr uint32_t N = ISO_PER_THREAD * (ISO_THREADS / 32), PER = N / 32;
      uint32_t *wl = &warpLine[0][0], *wc = &warpClk[0][0];
      uint32_t sl = 0, sc = 0;
      for (uint32_t k = 0; k < PER; k++)
      {
         sl += wl[lane * PER + k];
         sc += wc[lane * PER + k];
      }
      uint32_t il = sl, ic = sc;
      for (uint32_t o = 1; o < 32; o <<= 1)
      {
         const uint32_t vl = __shfl_up_sync(~0u, il, o), vc = __shfl_up_sync(~0u, ic, o);
         if (lane >= o)
         {
            il += vl;
            ic += vc;
         }
      }
      uint32_t el = il - sl, ec = ic - sc;
      for (uint32_t k = 0; k < PER; k++)
      {
         const uint32_t cl = wl[lane * PER + k], cc = wc[lane * PER + k];
         (&offLine[0][0])[lane * PER + k] = el;
         (&offClk[0][0])[lane * PER + k] = ec;
         el += cl;
         ec += cc;
      }
      if (lane == 31)
      {
         total[0] = il;
         total[1] = ic;
      }
   }
   __syncthreads();

   const uint64_t slot = (uint64_t) stream * a.n_tiles + tile;
   uint32_t *line = a.line + slot * a.line_cap;
   uint16_t *clk = a.clk + slot * a.clk_cap;
   const uint32_t below = (1u << lane) - 1;
#pragma unroll
   for (uint32_t j = 0; j < ISO_PER_THREAD; j++)
   {
      const uint32_t off = j * ISO_THREADS + threadIdx.x;
      const bool isLine = (fl[j] & F_LINE) != 0, isClk = (fl[j] & F_CLK_FALL) != 0;
      const uint32_t bl = __ballot_sync(~0u, isLine), bc = __ballot_sync(~0u, isClk);
      if (isLine)
      {
         const uint32_t k = offLine[j][warp] + __popc(bl & below);
         if (k < a.line_cap)
            line[k] = off | (fl[j] & ~F_CLK_FALL) << 12;
      }
      if (isClk)
      {
         const uint32_t k = offClk[j][warp] + __popc(bc & below);
         if (k < a.clk_cap)
            clk[k] = (uint16_t) off;
      }
   }
   if (threadIdx.x == 0)
   {
      a.line_count[slot] = total[0];
      a.clk_count[slot] = total[1];
      if (total[0] > a.line_cap || total[1] > a.clk_cap)
         atomicOr(a.overflow, 1u);
   }
}

// flags of an 8-bit sample (4 channels in the low bytes of w) after the one in p, compared as integers (sample_flags)
__device__ __forceinline__ uint32_t iso_u8_flags(uint32_t w, uint32_t p)
{
   const int d[4] = {(int) (w & 0xFF), (int) (w >> 8 & 0xFF), (int) (w >> 16 & 0xFF), (int) (w >> 24)};
   const int l[4] = {(int) (p & 0xFF), (int) (p >> 8 & 0xFF), (int) (p >> 16 & 0xFF), (int) (p >> 24)};
   return iso7816::sample_flags(d, l);
}

// the first sample of a stream after a.last, in float as RecordDevice reads 8-bit samples (b / 255.f): a pushed stream's
// previous sample can come from a buffer of another format
__device__ __forceinline__ uint32_t iso_u8_first_flags(uint32_t w, const float4 &last)
{
   const float d[4] = {(w & 0xFF) / 255.f, (w >> 8 & 0xFF) / 255.f, (w >> 16 & 0xFF) / 255.f, (w >> 24) / 255.f};
   const float l[4] = {last.x, last.y, last.z, last.w};
   return iso7816::sample_flags(d, l);
}

// 8-bit samples at stride 4, the streams' base and pitch 16-byte aligned: a sample is one 32-bit word, a thread loads 4
// consecutive samples with one 16-byte load and takes the sample before them from the lane below (lane 0: one word load)
__global__ void __launch_bounds__(ISO_THREADS) iso_edges_u8x4_kernel(const IsoEdgesArgs a)
{
   constexpr uint32_t K = 4;
   __shared__ IsoTileSlots<K> sh;

   const uint32_t tile = blockIdx.x, stream = blockIdx.y, lane = threadIdx.x & 31;
   const uint64_t t0 = (uint64_t) tile * ISO_TILE, n = a.n_samples;
   const uint32_t *base = (const uint32_t *) a.samples + (uint64_t) stream * n;

   // every load first, so that a thread has all of them in flight at once
   constexpr uint32_t J = IsoTileSlots<K>::J;
   uint32_t w[ISO_PER_THREAD], p[J];
#pragma unroll
   for (uint32_t j = 0; j < J; j++)
   {
      const uint64_t i = t0 + (j * ISO_THREADS + threadIdx.x) * K;
      if (i + K <= n)
      {
         const uint4 v = __ldg((const uint4 *) (base + i));
         w[j * K] = v.x;
         w[j * K + 1] = v.y;
         w[j * K + 2] = v.z;
         w[j * K + 3] = v.w;
      }
      else
      {
#pragma unroll
         for (uint32_t k = 0; k < K; k++)
            w[j * K + k] = i + k < n ? __ldg(base + i + k) : 0u;
      }
      p[j] = lane == 0 && i > 0 && i < n ? __ldg(base + i - 1) : 0u;
   }

   uint32_t fl[ISO_PER_THREAD];
#pragma unroll
   for (uint32_t j = 0; j < J; j++)
   {
      const uint64_t i = t0 + (j * ISO_THREADS + threadIdx.x) * K;
      const uint32_t up = __shfl_up_sync(~0u, w[j * K + K - 1], 1);
      if (lane)
         p[j] = up;
#pragma unroll
      for (uint32_t k = 0; k < K; k++)
      {
         const uint64_t s = i + k;
         fl[j * K + k] = s >= n ? 0u : s == 0 ? iso_u8_first_flags(w[0], a.last) : iso_u8_flags(w[j * K + k], k ? w[j * K + k - 1] : p[j]);
      }
      iso_tile_count<K>(sh, fl, j);
   }
   __syncthreads();
   iso_tile_scan<K>(sh);
   __syncthreads();
   iso_tile_write<K>(a, sh, fl);
}

// channels 0-3 of sample `at` of a staged sub-tile, as the decoder reads them: float32 as is, int16 as s / 32768.f; 8-bit
// samples as their integer values (their flags are those of b / 255.f, sample_flags)
template <class T>
struct IsoStaged;

template <>
struct IsoStaged<float>
{
   using V = float;
   static __device__ __forceinline__ void load(const unsigned char *p, V d[4])
   {
      for (int c = 0; c < 4; c++)
         d[c] = ((const float *) p)[c];
   }
   static __device__ __forceinline__ void last(const float4 &l, V d[4])
   {
      d[0] = l.x, d[1] = l.y, d[2] = l.z, d[3] = l.w;
   }
};

template <>
struct IsoStaged<int16_t>
{
   using V = float;
   static __device__ __forceinline__ void load(const unsigned char *p, V d[4])
   {
      for (int c = 0; c < 4; c++)
         d[c] = ((const int16_t *) p)[c] / 32768.f;
   }
   static __device__ __forceinline__ void last(const float4 &l, V d[4])
   {
      IsoStaged<float>::last(l, d);
   }
};

template <>
struct IsoStaged<uint8_t>
{
   using V = int;
   static __device__ __forceinline__ void load(const unsigned char *p, V d[4])
   {
      for (int c = 0; c < 4; c++)
         d[c] = p[c];
   }
};

// samples a staged kernel reads into shared memory at a time: 32 KB at 8 channels (a whole tile of 8-bit samples, half a
// tile of int16, a quarter of float32), so that 4 CTAs of 256 threads fit an SM by shared memory as by registers
template <class T>
__host__ __device__ constexpr uint32_t iso_sub()
{
   return 32768 / (8 * sizeof(T));
}

// bytes of shared memory a staged kernel needs at `bps` bytes per sample: a sub-tile and the sample before it, from the
// 16-byte boundary below them to the one above
template <class T>
__host__ __device__ constexpr uint32_t iso_stage_bytes(uint32_t bps)
{
   return ((iso_sub<T>() + 1) * bps + 31) & ~15u;
}

// Any element type T at any stride 4-8, any alignment of the streams' base and pitch (T-aligned): the tile is read
// iso_sub<T>() samples at a time.  The threads copy the sub-tile's bytes, and the sample before it, into shared memory with
// coalesced 16-byte loads where the bytes are 16-byte aligned and byte loads for the up to 15 bytes at either end, then
// each thread picks channels 0-3 of its samples there.  Channels 4 and up are read past.
template <class T>
__global__ void __launch_bounds__(ISO_THREADS) iso_edges_staged_kernel(const IsoEdgesArgs a, uint32_t channels)
{
   using V = typename IsoStaged<T>::V;
   constexpr uint32_t SUB = iso_sub<T>();
   __shared__ IsoTileSlots<1> sh;
   extern __shared__ uint4 stage[];
   unsigned char *sb = (unsigned char *) stage;

   const uint32_t tile = blockIdx.x, stream = blockIdx.y;
   const uint64_t t0 = (uint64_t) tile * ISO_TILE, n = a.n_samples;
   const uint32_t bps = channels * (uint32_t) sizeof(T);
   const unsigned char *base = (const unsigned char *) a.samples + (uint64_t) stream * n * bps;

   uint32_t fl[ISO_PER_THREAD];
#pragma unroll
   for (uint32_t sub = 0; sub < ISO_TILE / SUB; sub++)
   {
      const uint64_t s0 = t0 + sub * SUB;
      const uint64_t first = s0 ? s0 - 1 : 0, end = s0 + SUB < n ? s0 + SUB : n;
      const uintptr_t lo = (uintptr_t) (base + first * bps), hi = (uintptr_t) (base + end * bps);
      const uintptr_t a0 = lo & ~(uintptr_t) 15, w0 = (lo + 15) & ~(uintptr_t) 15, w1 = hi & ~(uintptr_t) 15;
      __syncthreads(); // the previous sub-tile is read
      if (s0 < n)
      {
         if (w0 <= w1)
         {
            for (uintptr_t k = threadIdx.x; k < (w1 - w0) / 16; k += ISO_THREADS)
               stage[(w0 - a0) / 16 + k] = __ldg((const uint4 *) w0 + k);
            if (threadIdx.x < w0 - lo)
               sb[lo - a0 + threadIdx.x] = __ldg((const unsigned char *) lo + threadIdx.x);
            if (threadIdx.x < hi - w1)
               sb[w1 - a0 + threadIdx.x] = __ldg((const unsigned char *) w1 + threadIdx.x);
         }
         else if (threadIdx.x < hi - lo) // within one 16-byte word
            sb[lo - a0 + threadIdx.x] = __ldg((const unsigned char *) lo + threadIdx.x);
      }
      __syncthreads();
#pragma unroll
      for (uint32_t jj = 0; jj < SUB / ISO_THREADS; jj++)
      {
         const uint32_t j = sub * (SUB / ISO_THREADS) + jj;
         const uint64_t i = s0 + jj * ISO_THREADS + threadIdx.x;
         uint32_t f = 0;
         if (i < n)
         {
            const unsigned char *p = sb + (lo - a0) + (i - first) * bps;
            V d[4], l[4];
            IsoStaged<T>::load(p, d);
            if (i > 0)
            {
               IsoStaged<T>::load(p - bps, l);
               f = iso7816::sample_flags(d, l);
            }
            else if constexpr (sizeof(T) == 1)
               f = iso_u8_first_flags(p[0] | p[1] << 8 | p[2] << 16 | (uint32_t) p[3] << 24, a.last);
            else
            {
               IsoStaged<T>::last(a.last, l);
               f = iso7816::sample_flags(d, l);
            }
         }
         fl[j] = f;
         iso_tile_count<1>(sh, fl, j);
      }
   }
   __syncthreads();
   iso_tile_scan<1>(sh);
   __syncthreads();
   iso_tile_write<1>(a, sh, fl);
}

// the event source of iso_walk(): the per-tile slots of one stream, read in tile order, at absolute samples from `base`
struct IsoDevEvents
{
   const uint32_t *line, *lineCount;
   const uint16_t *clk;
   const uint32_t *clkCount;
   uint32_t nTiles, lineCap, clkCap, base;
   uint32_t lt = 0, li = 0, ct = 0, ci = 0;

   __device__ uint32_t line_peek()
   {
      while (lt < nTiles && li >= lineCount[lt])
      {
         lt++;
         li = 0;
      }
      return lt < nTiles ? base + lt * ISO_TILE + (line[(uint64_t) lt * lineCap + li] & (ISO_TILE - 1)) : iso7816::NONE;
   }

   __device__ uint32_t line_pop()
   {
      return line[(uint64_t) lt * lineCap + li++] >> 12;
   }

   __device__ uint32_t clk_nth(uint32_t k)
   {
      uint32_t t = ct, i = ci;
      while (t < nTiles)
      {
         const uint32_t n = clkCount[t];
         if (i < n)
         {
            if (k < n - i)
               return base + t * ISO_TILE + clk[(uint64_t) t * clkCap + i + k];
            k -= n - i;
         }
         t++;
         i = 0;
      }
      return iso7816::NONE;
   }

   __device__ void clk_pop()
   {
      clk_skip(1);
   }

   __device__ void clk_skip(uint32_t k)
   {
      while (ct < nTiles)
      {
         const uint32_t n = clkCount[ct];
         if (ci + k <= n)
         {
            ci += k;
            return;
         }
         k -= n > ci ? n - ci : 0;
         ct++;
         ci = 0;
      }
   }
};

struct IsoWalkArgs
{
   uint32_t n_streams, stream0, n_samples, n_tiles, line_cap, clk_cap, sample_rate, stream_time;
   const uint32_t *line, *line_count, *clk_count;
   const uint16_t *clk;
   nfcb200_frame *pool;
   uint32_t pool_cap;
   uint32_t *pool_count;
   uint32_t *stream_count; // [n_streams] frames of each stream
   // a pushed stream (one): the decoder left by the previous buffer, where this buffer's end state goes, the buffer's first
   // sample and whether its sample rate restarts the decoder.  Unused in a batch: every stream starts fresh at sample 0.
   const iso7816::IsoStreamState *resume;
   iso7816::IsoStreamState *state_out;
   uint32_t base, restart;
};

struct IsoDevSink
{
   const IsoWalkArgs *a;
   uint32_t stream, rank;

   // every lane of the warp calls this with the same frame; lane 0 writes it
   __device__ void frame(const iso7816::IsoFrameOut &f)
   {
      const uint32_t k = (threadIdx.x & 31) == 0 ? atomicAdd(a->pool_count, 1u) : ~0u;
      if (k < a->pool_cap)
      {
         nfcb200_frame &o = a->pool[k];
         o.stream = stream;
         o.tech_type = f.techType;
         o.frame_type = f.frameType;
         o.frame_flags = f.frameFlags;
         o.frame_phase = f.framePhase;
         o.frame_rate = f.frameRate;
         o.length = f.length;
         o.reserved = rank;
         o.sample_start = f.sampleStart;
         o.sample_end = f.sampleEnd;
         o.sample_rate = a->sample_rate;
         o.time_start = f.timeStart;
         o.time_end = f.timeEnd;
         o.date_time = f.dateTime;
         const uint32_t n = f.length < iso7816::FRAME_BYTES ? f.length : iso7816::FRAME_BYTES;
         for (uint32_t i = 0; i < ((n + 63) & ~63u); i++)
            o.data[i] = i < n ? f.data[i] : 0;
      }
      rank++;
   }
};

// one warp per stream: every lane keeps the same state (iso_walk evaluates clock measurements across the lanes).  RESUME:
// a pushed stream, which starts from a.resume and stores its end state (the batch's instance has no such code)
template <bool RESUME>
__global__ void __launch_bounds__(32) iso_walk_kernel(const IsoWalkArgs a)
{
   const uint32_t s = blockIdx.x;
   IsoDevEvents ev;
   ev.line = a.line + (uint64_t) s * a.n_tiles * a.line_cap;
   ev.lineCount = a.line_count + (uint64_t) s * a.n_tiles;
   ev.clk = a.clk + (uint64_t) s * a.n_tiles * a.clk_cap;
   ev.clkCount = a.clk_count + (uint64_t) s * a.n_tiles;
   ev.nTiles = a.n_tiles;
   ev.lineCap = a.line_cap;
   ev.clkCap = a.clk_cap;
   ev.base = a.base;
   IsoDevSink sink {&a, a.stream0 + s, 0};
   iso7816::IsoMachine m;
   iso7816::IsoCarry c;
   if (RESUME)
   {
      m = a.resume->m;
      c = a.resume->c;
      if (a.restart)
         iso7816::iso_restart(m, c, a.sample_rate, a.stream_time);
      else
         iso7816::iso_resume(m, c, a.base);
      m.streamTime = a.stream_time;
   }
   else
   {
      iso7816::iso_init(m, a.sample_rate, a.stream_time);
      c = iso7816::iso_carry_init();
   }
   iso7816::iso_walk(m, c, ev, a.base + a.n_samples, sink);
   if (threadIdx.x == 0)
   {
      a.stream_count[s] = sink.rank;
      if (RESUME)
      {
         a.state_out->m = m;
         a.state_out->c = c;
      }
   }
}

// pooled frame k -> out[first[stream - stream0] + rank], the rank field cleared; first[] counts from the chunk's first frame
__global__ void iso_gather_kernel(const nfcb200_frame *pool, uint32_t count, const uint64_t *first, uint32_t stream0, nfcb200_frame *out)
{
   constexpr uint32_t WORDS = sizeof(nfcb200_frame) / 16;
   static_assert(sizeof(nfcb200_frame) % 16 == 0, "frames move as 16-byte words");
   const uint32_t lane = threadIdx.x & 31;
   for (uint64_t k = (blockIdx.x * (uint64_t) blockDim.x + threadIdx.x) / 32; k < count; k += (uint64_t) gridDim.x * blockDim.x / 32)
   {
      const nfcb200_frame &f = pool[k];
      nfcb200_frame *o = out + first[f.stream - stream0] + f.reserved;
      for (uint32_t w = lane; w < WORDS; w += 32)
         ((uint4 *) o)[w] = ((const uint4 *) &f)[w];
      __syncwarp();
      if (lane == 0)
         o->reserved = 0;
   }
}

} // namespace nfcb200

#endif
