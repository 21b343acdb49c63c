/*
 * adaptive.cuh -- the reference's "adaptive" signal (lab::SignalResamplingTask, lab-tasks SignalResamplingTask.cpp:138-274):
 * the reduced waveform its GUI draws in the signal view and TraceStorageTask stores in a .trz.  Every buffer is resampled
 * on its own; only its offset carries over.
 *
 *   radio  (processRadioSignal :168-229) a float running sum over a 51-sample window, updated in sample order; a sample is
 *          kept where it deviates from the window mean by more than 0.005 or 255 samples after the last kept one, a
 *          control point before a deviating sample that follows a gap, and the buffer's last sample
 *   logic  (processLogicSignal :231-274) per channel but CLK (channel 1): the first sample, every change against the
 *          previous sample, and one sample every 255 after the last kept one
 *
 * The per-sample steps are __host__ __device__ (radio_step, logic_step) so that tests/native/adaptive_host.cpp runs the
 * same arithmetic on the CPU.  The running sum is a non-associative float recurrence, so one thread owns one (stream,
 * buffer) and steps it in order; a batch has tens of thousands of buffers.  Each warp stages its 32 buffers through shared
 * memory 32 samples at a time with coalesced loads, every thread reading its own buffer's taps there.  Both kernels run
 * twice: COUNT writes the points of every (stream, list, buffer), the host scans them, EMIT writes the points in place.
 *
 * Deviations, where the reference is undefined:
 *   - a radio buffer shorter than 25 samples: the reference's initial sum reads past the buffer into recycled pool memory;
 *     here those samples are 0;
 *   - the reference's output buffer holds elements + elements / 255 points (:170).  A buffer yields at most elements + 1
 *     (every sample once, the first one twice when it already deviates), so a buffer shorter than 255 samples whose
 *     samples all deviate makes the reference write past its allocation.  Here every point the algorithm produces is
 *     returned.
 */
#ifndef NFCB200_ADAPTIVE_CUH
#define NFCB200_ADAPTIVE_CUH

#include <math.h>
#include <stdint.h>

#include "../../include/nfcb200.h"

#if defined(__CUDACC__)
#include "nfc_screen.cuh"
#define AD_HD __host__ __device__ __forceinline__
#else
#define AD_HD inline
#endif

namespace nfcb200 {

constexpr int AD_HALF = 25;               // WINDOW / 2 (:34, :177)
constexpr uint32_t AD_INTERVAL = 255;     // RADIO_INTERVAL, LOGIC_INTERVAL (:36-37)
constexpr uint64_t AD_MAX_BUFFER = 1ull << 24; // indices are stored as float(i): exact up to 2^24

// processRadioSignal's loop state: the running sum, the previous sample and the index of the last stored point
struct RadioState
{
   float avrg;
   float last;
   int c;
};

// the initial sum (:177-178) of x(0 .. 24) in order, samples at or past `limit` taken as 0
template <class X>
AD_HD RadioState radio_start(const X &x, int limit)
{
   RadioState s = {0.f, 0.f, 0};
   for (int i = 0; i < AD_HALF; i++)
      if (i < limit)
         s.avrg += x(i);
   return s;
}

// step i (:187-218): v = x[i], add = x[i + 25], sub = x[i - 26] (each read only where the reference reads it).  emit(value,
// index) for each point stored.  One IEEE operation at a time: the library has -fmad=false, the host build -ffp-contract=off.
template <class E>
AD_HD void radio_step(RadioState &s, int i, int limit, float v, float add, float sub, E &emit)
{
   if (i + AD_HALF < limit)
      s.avrg += add;
   if (i - AD_HALF - 1 >= 0)
      s.avrg -= sub;
   const float stdev = fabsf(v - s.avrg / 51.f);
   const bool dev = stdev > 0.005f; // float filter = THRESHOLD (a double converted to float)
   if (dev || i - s.c >= (int) AD_INTERVAL)
   {
      if (dev && s.c < i - 1)
         emit(s.last, i - 1);
      emit(v, i);
      s.c = i;
   }
   s.last = v;
}

// after the loop (:221-222)
template <class E>
AD_HD void radio_end(const RadioState &s, int limit, E &emit)
{
   if (s.c < limit - 1)
      emit(s.last, limit - 1);
}

// one logic channel's step at sample s >= 1 (:251-265); last / c start as x[0] / 0 after the first point (x[0], 0)
template <class E>
AD_HD void logic_step(float &last, uint32_t &c, uint32_t s, float v, E &emit)
{
   if (v != last || s - c >= AD_INTERVAL)
   {
      emit(v, s);
      last = v;
      c = s;
   }
}

// output list of logic channel n: channel 1 (CLK) has none, the others keep their order
AD_HD constexpr uint32_t logic_list(uint32_t n)
{
   return n == 0 ? 0 : n - 1;
}

#if defined(__CUDACC__)
struct AdaptiveArgs
{
   const void *samples;     // streams [n_streams][n_samples] of `channels` elements per sample (radio: 1 sample)
   uint64_t n_samples;
   uint64_t buffer_len;
   uint64_t offset;         // the stream position of each stream's first sample
   uint32_t n_buf;          // buffers per stream
   uint32_t n_streams;      // streams in this launch
   uint32_t stream0;        // batch index of the launch's first stream
   uint32_t channels;       // logic: channels per sample
   uint32_t lists;          // output lists per buffer: radio 1, logic channels - 1
   uint32_t *count;         // COUNT: points of list l of buffer b of stream s at [(s * lists + l) * n_buf + b]
   const uint64_t *first;   // EMIT: place in `out` of the first point of the same slot
   nfcb200_signal_point *out;
   uint64_t out_n;          // EMIT: places >= out_n are not written (the caller's capacity)
};

// where a point goes: counted, or written at its place
template <bool EMIT>
struct AdSink
{
   nfcb200_signal_point *out;
   uint64_t out_n;
   uint32_t stream, channel;
   uint64_t base;  // stream position of the buffer's first sample
   uint64_t place; // EMIT: next place; COUNT: points so far
   __device__ __forceinline__ void operator()(float value, int i)
   {
      if (EMIT && place < out_n)
      {
         nfcb200_signal_point p;
         p.stream = stream;
         p.channel = channel;
         p.sample = base + (uint32_t) (float) i; // stored as float(i), read back as (unsigned) float(i) (TraceStorageTask.cpp:680)
         p.value = value;
         p.reserved = 0;
         out[place] = p;
      }
      place++;
   }
};

// the buffer a thread owns and the warp's longest buffer
struct AdBuffer
{
   bool active;
   uint32_t stream, buf;
   uint64_t start; // sample index of the buffer's first sample within its stream
   int limit;
   int warpMax;
};

__device__ __forceinline__ AdBuffer ad_buffer(const AdaptiveArgs &a)
{
   AdBuffer b;
   const uint64_t g = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
   b.active = g < (uint64_t) a.n_streams * a.n_buf;
   b.stream = b.active ? (uint32_t) (g / a.n_buf) : 0;
   b.buf = b.active ? (uint32_t) (g % a.n_buf) : 0;
   b.start = (uint64_t) b.buf * a.buffer_len;
   b.limit = b.active ? (int) min(a.buffer_len, a.n_samples - b.start) : 0;
   int m = b.limit;
   for (int d = 16; d; d >>= 1)
      m = max(m, __shfl_xor_sync(~0u, m, d));
   b.warpMax = m;
   return b;
}

constexpr uint32_t AD_RADIO_THREADS = 64;
constexpr uint32_t AD_CHUNK = 32;                 // samples of each buffer staged at a time: one per lane
constexpr uint32_t AD_RING = 3 * AD_CHUNK;        // chunks k - 1, k, k + 1: the taps i - 26 .. i + 25 of chunk k
constexpr uint32_t AD_PITCH = 33;                 // [sample slot][buffer], padded: conflict-free both ways

// Radio: thread = (stream, buffer).  The warp stages chunk k + 1 of its 32 buffers (row b: lane l loads sample 32 (k + 1) + l
// of lane b's buffer), then every lane steps its own buffer through chunk k with the taps in the ring.
template <int SIG, bool EMIT>
__global__ void __launch_bounds__(AD_RADIO_THREADS) adaptive_radio_kernel(const AdaptiveArgs a)
{
   __shared__ float ring[AD_RADIO_THREADS / 32][AD_RING * AD_PITCH];
   float *r = ring[threadIdx.x / 32];
   const uint32_t lane = threadIdx.x % 32;
   const AdBuffer b = ad_buffer(a);
   const uint64_t sbase = (uint64_t) b.stream * a.n_samples + b.start; // this lane's first sample in the launch's streams

   auto stage = [&](int chunk) {
      const int i = chunk * (int) AD_CHUNK + (int) lane;
      float *slot = r + (i % AD_RING) * AD_PITCH;
#pragma unroll 8
      for (int row = 0; row < 32; row++)
      {
         const uint64_t rb = __shfl_sync(~0u, sbase, row);
         const int rl = __shfl_sync(~0u, b.limit, row);
         // K1's per-format magnitude (nfc_screen.cuh), at the sample's own address: indices pass 2^32 in a batch
         slot[row] = i < rl ? sample_from_raw((const unsigned char *) a.samples + (rb + i) * sig_bytes(SIG), SIG, 0) : 0.f;
      }
   };

   AdSink<EMIT> emit{a.out, a.out_n, a.stream0 + b.stream, 0, a.offset + b.start, 0};
   if (EMIT && b.active)
      emit.place = a.first[(uint64_t) b.stream * a.n_buf + b.buf];

   stage(0);
   stage(1);
   __syncwarp();
   RadioState s = radio_start([&](int i) { return r[i * AD_PITCH + lane]; }, b.limit);
   if (b.active)
      emit(r[lane], 0); // the first sample, always (:181)
   for (int k = 0; k * (int) AD_CHUNK < b.warpMax; k++)
   {
      for (int j = 0; j < (int) AD_CHUNK; j++)
      {
         const int i = k * (int) AD_CHUNK + j;
         if (i < b.limit)
         {
            const float v = r[(i % AD_RING) * AD_PITCH + lane];
            const float add = r[((i + AD_HALF) % AD_RING) * AD_PITCH + lane];
            const float sub = r[((i + AD_RING - AD_HALF - 1) % AD_RING) * AD_PITCH + lane];
            radio_step(s, i, b.limit, v, add, sub, emit);
         }
      }
      __syncwarp();
      stage(k + 2);
      __syncwarp();
   }
   if (b.active)
   {
      radio_end(s, b.limit, emit);
      if (!EMIT)
         a.count[(uint64_t) b.stream * a.n_buf + b.buf] = (uint32_t) emit.place;
   }
}

// Logic: thread = (stream, buffer), every channel but CLK.  The warp stages 32 samples of its 32 buffers, all channels
// (row b: the 32 * channels elements of lane b's buffer, converted to float as the reference reads them), then every lane
// steps its buffer through them.  Rows are padded by one float: conflict-free both ways.
template <class T>
__device__ __forceinline__ float ad_logic_value(T v);
template <>
__device__ __forceinline__ float ad_logic_value<float>(float v)
{
   return v;
}
template <>
__device__ __forceinline__ float ad_logic_value<int16_t>(int16_t v)
{
   return v / 32768.f;
}
template <>
__device__ __forceinline__ float ad_logic_value<uint8_t>(uint8_t v)
{
   return v / 255.f; // RecordDevice.cpp:244-245
}

constexpr uint32_t AD_LOGIC_MAX_CH = 8;

__host__ __device__ constexpr uint32_t ad_logic_pitch(uint32_t channels)
{
   return AD_CHUNK * channels + 1;
}

template <class T, bool EMIT>
__global__ void __launch_bounds__(32) adaptive_logic_kernel(const AdaptiveArgs a)
{
   extern __shared__ float stage[]; // [32 rows][ad_logic_pitch(channels)]
   const uint32_t lane = threadIdx.x;
   const uint32_t ch = a.channels, pitch = ad_logic_pitch(ch), rowElems = AD_CHUNK * ch;
   const AdBuffer b = ad_buffer(a);
   const T *base = (const T *) a.samples;
   const uint64_t ebase = ((uint64_t) b.stream * a.n_samples + b.start) * ch; // this lane's first element

   float last[AD_LOGIC_MAX_CH];
   uint32_t c[AD_LOGIC_MAX_CH];
   uint64_t place[AD_LOGIC_MAX_CH];
#pragma unroll
   for (uint32_t n = 0; n < AD_LOGIC_MAX_CH; n++)
   {
      last[n] = 0.f;
      c[n] = 0;
      place[n] = 0;
      if (EMIT && b.active && n < ch && n != 1)
         place[n] = a.first[((uint64_t) b.stream * a.lists + logic_list(n)) * a.n_buf + b.buf];
   }
   AdSink<EMIT> emit{a.out, a.out_n, a.stream0 + b.stream, 0, a.offset + b.start, 0};
   const float *mine = stage + lane * pitch;

   for (int k = 0; k * (int) AD_CHUNK < b.warpMax; k++)
   {
      __syncwarp();
      for (int row = 0; row < 32; row++)
      {
         const uint64_t rb = __shfl_sync(~0u, ebase, row);
         const int rl = __shfl_sync(~0u, b.limit, row);
         const uint32_t avail = (uint32_t) max(0, min((int) AD_CHUNK, rl - k * (int) AD_CHUNK)) * ch;
         for (uint32_t e = lane; e < rowElems; e += 32)
            stage[row * pitch + e] = e < avail ? ad_logic_value<T>(base[rb + (uint64_t) k * rowElems + e]) : 0.f;
      }
      __syncwarp();
      for (int j = 0; j < (int) AD_CHUNK; j++)
      {
         const int s = k * (int) AD_CHUNK + j;
         if (s >= b.limit)
            break;
#pragma unroll
         for (uint32_t n = 0; n < AD_LOGIC_MAX_CH; n++)
         {
            if (n >= ch || n == 1)
               continue;
            const float v = mine[j * ch + n];
            emit.channel = n;
            emit.place = place[n];
            if (s == 0)
            {
               emit(v, 0); // the first point (:245-248)
               last[n] = v;
            }
            else
               logic_step(last[n], c[n], (uint32_t) s, v, emit);
            place[n] = emit.place;
         }
      }
   }
   if (!EMIT && b.active)
   {
#pragma unroll
      for (uint32_t n = 0; n < AD_LOGIC_MAX_CH; n++)
         if (n < ch && n != 1)
            a.count[((uint64_t) b.stream * a.lists + logic_list(n)) * a.n_buf + b.buf] = (uint32_t) place[n];
   }
}

#endif // __CUDACC__

} // namespace nfcb200

#endif
