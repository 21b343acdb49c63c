/*
 * adaptive.cu -- nfcb200_adaptive_radio / nfcb200_adaptive_logic: the reference's adaptive signal (adaptive.cuh) of a
 * batch.  Per group of streams: the COUNT kernel, the points per (stream, list, buffer) to the host, a scan there, then the
 * EMIT kernel a window of whole streams at a time into a device buffer that is copied to the caller's.
 */
#include <vector>

#include "host.h"
#include "adaptive.cuh"

using namespace nfcb200;

namespace {

constexpr uint64_t AD_WINDOW_POINTS = 1ull << 22; // least points per emit window (96 MB), or one stream's when it has more

template <bool EMIT>
void launch(int sigtype, const AdaptiveArgs &a, cudaStream_t st)
{
   const uint64_t threads = (uint64_t) a.n_streams * a.n_buf;
   if (sigtype >= NFCB200_SIG_LOGIC_F32)
   {
      const unsigned grid = (unsigned) ((threads + 31) / 32);
      const size_t smem = 32 * ad_logic_pitch(a.channels) * sizeof(float);
      if (sigtype == NFCB200_SIG_LOGIC_F32)
         adaptive_logic_kernel<float, EMIT><<<grid, 32, smem, st>>>(a);
      else if (sigtype == NFCB200_SIG_LOGIC_S16)
         adaptive_logic_kernel<int16_t, EMIT><<<grid, 32, smem, st>>>(a);
      else
         adaptive_logic_kernel<uint8_t, EMIT><<<grid, 32, smem, st>>>(a);
      return;
   }
   const unsigned grid = (unsigned) ((threads + AD_RADIO_THREADS - 1) / AD_RADIO_THREADS);
   switch (sigtype)
   {
      case NFCB200_SIG_IQ_F32:
         adaptive_radio_kernel<SIG_IQ_F32, EMIT><<<grid, AD_RADIO_THREADS, 0, st>>>(a);
         break;
      case NFCB200_SIG_MAG_F32:
         adaptive_radio_kernel<SIG_MAG_F32, EMIT><<<grid, AD_RADIO_THREADS, 0, st>>>(a);
         break;
      case NFCB200_SIG_MAG_S16:
         adaptive_radio_kernel<SIG_MAG_S16, EMIT><<<grid, AD_RADIO_THREADS, 0, st>>>(a);
         break;
      default:
         adaptive_radio_kernel<SIG_IQ_S16, EMIT><<<grid, AD_RADIO_THREADS, 0, st>>>(a);
         break;
   }
}

// bytes of one sample (all channels) and the alignment device input needs
uint32_t sample_bytes(int sigtype, uint32_t channels)
{
   switch (sigtype)
   {
      case NFCB200_SIG_LOGIC_F32:
         return 4 * channels;
      case NFCB200_SIG_LOGIC_S16:
         return 2 * channels;
      case NFCB200_SIG_LOGIC_U8:
         return channels;
      default:
         return sig_bytes(sigtype);
   }
}

uint32_t sample_align(int sigtype)
{
   switch (sigtype)
   {
      case NFCB200_SIG_IQ_F32:
         return 8;
      case NFCB200_SIG_IQ_S16:
      case NFCB200_SIG_MAG_F32:
      case NFCB200_SIG_LOGIC_F32:
         return 4;
      case NFCB200_SIG_LOGIC_U8:
         return 1;
      default:
         return 2;
   }
}

// channels == 0: radio
int adaptive(nfcb200_handle *h, const void *samples, int samples_on_device, int sigtype, uint32_t channels, uint32_t n_streams, uint64_t n_samples,
             uint32_t sample_rate, uint64_t buffer_len, uint64_t offset, nfcb200_signal_point *out, uint64_t cap, uint64_t *n_out)
{
   if (n_out)
      *n_out = 0;
   if (!h)
      return fail(NFCB200_ERR_INVALID, "null handle");
   const bool logic = channels != 0;
   if (!logic && (sigtype < NFCB200_SIG_IQ_F32 || sigtype > NFCB200_SIG_IQ_S16))
      return fail(NFCB200_ERR_INVALID, "signal type %d is not a radio format", sigtype);
   if (logic && (sigtype < NFCB200_SIG_LOGIC_F32 || sigtype > NFCB200_SIG_LOGIC_U8))
      return fail(NFCB200_ERR_INVALID, "signal type %d is not a logic format", sigtype);
   if (logic && (channels < 4 || channels > AD_LOGIC_MAX_CH))
      return fail(NFCB200_ERR_INVALID, "%u channels: logic captures have 4 to 8", channels);
   if (!samples || n_streams == 0 || n_samples == 0)
      return fail(NFCB200_ERR_INVALID, "empty batch");
   if (cap && !out)
      return fail(NFCB200_ERR_INVALID, "null point buffer");
   if (sample_rate == 0)
      return fail(NFCB200_ERR_INVALID, "sample rate of 0");
   if (buffer_len == 0)
      return fail(NFCB200_ERR_INVALID, "buffer of 0 samples");
   if (buffer_len > AD_MAX_BUFFER)
      return fail(NFCB200_ERR_UNSUPPORTED, "buffers of %llu samples: indices are stored as float, exact up to 2^24",
                  (unsigned long long) buffer_len);
   if (offset > (1ull << 32) || n_samples > (1ull << 32) - offset)
      return fail(NFCB200_ERR_UNSUPPORTED, "streams reaching position 2^32 exceed the 32-bit sample offsets of the .trz format "
                                           "(TraceStorageTask.cpp:680)");
   const uint32_t bps = sample_bytes(sigtype, logic ? channels : 1);
   if (samples_on_device && ((uintptr_t) samples % sample_align(sigtype)))
      return fail(NFCB200_ERR_INVALID, "device samples not aligned to %u bytes", sample_align(sigtype));

   CUDA_TRY(cudaSetDevice(h->device));
   cudaStream_t st = h->stream;
   auto &A = h->adapt;
   const uint64_t n_buf = (n_samples + buffer_len - 1) / buffer_len;
   const uint32_t lists = logic ? channels - 1 : 1;
   const uint64_t slotsPerStream = lists * n_buf;
   uint64_t total = 0; // points of the streams before the current group: the place of its first point
   // An emit launch steps every buffer of its window from the first sample to the last, one thread each, so its time is
   // that of one buffer however few threads it has: windows as large as half the free device memory, few launches.
   size_t freeBytes = 0, totalBytes = 0;
   CUDA_TRY(cudaMemGetInfo(&freeBytes, &totalBytes));
   const uint64_t windowPoints = std::max<uint64_t>(AD_WINDOW_POINTS, freeBytes / 2 / sizeof(nfcb200_signal_point));
   std::vector<uint64_t> first;

   AdaptiveArgs a = {};
   a.n_samples = n_samples;
   a.buffer_len = buffer_len;
   a.offset = offset;
   a.n_buf = (uint32_t) n_buf;
   a.channels = logic ? channels : 1;
   a.lists = lists;

   auto group = [&](uint32_t s0, uint32_t sc, const void *dSamples) -> int {
      const uint64_t slots = sc * slotsPerStream;
      int rc;
      if ((rc = A.count.reserve(slots * sizeof(uint32_t))) || (rc = A.hCount.reserve(slots * sizeof(uint32_t))))
         return rc;
      a.samples = dSamples;
      a.n_streams = sc;
      a.stream0 = s0;
      a.count = A.count.as<uint32_t>();
      launch<false>(sigtype, a, st);
      CUDA_TRY(cudaGetLastError());
      CUDA_TRY(cudaMemcpyAsync(A.hCount.ptr, A.count.ptr, slots * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
      CUDA_TRY(cudaStreamSynchronize(st));

      // places, then the emit windows: whole streams, up to windowPoints points each, those below cap only
      const uint32_t *cnt = A.hCount.as<uint32_t>();
      first.resize(slots);
      std::vector<uint64_t> streamFirst(sc + 1);
      uint64_t place = total;
      for (uint64_t k = 0; k < slots; k++)
      {
         if (k % slotsPerStream == 0)
            streamFirst[k / slotsPerStream] = place;
         first[k] = place;
         place += cnt[k];
      }
      streamFirst[sc] = place;
      total = place;

      for (uint32_t w0 = 0; w0 < sc && streamFirst[w0] < cap;)
      {
         uint32_t w1 = w0 + 1;
         while (w1 < sc && streamFirst[w1 + 1] - streamFirst[w0] <= windowPoints && streamFirst[w1] < cap)
            w1++;
         const uint64_t lo = streamFirst[w0], n = std::min(streamFirst[w1], cap) - lo;
         if (n)
         {
            std::vector<uint64_t> rel(first.begin() + w0 * slotsPerStream, first.begin() + w1 * slotsPerStream);
            for (auto &p: rel)
               p -= lo;
            if ((rc = A.first.reserve(rel.size() * sizeof(uint64_t))) || (rc = A.out.reserve(n * sizeof(nfcb200_signal_point))))
               return rc;
            CUDA_TRY(cudaMemcpyAsync(A.first.ptr, rel.data(), rel.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
            AdaptiveArgs e = a;
            e.samples = (const unsigned char *) dSamples + (uint64_t) w0 * n_samples * bps;
            e.n_streams = w1 - w0;
            e.stream0 = s0 + w0;
            e.first = A.first.as<uint64_t>();
            e.out = A.out.as<nfcb200_signal_point>();
            e.out_n = n;
            launch<true>(sigtype, e, st);
            CUDA_TRY(cudaGetLastError());
            CUDA_TRY(cudaMemcpyAsync(out + lo, A.out.ptr, n * sizeof(nfcb200_signal_point), cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaStreamSynchronize(st)); // `rel` and the window buffer are reused by the next window
         }
         w0 = w1;
      }
      return 0;
   };
   // a group's buffer indices are 32-bit, and so is the grid of its launches
   const uint32_t limit = (uint32_t) std::max<uint64_t>(1, std::min<uint64_t>(~0u, (1ull << 31) / n_buf));
   int rc = for_each_stream_group(samples, samples_on_device, n_streams, n_samples * bps, limit, A.in, st, group);
   if (rc)
      return rc;
   CUDA_TRY(cudaStreamSynchronize(st));
   if (n_out)
      *n_out = total;
   if (total > cap)
      return fail(NFCB200_ERR_CAPACITY, "%llu points but room for %llu only", (unsigned long long) total, (unsigned long long) cap);
   return 0;
}

} // namespace

extern "C" {

int nfcb200_adaptive_radio(nfcb200_handle *h, const void *samples, int samples_on_device, int sigtype, uint32_t n_streams, uint64_t n_samples,
                           uint32_t sample_rate, uint64_t buffer_len, uint64_t offset, nfcb200_signal_point *out, uint64_t cap, uint64_t *n_out)
{
   return adaptive(h, samples, samples_on_device, sigtype, 0, n_streams, n_samples, sample_rate, buffer_len, offset, out, cap, n_out);
}

int nfcb200_adaptive_logic(nfcb200_handle *h, const void *samples, int samples_on_device, int sigtype, uint32_t channels, uint32_t n_streams,
                           uint64_t n_samples, uint32_t sample_rate, uint64_t buffer_len, uint64_t offset, nfcb200_signal_point *out, uint64_t cap,
                           uint64_t *n_out)
{
   if (channels == 0)
      return fail(NFCB200_ERR_INVALID, "0 channels: logic captures have 4 to 8");
   return adaptive(h, samples, samples_on_device, sigtype, channels, n_streams, n_samples, sample_rate, buffer_len, offset, out, cap, n_out);
}

}
