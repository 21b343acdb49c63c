/*
 * spectrum.cu -- nfcb200_spectrum / nfcb200_spectrum_shape: the FFT spectrum of IQ (FourierProcessTask::process at every
 * hop, nfc_spectrum.cuh).
 */
#include "host.h"
#include "nfc_spectrum.cuh"

using namespace nfcb200;

static void launch_spectrum(const nfcb200_handle *h, bool s16, const SpecLaunch &L, cudaStream_t st)
{
   const uint64_t grid = std::min<uint64_t>(L.count, (uint64_t) h->smCount * SPEC_BLOCKS_PER_SM);
   if (s16)
      spectrum_kernel<true><<<(unsigned) grid, SPEC_THREADS, 0, st>>>(L);
   else
      spectrum_kernel<false><<<(unsigned) grid, SPEC_THREADS, 0, st>>>(L);
}

extern "C" {

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

int nfcb200_spectrum(nfcb200_handle *h, const void *samples, int samples_on_device, int sigtype, uint32_t n_streams, uint64_t n_samples,
                     uint32_t sample_rate, uint64_t hop, float *out, int out_on_device, uint64_t cap, uint64_t *n_frames)
{
   if (!h)
      return fail(NFCB200_ERR_INVALID, "null handle");
   if (n_frames)
      *n_frames = 0;
   if (sigtype < NFCB200_SIG_IQ_F32 || sigtype > NFCB200_SIG_IQ_S16)
      return fail(NFCB200_ERR_INVALID, "unknown signal type %d", sigtype);
   if (!samples || n_streams == 0 || n_samples == 0)
      return fail(NFCB200_ERR_INVALID, "empty batch");
   if (cap && !out)
      return fail(NFCB200_ERR_INVALID, "null spectrum buffer");
   if (sigtype != NFCB200_SIG_IQ_F32 && sigtype != NFCB200_SIG_IQ_S16)
      return fail(NFCB200_ERR_UNSUPPORTED, "the spectrum needs IQ samples (FourierProcessTask.cpp:234 skips other buffers)");
   uint64_t nf = 0;
   uint32_t dec = 0;
   int rc = nfcb200_spectrum_shape(n_samples, sample_rate, hop, &nf, &dec);
   if (rc)
      return rc;
   const bool s16 = sigtype == NFCB200_SIG_IQ_S16;
   const uint32_t bs = s16 ? 4 : 8;
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
   auto &S = h->spec;

   if (!S.tablesReady)
   {
      SpecCx tw[SPEC_LEN];
      float win[SPEC_LEN];
      spectrum_tables(tw, win);
      rc = S.tables.reserve(sizeof(tw) + sizeof(win));
      if (rc)
         return rc;
      CUDA_TRY(cudaMemcpy(S.tables.ptr, tw, sizeof(tw), cudaMemcpyHostToDevice));
      CUDA_TRY(cudaMemcpy(S.tables.as<unsigned char>() + sizeof(tw), win, sizeof(win), cudaMemcpyHostToDevice));
      S.tablesReady = true;
   }

   SpecLaunch L = {};
   L.n_samples = n_samples;
   L.hop = hop;
   L.n_frames = nf;
   L.decimation = dec;
   L.tw = S.tables.as<SpecCx>();
   L.win = (const float *) (S.tables.as<SpecCx>() + SPEC_LEN);

   // host output is staged a group of frames at a time (256 MB)
   const uint64_t chunkFrames = 1ull << 16;
   if (!out_on_device && (rc = S.out.reserve(std::min(total, chunkFrames) * SPEC_LEN * sizeof(float))))
      return rc;

   // one group of streams: the spectrum of its frames, written to `out` directly or through the staging buffer
   auto group = [&](uint32_t s0, uint32_t sc, const void *dSamples) -> int {
      L.samples = dSamples;
      L.s0 = s0;
      const uint64_t g1 = (uint64_t) (s0 + sc) * nf;
      for (uint64_t g0 = (uint64_t) s0 * nf; g0 < g1;)
      {
         L.g0 = g0;
         L.count = out_on_device ? g1 - g0 : std::min(chunkFrames, g1 - g0);
         L.out = out_on_device ? out + g0 * SPEC_LEN : S.out.as<float>();
         launch_spectrum(h, s16, L, st);
         CUDA_TRY(cudaGetLastError());
         if (!out_on_device)
            CUDA_TRY(cudaMemcpyAsync(out + g0 * SPEC_LEN, S.out.ptr, L.count * SPEC_LEN * sizeof(float), cudaMemcpyDeviceToHost, st));
         g0 += L.count;
      }
      return 0;
   };
   if ((rc = for_each_stream_group(samples, samples_on_device, n_streams, n_samples * bs, ~0u, S.in, st, group)))
      return rc;
   CUDA_TRY(cudaStreamSynchronize(st));
   return 0;
}

}
