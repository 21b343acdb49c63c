/*
 * oracle/ref_fft.cpp -- TEST INFRASTRUCTURE ONLY: the reference's FFT spectrum frame (lab::FourierProcessTask::process,
 * src/nfc-lib/lib-lab/lab-tasks/src/main/cpp/tasks/FourierProcessTask.cpp:223-352) over float32 IQ, for the spectrum tests.
 *
 * The transform is the reference's own mufft (lib-ext/mufft, compiled unmodified by oracle/fft.mk).  The task object
 * around it is not driven: it runs on a worker thread that wakes every 10 ms and transforms whichever buffer was published
 * last (:172-179, :105-108), so which buffer a given spectrum belongs to is a matter of timing.  The steps around the
 * transform are restated here, each with the lines it restates.  Compiled with the reference's release flags, no FMA.
 */
#include <cmath>
#include <cstdint>
#include <cstring>

extern "C" {
#include <fft.h>
}

static const int LENGTH = 1024;      // construct() -> Impl(int length = 1024, int window = Hamming), :87, :371-374
static const int BANDWIDTH = 10E6 / 16; // :49

extern "C" {

// frames [n_frames][1024] of buffers that begin at samples 0, hop, 2 hop, ... of `iq` ([n_samples][2] float32); returns
// the frame count, or -1 where the reference's decimation is 0 (sample rate below 625 kHz)
long nfcref_fft(const float *iq, uint64_t n_samples, uint32_t sample_rate, uint64_t hop, float *out, long cap_frames)
{
   // :239 decimation = static_cast<int>(localBuffer.sampleRate() / bandwidth): unsigned int / int, an unsigned division
   const int decimation = static_cast<int>(sample_rate / BANDWIDTH);
   if (decimation == 0 || hop == 0)
      return -1;

   // :90-96 buffers and plan
   float *fftIn = static_cast<float *>(mufft_alloc(LENGTH * sizeof(float) * 2));
   float *fftOut = static_cast<float *>(mufft_alloc(LENGTH * sizeof(float) * 2));
   float *fftWin = static_cast<float *>(mufft_alloc(LENGTH * sizeof(float) * 2));
   float *fftMag = static_cast<float *>(mufft_alloc(LENGTH * sizeof(float)));
   mufft_plan_1d *fftC2C = mufft_create_plan_1d_c2c(LENGTH, MUFFT_FORWARD, MUFFT_FLAG_CPU_NO_AVX);

   // :126-127 the Hamming case of start()
   for (int n = 0, i = 0; n < LENGTH; ++n, i += 2)
      fftWin[i + 0] = fftWin[i + 1] = static_cast<float>(std::pow(std::sin(static_cast<float>(M_PI * n / LENGTH)), 2));

   long frames = 0;
   // :242 a buffer needs length * decimation samples
   for (uint64_t b = 0; b + (uint64_t) LENGTH * decimation <= n_samples && frames < cap_frames; b += hop, frames++)
   {
      const float *data = iq + 2 * b;

      // :250-263 the SSE2 branch (lab-tasks/CMakeLists.txt:17-19 builds it on x86): floats n .. n + 7 of fftIn are
      // floats i * decimation .. i * decimation + 7 of data times the window, i and n stepping by 8 floats
      for (int i = 0, n = 0; n < (LENGTH << 1); i += 8, n += 8)
         for (int e = 0; e < 8; e++)
            fftIn[n + e] = data[i * decimation + e] * fftWin[n + e];

      // :276
      mufft_execute_plan_1d(fftC2C, fftOut, fftIn);

      // :280-329 sqrt(I^2 + Q^2): _mm_mul_ps, _mm_add_ps, _mm_sqrt_ps, one IEEE operation each
      for (int i = 0; i < LENGTH; i++)
      {
         const float I2 = fftOut[2 * i] * fftOut[2 * i];
         const float Q2 = fftOut[2 * i + 1] * fftOut[2 * i + 1];
         fftMag[i] = std::sqrt(I2 + Q2);
      }

      // :345 negative frequencies first
      float *o = out + (uint64_t) frames * LENGTH;
      std::memcpy(o, fftMag + (LENGTH >> 1), (LENGTH >> 1) * sizeof(float));
      std::memcpy(o + (LENGTH >> 1), fftMag, (LENGTH >> 1) * sizeof(float));
   }

   mufft_free(fftIn);
   mufft_free(fftOut);
   mufft_free(fftMag);
   mufft_free(fftWin);
   mufft_free_plan_1d(fftC2C);
   return frames;
}
}
