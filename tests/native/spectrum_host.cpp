/*
 * tests/native/spectrum_host.cpp -- TEST-ONLY host build of the spectrum transform (csrc/nfc_spectrum.cuh).
 *
 * Runs the kernel's arithmetic in the kernel's order, one butterfly index j at a time, so that the device result can be
 * compared with it bit for bit and the transform can be checked against the reference without a GPU.  Never linked into
 * the product library.
 *
 * Build (tests/test_spectrum.py does this): g++ -O2 -msse2 -mfpmath=sse -ffp-contract=off -shared -fPIC
 */
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../nfc_laboratory_b200/csrc/nfc_spectrum.cuh"

using namespace nfcb200;

// one frame: the 1024 window positions of a buffer starting at `frame`, into 1024 shifted magnitudes
template <bool S16>
static void frame_host(const void *frame, uint32_t dec, const SpecCx *tw, const float *win, float *out)
{
   std::vector<SpecCx> x(SPEC_LEN), y(SPEC_LEN);
   for (uint32_t j = 0; j < SPEC_LEN / 8; j++)
   {
      SpecCx v[8];
      for (uint32_t r = 0; r < 8; r++)
      {
         const uint32_t k = j + r * (SPEC_LEN / 8);
         const uint64_t idx = spec_offset(k, dec);
         if (S16)
         {
            const short *q = (const short *) frame + 2 * idx;
            v[r] = spec_windowed_s16(q[0], q[1], win[k]);
         }
         else
         {
            const float *q = (const float *) frame + 2 * idx;
            v[r] = spec_windowed(q[0], q[1], win[k]);
         }
      }
      dft8(v);
      for (uint32_t r = 0; r < 8; r++)
         x[spec_dest(j, 1, 8, r)] = v[r];
   }
   for (uint32_t ns = 8; ns <= 64; ns *= 8)
   {
      for (uint32_t j = 0; j < SPEC_LEN / 8; j++)
      {
         SpecCx v[8];
         for (uint32_t r = 0; r < 8; r++)
            v[r] = x[j + r * (SPEC_LEN / 8)];
         spec_twiddle8(v, tw, j, ns);
         dft8(v);
         for (uint32_t r = 0; r < 8; r++)
            y[spec_dest(j, ns, 8, r)] = v[r];
      }
      x.swap(y);
   }
   for (uint32_t j = 0; j < SPEC_LEN / 2; j++)
      spec_last(x[j], x[j + SPEC_LEN / 2], tw[j], out[j + SPEC_LEN / 2], out[j]);
}

extern "C" {

// the same contract as nfcb200_spectrum with host memory on both sides; sigtype 1 float32 IQ, 4 int16 IQ.  Returns the
// frames per stream, or -1 for an argument the library would reject
long spectrum_host(const void *samples, int sigtype, uint32_t n_streams, uint64_t n_samples, uint32_t sample_rate, uint64_t hop, float *out)
{
   if ((sigtype != 1 && sigtype != 4) || hop == 0 || sample_rate < SPEC_BANDWIDTH)
      return -1;
   const uint32_t dec = spectrum_decimation(sample_rate);
   const uint64_t nf = spectrum_frames(n_samples, dec, hop);
   SpecCx tw[SPEC_LEN];
   float win[SPEC_LEN];
   spectrum_tables(tw, win);
   const uint64_t bs = sigtype == 1 ? 8 : 4;
   for (uint64_t s = 0; s < n_streams; s++)
      for (uint64_t f = 0; f < nf; f++)
      {
         const unsigned char *frame = (const unsigned char *) samples + (s * n_samples + f * hop) * bs;
         float *o = out + (s * nf + f) * SPEC_LEN;
         if (sigtype == 1)
            frame_host<false>(frame, dec, tw, win, o);
         else
            frame_host<true>(frame, dec, tw, win, o);
      }
   return (long) nf;
}

// the window as uploaded to the device (spectrum_tables)
void spectrum_host_window(float *win)
{
   SpecCx tw[SPEC_LEN];
   spectrum_tables(tw, win);
}
}
