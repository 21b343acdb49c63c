/*
 * tests/native/adaptive_host.cpp -- TEST-ONLY host build of the adaptive signal (csrc/adaptive.cuh).
 *
 * Runs the kernels' per-sample steps (radio_start / radio_step / radio_end, logic_step) over one stream of float values,
 * buffer after buffer, so that the device result can be compared with it bit for bit and the algorithm can be checked
 * against the reference without a GPU.  Input is what the kernels step: the magnitude (radio), the channel values as the
 * reference reads them (logic).  Never linked into the product library.
 *
 * Build (tests/adaptive_ref.py does this): g++ -O2 -msse2 -mfpmath=sse -ffp-contract=off -shared -fPIC
 */
#include <cstdint>

#include "../../nfc_laboratory_b200/csrc/adaptive.cuh"

using namespace nfcb200;

namespace {

struct Sink
{
   float *val;
   uint64_t *sample;
   uint32_t *channel;
   uint64_t cap, n, base;
   uint32_t ch;
   void operator()(float v, int i)
   {
      if (n < cap)
      {
         val[n] = v;
         sample[n] = base + (uint32_t) (float) i;
         if (channel)
            channel[n] = ch;
      }
      n++;
   }
};

}

extern "C" {

// the points of one radio stream x[0 .. n) cut into buffers of buffer_len: returns their number, writes up to cap
uint64_t adaptive_radio_host(const float *x, uint64_t n, uint64_t buffer_len, uint64_t offset, float *val, uint64_t *sample, uint64_t cap)
{
   Sink out{val, sample, nullptr, cap, 0, 0, 0};
   for (uint64_t b0 = 0; b0 < n; b0 += buffer_len)
   {
      const float *xb = x + b0;
      const int limit = (int) (n - b0 < buffer_len ? n - b0 : buffer_len);
      auto tap = [&](int i) { return i >= 0 && i < limit ? xb[i] : 0.f; };
      out.base = offset + b0;
      RadioState s = radio_start(tap, limit);
      out(xb[0], 0);
      for (int i = 0; i < limit; i++)
         radio_step(s, i, limit, xb[i], tap(i + AD_HALF), tap(i - AD_HALF - 1), out);
      radio_end(s, limit, out);
   }
   return out.n;
}

// the points of one logic stream x[0 .. n)[ch], ordered by (channel, buffer, emission order)
uint64_t adaptive_logic_host(const float *x, uint32_t ch, uint64_t n, uint64_t buffer_len, uint64_t offset, float *val, uint64_t *sample,
                             uint32_t *channel, uint64_t cap)
{
   Sink out{val, sample, channel, cap, 0, 0, 0};
   for (uint32_t c = 0; c < ch; c++)
   {
      if (c == 1)
         continue;
      out.ch = c;
      for (uint64_t b0 = 0; b0 < n; b0 += buffer_len)
      {
         const uint64_t limit = n - b0 < buffer_len ? n - b0 : buffer_len;
         out.base = offset + b0;
         float last = x[b0 * ch + c];
         uint32_t kept = 0;
         out(last, 0);
         for (uint32_t s = 1; s < limit; s++)
            logic_step(last, kept, s, x[(b0 + s) * ch + c], out);
      }
   }
   return out.n;
}
}
