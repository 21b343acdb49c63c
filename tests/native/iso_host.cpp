/*
 * tests/native/iso_host.cpp -- TEST-ONLY host build of the ISO 7816 decoder (csrc/iso_core.h).
 *
 * Finds the events of a 4-channel logic capture (IO, CLK, RST, VCC) the way iso_edges_kernel does and walks them with
 * iso_walk(), the code the walk kernel runs, so that the event-driven decoder can be checked against the reference
 * without a GPU.  Never linked into the product library.
 *
 * Build (tests/iso_ref.py does this): g++ -O2 -msse2 -mfpmath=sse -ffp-contract=off -shared -fPIC
 */
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../include/nfcb200.h"
#include "../../nfc_laboratory_b200/csrc/iso_core.h"

using namespace iso7816;

struct HostEvents
{
   std::vector<uint32_t> lineAt, lineFlags, clk;
   size_t li = 0, ci = 0;

   uint32_t line_peek() const { return li < lineAt.size() ? lineAt[li] : NONE; }
   uint32_t line_pop() { return lineFlags[li++]; }
   uint32_t clk_nth(uint32_t k) const { return ci + k < clk.size() ? clk[ci + k] : NONE; }
   void clk_pop() { ci++; }
   void clk_skip(uint32_t k) { ci += k; }
};

struct HostSink
{
   nfcb200_frame *out;
   long cap, count;
   uint32_t stream, rate;

   void frame(const IsoFrameOut &f)
   {
      if (count < cap)
      {
         nfcb200_frame &o = out[count];
         std::memset(&o, 0, sizeof(o));
         o.stream = stream;
         o.tech_type = f.techType;
         o.frame_type = f.frameType;
         o.frame_flags = f.frameFlags;
         o.frame_phase = f.framePhase;
         o.frame_rate = f.frameRate;
         o.length = f.length;
         o.sample_start = f.sampleStart;
         o.sample_end = f.sampleEnd;
         o.sample_rate = rate;
         o.time_start = f.timeStart;
         o.time_end = f.timeEnd;
         o.date_time = f.dateTime;
         for (uint32_t i = 0; i < f.length && i < FRAME_BYTES; i++)
            o.data[i] = f.data[i];
      }
      count++;
   }
};

extern "C" {

/* samples: [n_streams][n][4] float32 (sigtype 5) or int16 (sigtype 6).  Returns the number of frames (may exceed cap). */
long iso_host_decode(const void *samples, int sigtype, uint32_t n_streams, uint64_t n, uint32_t rate, uint32_t stream_time, nfcb200_frame *out,
                     long cap)
{
   HostSink sink {out, cap, 0, 0, rate};
   IsoMachine *m = new IsoMachine;
   for (uint32_t s = 0; s < n_streams; s++)
   {
      HostEvents ev;
      float last[4] = {0, 0, 0, 0};
      for (uint64_t i = 0; i < n; i++)
      {
         float d[4];
         for (int c = 0; c < 4; c++)
            d[c] = sigtype == 6 ? ((const int16_t *) samples)[(s * n + i) * 4 + c] / 32768.f : ((const float *) samples)[(s * n + i) * 4 + c];
         const uint32_t f = sample_flags(d, last);
         if (f & F_LINE)
         {
            ev.lineAt.push_back((uint32_t) i);
            ev.lineFlags.push_back(f & ~F_CLK_FALL);
         }
         if (f & F_CLK_FALL)
            ev.clk.push_back((uint32_t) i);
         std::memcpy(last, d, sizeof(last));
      }
      sink.stream = s;
      iso_init(*m, rate, stream_time);
      iso_walk(*m, ev, (uint32_t) n, sink);
   }
   delete m;
   return sink.count;
}
}
