/*
 * tests/native/iso_stream_host.cpp -- TEST-ONLY host build of the streaming ISO 7816 decode (nfcb200_iso7816_stream_push).
 *
 * Pushes a 4-channel logic capture buffer by buffer through the code the device runs per push: the events of each buffer
 * against the last sample of the previous one (iso_edges_kernel's `last`), then iso_restart() on a new sample rate or
 * iso_resume() otherwise, and iso_walk() from the buffer's first sample with the carried IsoCarry.  Never linked into the
 * product library.
 *
 * Build (tests/iso_stream_ref.py does this): g++ -O2 -msse2 -mfpmath=sse -ffp-contract=off -shared -fPIC
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
   uint32_t rate;

   void frame(const IsoFrameOut &f)
   {
      if (count < cap)
      {
         nfcb200_frame &o = out[count];
         std::memset(&o, 0, sizeof(o));
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

/* samples: [n][4] float32 (sigtype 5) or int16 (sigtype 6), pushed as n_chunks buffers of chunks[i] samples at rates[i]
 * S/s.  Returns the number of frames (may exceed cap). */
long iso_host_stream(const void *samples, int sigtype, uint64_t n, const uint64_t *chunks, const uint32_t *rates, uint32_t n_chunks,
                     uint32_t stream_time, nfcb200_frame *out, long cap)
{
   HostSink sink {out, cap, 0, 0};
   IsoStreamState *st = new IsoStreamState;
   std::memset(st, 0, sizeof(*st));
   float last[4] = {0, 0, 0, 0};
   bool init = false;
   uint32_t rate = 0, clock = 0;
   uint64_t at = 0;
   for (uint32_t k = 0; k < n_chunks && at < n; k++)
   {
      const uint64_t len = chunks[k] < n - at ? chunks[k] : n - at;
      if (len == 0)
         continue; // nextFrames({}) decodes nothing
      const bool restart = !init || rate != rates[k];
      const uint32_t base = restart ? 0 : clock;
      HostEvents ev;
      for (uint64_t i = 0; i < len; i++)
      {
         float d[4];
         for (int c = 0; c < 4; c++)
            d[c] = sigtype == 6 ? ((const int16_t *) samples)[(at + i) * 4 + c] / 32768.f : ((const float *) samples)[(at + i) * 4 + c];
         const uint32_t f = sample_flags(d, last);
         if (f & F_LINE)
         {
            ev.lineAt.push_back(base + (uint32_t) i);
            ev.lineFlags.push_back(f & ~F_CLK_FALL);
         }
         if (f & F_CLK_FALL)
            ev.clk.push_back(base + (uint32_t) i);
         std::memcpy(last, d, sizeof(last));
      }
      if (restart)
         iso_restart(st->m, st->c, rates[k], stream_time);
      else
         iso_resume(st->m, st->c, base);
      st->m.streamTime = stream_time;
      sink.rate = rates[k];
      iso_walk(st->m, st->c, ev, base + (uint32_t) len, sink);
      init = true;
      rate = rates[k];
      clock = base + (uint32_t) len;
      at += len;
   }
   delete st;
   return sink.count;
}
}
