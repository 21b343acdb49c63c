/*
 * ref_iso_stream.cpp -- C wrapper around ONE lab::IsoDecoder fed a capture buffer by buffer (built by oracle/iso_stream.mk).
 * TEST INFRASTRUCTURE ONLY.  The answer for a chunk plan is one nextFrames() call per chunk, each a 4-channel
 * SIGNAL_TYPE_LOGIC_SAMPLES buffer at that chunk's sample rate, then nextFrames({}) -- what the reference's
 * LogicDecoderTask does with the buffers of a live capture (LogicDecoderTask.cpp:300, then :186 on stop).
 *
 * The same file links against two implementations of lab::IsoDecoder: the reference's own units
 * (_ref/libnfcref_iso_stream.so) and the drop-in nfc_laboratory_b200/shim/IsoDecoderB200.cpp over libnfcb200.so
 * (_ref/libnfcref_iso_b200.so).  Like ref_iso.cpp, operator new returns zeroed memory, so the reference's reads of memory
 * it never wrote (the sample before the first, frame bytes past a frame's end) see 0.
 */
#include <cstdlib>
#include <cstring>
#include <list>
#include <new>

#include <hw/SignalType.h>
#include <hw/SignalBuffer.h>
#include <lab/data/RawFrame.h>
#include <lab/iso/IsoDecoder.h>

#include <nfcb200.h>

void *operator new(std::size_t n)
{
   if (void *p = std::calloc(1, n ? n : 1))
      return p;
   throw std::bad_alloc();
}

void *operator new[](std::size_t n)
{
   return operator new(n);
}

void operator delete(void *p) noexcept
{
   std::free(p);
}

void operator delete[](void *p) noexcept
{
   std::free(p);
}

void operator delete(void *p, std::size_t) noexcept
{
   std::free(p);
}

void operator delete[](void *p, std::size_t) noexcept
{
   std::free(p);
}

extern "C" {

/* samples: n x 4 floats cut into n_chunks buffers of chunks[i] samples at rates[i] S/s (the chunks sum to n).  Writes up
 * to cap frames, returns the number decoded (may exceed cap). */
long ref_iso_decode_chunks(const float *samples, unsigned long n, const unsigned int *rates, unsigned int stream_time, const unsigned long *chunks,
                           unsigned long n_chunks, nfcb200_frame *out, long cap)
{
   long k = 0;
   {
   lab::IsoDecoder decoder;
   decoder.setStreamTime(stream_time);

   std::list<lab::RawFrame> frames;
   unsigned long at = 0;
   for (unsigned long c = 0; c < n_chunks && at < n; c++)
   {
      const unsigned long len = chunks[c] < n - at ? chunks[c] : n - at;
      hw::SignalBuffer buffer((unsigned int) (len * 4), 4, 1, rates[c], 0, 0, hw::SignalType::SIGNAL_TYPE_LOGIC_SAMPLES);
      buffer.put(samples + at * 4, (unsigned int) (len * 4)).flip();
      frames.splice(frames.end(), decoder.nextFrames(buffer));
      at += len;
   }
   frames.splice(frames.end(), decoder.nextFrames({}));

   for (const auto &f: frames)
   {
      if (k < cap)
      {
         nfcb200_frame &o = out[k];
         std::memset(&o, 0, sizeof(o));
         o.tech_type = f.techType();
         o.frame_type = f.frameType();
         o.frame_flags = f.frameFlags();
         o.frame_phase = f.framePhase();
         o.frame_rate = f.frameRate();
         o.length = f.limit();
         o.sample_start = f.sampleStart();
         o.sample_end = f.sampleEnd();
         o.sample_rate = f.sampleRate();
         o.time_start = f.timeStart();
         o.time_end = f.timeEnd();
         o.date_time = f.dateTime();
         for (unsigned i = 0; i < o.length && i < sizeof(o.data); i++)
            o.data[i] = f[i];
      }
      k++;
   }
   }
   return k;
}
}
