/*
 * ref_iso.cpp -- C wrapper around the reference's UNMODIFIED lab::IsoDecoder (built by oracle/iso.mk).  TEST
 * INFRASTRUCTURE ONLY.  The answer for a capture is one nextFrames() call on the whole capture as a 4-channel
 * SIGNAL_TYPE_LOGIC_SAMPLES buffer (IO, CLK, RST, VCC), then nextFrames({}) -- what the reference's logic decoder task
 * does with a capture handed to it in one buffer.
 *
 * The decoder reads memory it never writes: the "previous sample" of the first sample (IsoTech.cpp:43 compares an
 * unsigned clock with 0, so the initialisation never runs) and frame bytes past a frame's end (Iso7816.cpp:1042-1145,
 * 1183-1192).  This library's operator new returns zeroed memory (iso.mk links with -Bsymbolic, so the reference units
 * use it), so those reads see 0 and the answer does not depend on what the process allocated before.
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

static void put_frame(const lab::RawFrame &f, nfcb200_frame &o)
{
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

extern "C" {

/* samples: n x 4 floats.  Writes up to cap frames, returns the number decoded (may exceed cap). */
long ref_iso_decode(const float *samples, unsigned long n, unsigned int sample_rate, unsigned int stream_time, nfcb200_frame *out, long cap)
{
   long k = 0;
   {
   lab::IsoDecoder decoder;
   decoder.setStreamTime(stream_time);

   hw::SignalBuffer buffer((unsigned int) (n * 4), 4, 1, sample_rate, 0, 0, hw::SignalType::SIGNAL_TYPE_LOGIC_SAMPLES);
   buffer.put(samples, (unsigned int) (n * 4)).flip();

   std::list<lab::RawFrame> frames = decoder.nextFrames(buffer);
   frames.splice(frames.end(), decoder.nextFrames({}));

   for (const auto &f: frames)
   {
      if (k < cap)
         put_frame(f, out[k]);
      k++;
   }
   }
   return k;
}
}
