/*
 * IsoDecoderB200.cpp -- drop-in implementation of the reference class lab::IsoDecoder on top of libnfcb200.so.
 *
 * Like NfcDecoderB200.cpp for the radio side: whoever provides liblab-logic provides the decoder
 * (lab-logic/src/main/include/lab/iso/IsoDecoder.h:33-68, pimpl std::shared_ptr<Impl>).  This file is compiled INSTEAD of
 * the reference's lab-logic/src/main/cpp/{IsoDecoder,IsoTech}.cpp and tech/Iso7816.cpp, against the reference's own
 * UNMODIFIED headers, and forwards every call to the ISO 7816 stream calls of include/nfcb200.h, so LogicDecoderTask
 * compiles and links unchanged (INTEGRATION.md).
 *
 * Behaviour mirrored from IsoDecoder.cpp: nextFrames() of a logic buffer decodes it and carries the decoder to the next
 * one; a buffer at another sample rate restarts the decoder (:172-178); nextFrames() of an invalid buffer decodes nothing
 * (:184-208, IsoTech.cpp:31-32); initialize() restarts the decoder at the next buffer.  Debug is accepted and ignored.
 * setEnableISO7816(false) keeps pushing the samples, so the sample clock advances, and drops the frames (DESIGN.md
 * section 13 lists where that differs from the reference).
 */
#include <list>
#include <memory>
#include <string>
#include <vector>

#include <hw/SignalType.h>
#include <hw/SignalBuffer.h>

#include <lab/data/RawFrame.h>
#include <lab/iso/IsoDecoder.h>

#include <nfcb200.h>

namespace lab {

struct IsoDecoder::Impl
{
   nfcb200_config cfg {};
   nfcb200_handle *handle = nullptr;
   bool debugEnabled = false;
   bool iso7816Enabled = true;
   long sampleRate = 0;
   bool dirty = true; // stream time changed since the handle last saw the configuration
   std::vector<nfcb200_frame> frames;
   int lastStatus = 0;      // status of the last library call (0 = ok): lab::IsoDecoder has no error channel and its caller
   std::string lastMessage; // (LogicDecoderTask.cpp:300) no try / catch -- failures are kept here, never thrown

   Impl()
   {
      nfcb200_config_default(&cfg);
      frames.resize(4096);
   }

   ~Impl()
   {
      if (handle)
         nfcb200_destroy(handle);
   }

   bool note(int rc)
   {
      lastStatus = rc;
      lastMessage = rc ? nfcb200_last_error() : "";
      return rc == 0;
   }

   bool ensure()
   {
      if (!handle && !note(nfcb200_create(&cfg, &handle)))
      {
         handle = nullptr;
         return false;
      }
      if (dirty)
      {
         note(nfcb200_configure(handle, &cfg));
         dirty = false;
      }
      return true;
   }

   void initialize()
   {
      if (ensure())
         note(nfcb200_iso7816_stream_reset(handle));
   }

   static RawFrame convert(const nfcb200_frame &f)
   {
      RawFrame frame(f.tech_type, f.frame_type);
      frame.setFramePhase(f.frame_phase);
      frame.setFrameFlags(f.frame_flags);
      frame.setFrameRate(f.frame_rate);
      frame.setSampleStart(f.sample_start);
      frame.setSampleEnd(f.sample_end);
      frame.setSampleRate(f.sample_rate);
      frame.setTimeStart(f.time_start);
      frame.setTimeEnd(f.time_end);
      frame.setDateTime(f.date_time);
      frame.put(f.data, f.length).flip();
      return frame;
   }

   std::list<RawFrame> nextFrames(hw::SignalBuffer &samples)
   {
      std::list<RawFrame> result;

      if (!ensure())
         return result; // no device: an empty list, the reason is in lastMessage

      uint64_t count = 0;
      int rc;

      if (samples.isValid())
      {
         sampleRate = samples.sampleRate();

         // only logic buffers carry samples for this decoder (IsoTech.cpp:33); it reads channels 0-3 of buffers of 4 to 8
         // channels (a stride outside that range is ignored, DESIGN.md section 13)
         const unsigned int stride = samples.stride();

         if (samples.type() != hw::SignalType::SIGNAL_TYPE_LOGIC_SAMPLES || stride < 4 || stride > 8)
            return result;

         const uint64_t n = samples.remaining() / stride;

         if (n == 0)
            return result;

         rc = nfcb200_iso7816_stream_push_ch(handle, samples.data() + samples.position(), NFCB200_SIG_LOGIC_F32, stride, n, (uint32_t) sampleRate,
                                             frames.data(), frames.size(), &count);
      }
      else
      {
         rc = nfcb200_iso7816_stream_push(handle, nullptr, NFCB200_SIG_LOGIC_F32, 0, (uint32_t) sampleRate, frames.data(), frames.size(), &count);
      }

      for (uint64_t i = 0; i < count; i++)
         result.push_back(convert(frames[i]));

      // more frames than the buffer holds: drain the rest (nothing is dropped, nothing is thrown)
      while (rc == NFCB200_ERR_CAPACITY)
      {
         uint64_t left = 0;
         if (nfcb200_iso7816_stream_pending(handle, frames.data(), frames.size(), &count, &left) != 0)
            break;
         for (uint64_t i = 0; i < count; i++)
            result.push_back(convert(frames[i]));
         if (left == 0)
            rc = 0;
      }

      note(rc);

      if (!iso7816Enabled)
         result.clear();

      return result;
   }
};

IsoDecoder::IsoDecoder() : impl(std::make_shared<Impl>())
{
}

void IsoDecoder::initialize()
{
   impl->initialize();
}

void IsoDecoder::cleanup()
{
}

std::list<RawFrame> IsoDecoder::nextFrames(hw::SignalBuffer samples)
{
   return impl->nextFrames(samples);
}

bool IsoDecoder::isDebugEnabled() const { return impl->debugEnabled; }
void IsoDecoder::setEnableDebug(bool enabled) { impl->debugEnabled = enabled; }

bool IsoDecoder::isISO7816Enabled() const { return impl->iso7816Enabled; }
void IsoDecoder::setEnableISO7816(bool enabled) { impl->iso7816Enabled = enabled; }

long IsoDecoder::sampleRate() const { return impl->sampleRate; }
void IsoDecoder::setSampleRate(long sampleRate) { impl->sampleRate = sampleRate; }

long IsoDecoder::streamTime() const { return impl->cfg.stream_time; }
void IsoDecoder::setStreamTime(long referenceTime) { impl->cfg.stream_time = (uint32_t) referenceTime; impl->dirty = true; }

}
