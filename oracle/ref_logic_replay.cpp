/*
 * ref_logic_replay.cpp -- the reference's logic capture files end to end (built by oracle/logic_replay.mk).  TEST
 * INFRASTRUCTURE ONLY.
 *
 *   ref_logic_write   writes an 8-bit logic WAV with the reference's hw::RecordDevice in Write mode, as
 *                     SignalStorageTask::writeLogic does (SAMPLE_SIZE_8, one channel per buffer stride), with a given
 *                     epoch and channel keys so that the file is reproducible;
 *   ref_logic_read    reads one back with RecordDevice in Read mode: rate, channels, epoch, keys and the samples as floats;
 *   ref_logic_replay  replays one as SignalStorageTask::readLogic streams it (65 536-sample SIGNAL_TYPE_LOGIC_SAMPLES
 *                     buffers of the file's channel count) into ONE lab::IsoDecoder, nextFrames() per buffer, then
 *                     nextFrames({}) at the end of the file.
 *
 * Like ref_iso_stream.cpp, the file links against the reference's own lab::IsoDecoder (_ref/libnfcref_logic_replay.so)
 * and against the drop-in nfc_laboratory_b200/shim/IsoDecoderB200.cpp over libnfcb200.so (_ref/libnfcref_logic_b200.so),
 * and operator new returns zeroed memory.
 */
#include <cstdlib>
#include <cstring>
#include <list>
#include <new>
#include <vector>

#include <hw/RecordDevice.h>
#include <hw/SignalBuffer.h>
#include <hw/SignalType.h>
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

static constexpr unsigned int BUFFER_SAMPLES = 65536; // SignalStorageTask::readLogic

extern "C" {

/* x: n samples of `channels` floats.  Returns 0, or -1 when the file could not be written. */
int ref_logic_write(const char *path, const float *x, unsigned long n, unsigned int channels, unsigned int rate, unsigned int epoch, const int *keys,
                    unsigned int n_keys)
{
   hw::RecordDevice device(path);
   device.set(hw::SignalDevice::PARAM_SAMPLE_RATE, rate);
   device.set(hw::SignalDevice::PARAM_SAMPLE_SIZE, (unsigned int) hw::SAMPLE_SIZE_8);
   device.set(hw::SignalDevice::PARAM_CHANNEL_COUNT, channels);
   device.set(hw::SignalDevice::PARAM_CHANNEL_KEYS, std::vector<int>(keys, keys + n_keys));
   if (!device.open(hw::RecordDevice::Mode::Write))
      return -1;
   // open() stamps the current time; the header is written again with this epoch on close()
   device.set(hw::SignalDevice::PARAM_STREAM_TIME, epoch);
   for (unsigned long at = 0; at < n; at += BUFFER_SAMPLES)
   {
      const unsigned long len = n - at < BUFFER_SAMPLES ? n - at : BUFFER_SAMPLES;
      hw::SignalBuffer buffer((unsigned int) (len * channels), channels, 1, rate, at, 0, hw::SignalType::SIGNAL_TYPE_LOGIC_SAMPLES);
      buffer.put(x + at * channels, (unsigned int) (len * channels)).flip();
      if (device.write(buffer) < 0)
         return -1;
   }
   device.close();
   return 0;
}

/* header fields into rate / channels / epoch / keys[8], up to cap samples of floats into out.  Returns the samples read
 * (may exceed cap), or -1 when the file is not an 8-bit logic file RecordDevice opens. */
long ref_logic_read(const char *path, unsigned int *rate, unsigned int *channels, unsigned int *epoch, int *keys, float *out, unsigned long cap)
{
   hw::RecordDevice device(path);
   if (!device.open(hw::RecordDevice::Mode::Read) || std::get<unsigned int>(device.get(hw::SignalDevice::PARAM_SAMPLE_SIZE)) != hw::SAMPLE_SIZE_8)
      return -1;
   *rate = std::get<unsigned int>(device.get(hw::SignalDevice::PARAM_SAMPLE_RATE));
   *channels = std::get<unsigned int>(device.get(hw::SignalDevice::PARAM_CHANNEL_COUNT));
   *epoch = std::get<unsigned int>(device.get(hw::SignalDevice::PARAM_STREAM_TIME));
   const auto k = std::get<std::vector<int>>(device.get(hw::SignalDevice::PARAM_CHANNEL_KEYS));
   for (unsigned i = 0; i < 8; i++)
      keys[i] = i < k.size() ? k[i] : 0;
   long total = 0;
   while (device.isOpen() && !device.isEof())
   {
      hw::SignalBuffer buffer(BUFFER_SAMPLES * *channels, *channels, 1, *rate, 0, 0, hw::SignalType::SIGNAL_TYPE_LOGIC_SAMPLES);
      if (device.read(buffer) <= 0)
         break;
      const unsigned long got = buffer.elements();
      for (unsigned long i = 0; i < got * *channels; i++)
         if (total * *channels + i < cap * *channels)
            out[total * *channels + i] = buffer.data()[i];
      total += got;
   }
   return total;
}

/* the frames of one logic WAV replayed as SignalStorageTask::readLogic streams it.  Writes up to cap frames, returns the
 * number decoded (may exceed cap), or -1 when the file is not an 8-bit logic file. */
long ref_logic_replay(const char *path, unsigned int stream_time, nfcb200_frame *out, long cap)
{
   long k = 0;
   {
   hw::RecordDevice device(path);
   if (!device.open(hw::RecordDevice::Mode::Read) || std::get<unsigned int>(device.get(hw::SignalDevice::PARAM_SAMPLE_SIZE)) != hw::SAMPLE_SIZE_8)
      return -1;
   const unsigned int rate = std::get<unsigned int>(device.get(hw::SignalDevice::PARAM_SAMPLE_RATE));
   const unsigned int channels = std::get<unsigned int>(device.get(hw::SignalDevice::PARAM_CHANNEL_COUNT));

   lab::IsoDecoder decoder;
   decoder.setStreamTime(stream_time);

   std::list<lab::RawFrame> frames;
   while (true)
   {
      const unsigned int offset = std::get<unsigned int>(device.get(hw::SignalDevice::PARAM_SAMPLE_OFFSET));
      hw::SignalBuffer buffer(BUFFER_SAMPLES * channels, channels, 1, rate, offset, 0, hw::SignalType::SIGNAL_TYPE_LOGIC_SAMPLES);
      if (device.read(buffer) > 0)
         frames.splice(frames.end(), decoder.nextFrames(buffer));
      if (device.isEof() || !device.isOpen())
         break;
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
