/*
 * oracle/ref_adaptive.cpp -- TEST INFRASTRUCTURE ONLY: the reference's UNMODIFIED lab::SignalResamplingTask and
 * lab::TraceStorageTask (built by oracle/adaptive.mk), driven through their subjects as the reference's GUI drives them.
 *
 * A stream is cut into buffers as SignalStorageTask::readRadio / readLogic cut a file (SignalStorageTask.cpp:323-437):
 * buffer_len samples at a time, the last buffer shorter, offset() the position of the buffer's first sample.  Each buffer
 * is published on "radio.signal.raw" (SIGNAL_TYPE_RADIO_SAMPLES, the magnitude) or "logic.signal.raw"
 * (SIGNAL_TYPE_LOGIC_SAMPLES, `channels` floats per sample) and the resampler's loop() is run once for it; the buffers it
 * publishes on "adaptive.signal" are collected.  With a file name the trace task, subscribed to "adaptive.signal" as well,
 * is then sent its Write command on "storage.command" and writes the .trz (frame.json and the .apcm entries).
 *
 * The tasks' loop() is protected in rt::Worker; Loop below names it through a derived class, which C++ allows, and calls
 * it on this thread: no worker threads, so the order of buffers is the order of publication.  lab-tasks is compiled without
 * OpenMP, so processLogicSignal's channels come in order.
 */
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include <rt/Event.h>
#include <rt/Subject.h>
#include <rt/Worker.h>

#include <hw/SignalBuffer.h>
#include <hw/SignalType.h>

#include <lab/tasks/SignalResamplingTask.h>
#include <lab/tasks/TraceStorageTask.h>

namespace {

struct Loop : rt::Worker
{
   static bool run(rt::Worker *w)
   {
      return (w->*(&Loop::loop))();
   }
};

}

extern "C" {

/*
 * x: [n][channels] floats, channels == 0 for radio (then [n] magnitudes).  Points are written ordered as the resampler
 * publishes them (buffer, then channel, then emission order): value, offset() + (unsigned) index, channel (buffer id).
 * Returns the number of points (writes up to cap) or -1.  trz: when not null, the trace task writes this file; with
 * has_range the command carries timeStart / timeEnd, without it carries neither.
 */
long nfcref_adaptive(const float *x, uint32_t channels, uint64_t n, uint32_t rate, uint64_t buffer_len, uint64_t offset, float *val, uint64_t *sample,
                     uint32_t *channel, long cap, const char *trz, int has_range, double time_start, double time_end)
{
   const bool logic = channels != 0;
   const uint32_t stride = logic ? channels : 1;
   rt::Worker *resampler = lab::SignalResamplingTask::construct();
   rt::Worker *storage = trz ? lab::TraceStorageTask::construct() : nullptr;

   long count = 0;
   int rc = 0;
   {
   auto *adaptive = rt::Subject<hw::SignalBuffer>::name("adaptive.signal");
   auto sub = adaptive->subscribe([&](const hw::SignalBuffer &b) {
      if (!b.isValid())
         return;
      for (unsigned int i = 0; i < b.limit(); i += b.stride(), count++)
      {
         if (count < cap)
         {
            val[count] = b[i];
            sample[count] = b.offset() + static_cast<unsigned int>(b[i + 1]);
            channel[count] = b.id();
         }
      }
   });

   auto *raw = rt::Subject<hw::SignalBuffer>::name(logic ? "logic.signal.raw" : "radio.signal.raw");
   for (uint64_t b0 = 0; b0 < n; b0 += buffer_len)
   {
      const uint64_t len = n - b0 < buffer_len ? n - b0 : buffer_len;
      hw::SignalBuffer buffer((unsigned int) (len * stride), stride, 1, rate, offset + b0, 0,
                              logic ? hw::SignalType::SIGNAL_TYPE_LOGIC_SAMPLES : hw::SignalType::SIGNAL_TYPE_RADIO_SAMPLES);
      for (uint64_t k = 0; k < len * stride; k++)
         buffer.put(x[b0 * stride + k]);
      buffer.flip();
      raw->next(buffer);
      Loop::run(resampler);
   }

   if (storage)
   {
      std::string data = std::string("{\"fileName\":\"") + trz + "\"";
      if (has_range)
      {
         char range[128];
         snprintf(range, sizeof(range), ",\"timeStart\":%.17g,\"timeEnd\":%.17g", time_start, time_end);
         data += range;
      }
      data += "}";
      bool done = false;
      auto *command = rt::Subject<rt::Event>::name("storage.command");
      command->next({lab::TraceStorageTask::Write, [&]() { done = true; }, [&](int, const std::string &) { rc = -1; },
                     {{"data", data}}});
      Loop::run(storage);
      if (!done)
         rc = -1;
   }

   } // the subscription ends here
   delete storage;
   delete resampler;
   return rc ? -1 : count;
}
}
