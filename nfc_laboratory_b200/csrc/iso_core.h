/*
 * iso_core.h -- the ISO 7816 contact smart-card decoder (lab::IsoDecoder with lab::Iso7816, IsoDecoder.cpp:164-215,
 * IsoTech.cpp:31-75, Iso7816.cpp:244-1435) restated as __host__ __device__ code driven by events instead of samples.
 *
 * The reference steps a state machine on every sample of a 4-channel logic capture (IO, CLK, RST, VCC).  A step reads
 * the sample only through the sign of each channel's edge (sample - previous sample), whether IO and VCC are above 0, and
 * comparisons of the sample clock with three timers of the modulation status (searchStartTime / searchEndTime /
 * searchSyncTime).  So a step on a sample where no IO / RST / VCC edge and no counted CLK falling edge happens depends on
 * the state alone until the clock crosses one of those timers: if such a step leaves the state unchanged, so do all the
 * following ones up to the next timer or edge.  iso_walk() therefore steps only
 *   - samples with an IO, RST or VCC edge (line events),
 *   - the CLK falling edge that brings the clock counter to 10 (Iso7816.cpp:319: the only one that measures the clock),
 *   - the sample after a step that changed the state, and the next timer after one that did not.
 * The other CLK falling edges are counted in bulk.  The clock fields of the modulation status are written only by a CLK
 * falling edge and read by nothing else, so they are left out of the comparison.
 *
 * Timing math is double, in the reference's operation order (the unit is compiled with -fmad=false); conversions of a
 * double to an unsigned field follow the x86-64 code the reference build runs (iso_d2u / iso_d2ul).
 *
 * Deviations (DESIGN.md section 13): the frame payload holds 512 bytes (the reference's frameData holds 1024 with no
 * bound check): later bytes are counted but not stored and the frame is flagged Truncated; bytes past the end of a frame
 * read as 0 (the reference reads whatever its buffer holds there); the sample before the first one is taken as 0 on every
 * channel (the reference leaves it uninitialised, IsoTech.cpp:43 compares an unsigned clock with 0).
 */
#ifndef NFCB200_ISO_CORE_H
#define NFCB200_ISO_CORE_H

#include <stdint.h>

#ifdef __CUDACC__
#define ISO_HD __host__ __device__ __forceinline__
#else
#include <cmath>
#define ISO_HD inline
#endif

namespace iso7816 {

constexpr uint32_t NONE = 0xFFFFFFFFu;
constexpr uint32_t FRAME_BYTES = 512;

// per-sample flags: edge classes of IO / RST / VCC (edge < 0, > 0, != 0), IO and VCC above 0, CLK falling edge
enum : uint32_t
{
   F_IO_NEG = 1u << 0, F_IO_POS = 1u << 1, F_IO_CHG = 1u << 2,
   F_RST_NEG = 1u << 3, F_RST_POS = 1u << 4, F_RST_CHG = 1u << 5,
   F_VCC_NEG = 1u << 6, F_VCC_POS = 1u << 7, F_VCC_CHG = 1u << 8,
   F_IO_HIGH = 1u << 9, F_VCC_HIGH = 1u << 10,
   F_CLK_FALL = 1u << 11,
   F_LINE = F_IO_CHG | F_RST_CHG | F_VCC_CHG,
   F_LEVELS = F_IO_HIGH | F_VCC_HIGH,
   F_BITS = 12
};

// flags of one sample from its 4 channels and the previous sample's (IsoTech.cpp:52-58: edge = data - last, in float).
// T = int: 8-bit samples b as their integer values.  The flags are those of b / 255.f: that map is strictly increasing and
// 0 only at b = 0, and the float difference of two distinct values is never 0, so every sign test gives the same answer.
template <class T>
ISO_HD uint32_t sample_flags(const T d[4], const T l[4])
{
   const T io = d[0] - l[0], clk = d[1] - l[1], rst = d[2] - l[2], vcc = d[3] - l[3];
   uint32_t f = 0;
   f |= io < 0 ? F_IO_NEG : 0u;
   f |= io > 0 ? F_IO_POS : 0u;
   f |= io != 0 ? F_IO_CHG : 0u;
   f |= rst < 0 ? F_RST_NEG : 0u;
   f |= rst > 0 ? F_RST_POS : 0u;
   f |= rst != 0 ? F_RST_CHG : 0u;
   f |= vcc < 0 ? F_VCC_NEG : 0u;
   f |= vcc > 0 ? F_VCC_POS : 0u;
   f |= vcc != 0 ? F_VCC_CHG : 0u;
   f |= d[0] > 0 ? F_IO_HIGH : 0u;
   f |= d[3] > 0 ? F_VCC_HIGH : 0u;
   f |= clk < 0 ? F_CLK_FALL : 0u;
   return f;
}

// frame constants (lab-data RawFrame.h:41-82)
enum : uint32_t
{
   TECH_ISO_ANY = 0x0200, TECH_ISO7816 = 0x0201,
   VCC_LOW = 0x0200, VCC_HIGH = 0x0201, RST_LOW = 0x0202, RST_HIGH = 0x0203,
   ATR_FRAME = 0x0210, REQUEST_FRAME = 0x0211, RESPONSE_FRAME = 0x0212, EXCHANGE_FRAME = 0x0213,
   ISO_ANY_PHASE = 0x0200,
   FLAG_TRUNCATED = 0x08, FLAG_PARITY = 0x10, FLAG_CRC = 0x20
};

// Iso.h:28-67
ISO_HD int fi_table(uint32_t i)
{
   const int t[16] = {0, 372, 558, 744, 1116, 1488, 1860, 0, 0, 512, 768, 1024, 1536, 2048, 0, 0};
   return t[i & 15];
}
ISO_HD int di_table(uint32_t i)
{
   const int t[16] = {0, 1, 2, 4, 8, 16, 32, 64, 12, 20, 0, 0, 0, 0, 0, 0};
   return t[i & 15];
}
ISO_HD int bwt_table(uint32_t i)
{
   const int t[16] = {960, 1920, 3840, 7680, 15360, 30720, 61440, 122880, 245760, 491520, 0, 0, 0, 0, 0, 0};
   return t[i & 15];
}
ISO_HD int cwt_table(uint32_t i)
{
   return 1 << (i & 15);
}

constexpr uint32_t FI_DEF = 1, DI_DEF = 1, IFSC_DEF = 254, CGT_DEF = 12, CWT_DEF = 9600, BGT_DEF = 22, BWT_DEF = 9600, EGT_DEF = 0;

// x86-64 double -> unsigned int: cvttsd2si into a 64-bit register, low 32 bits kept (out of range and NaN give 0)
ISO_HD int64_t iso_cvt64(double x)
{
   return (x > -9223372036854775808.0 && x < 9223372036854775808.0) ? (int64_t) x : (int64_t) 0x8000000000000000ull;
}
ISO_HD uint32_t iso_d2u(double x)
{
   return (uint32_t) (uint64_t) iso_cvt64(x);
}
// x86-64 double -> unsigned long: values from 2^63 up are converted after subtracting 2^63
ISO_HD uint64_t iso_d2ul(double x)
{
   if (x >= 9223372036854775808.0)
      return (uint64_t) iso_cvt64(x - 9223372036854775808.0) ^ 0x8000000000000000ull;
   return (uint64_t) iso_cvt64(x);
}

enum : uint32_t { MODE_RESET = 0, MODE_SYNC = 1, MODE_TS = 2, MODE_ATR = 3 };
enum : uint32_t { LOOP_DETECT = 0, LOOP_T0 = 1, LOOP_T1 = 2, LOOP_TX = 3 };
enum : int { SYM_INCOMPLETE = -1, SYM_TIMEOUT = 0, SYM_FULL = 1, SYM_POWER_LOW = 8, SYM_RESET_LOW = 9 };
enum : int { RES_INVALID = -1, RES_SUCCESS = 0, RES_FAILED = 1 };
enum : uint32_t { DIRECT = 1, INVERSE = 2 };

// the compared part of the state: every field is 4 or 8 bytes and 8-byte fields come in aligned pairs, so there is no
// padding and the state compares word by word
struct IsoState
{
   // IsoModulationStatus (IsoTech.h:136-152) without its clock fields
   uint32_t searchModeState, searchStartTime, searchEndTime, searchSyncTime, syncStartTime, syncEndTime;
   // IsoProtocolStatus (Iso7816.cpp:128-201)
   uint32_t protocolType, errorCodeType, symbolConvention, protocolParametersChange;
   double clockFrequency, elementaryTimeUnit, elementaryTime, elementaryHalfTime;
   uint32_t frequencyFactorIndex, frequencyFactor, baudRateFactorIndex, baudRateFactor;
   uint32_t extraGuardTimeUnits, extraGuardTime, characterGuardTimeUnits, characterGuardTime;
   uint32_t characterWaitingTimeUnits, characterWaitingTime, blockGuardTimeUnits, blockGuardTime;
   uint32_t blockWaitingTimeUnits, blockWaitingTime, maximumInformationSize, locked;
   // IsoSymbolStatus (IsoTech.h:157-164)
   uint32_t symValue, symData;
   uint64_t symSync, symStart, symEnd;
   // IsoCharacterStatus (IsoTech.h:169-177)
   uint32_t chrBits, chrData, chrFlags, chrParity;
   uint64_t chrStart, chrEnd;
   // IsoFrameStatus (IsoTech.h:182-196) without its bytes
   uint32_t frameType, symbolRate, frameStart, frameEnd, frameFlags, guardTime, waitingTime, frameSize;
   // which loop of IsoDecoder::nextFrames runs (detect or one of decodeStreamT0 / T1 / Tx), frames emitted so far
   uint32_t loop, frames;
};

struct IsoMachine
{
   IsoState s;
   // clock fields of the modulation status
   uint32_t clockEdgeTime, clockCounter;
   double clockFrequencyMod;
   // decoder
   uint32_t sampleRate, streamTime;
   double sampleTime;
   uint8_t frameData[FRAME_BYTES];
};

// one decoded frame, as lab::RawFrame holds it
struct IsoFrameOut
{
   uint32_t techType, frameType, frameFlags, framePhase, frameRate, length;
   uint64_t sampleStart, sampleEnd;
   double timeStart, timeEnd, dateTime;
   const uint8_t *data; // `length` bytes, at most FRAME_BYTES stored
};

ISO_HD bool state_equal(const IsoState &a, const IsoState &b)
{
   const uint32_t *x = (const uint32_t *) &a, *y = (const uint32_t *) &b;
   for (unsigned i = 0; i < sizeof(IsoState) / 4; i++)
      if (x[i] != y[i])
         return false;
   return true;
}

template <class Sink>
struct IsoStep
{
   IsoMachine &m;
   Sink &sink;
   uint32_t clock, f;

   ISO_HD uint32_t byte(uint32_t i) const
   {
      return i < m.s.frameSize && i < FRAME_BYTES ? m.frameData[i] : 0u;
   }

   // Iso7816.cpp:1378-1435
   ISO_HD void updateProtocol(const double clockFrequency, const uint32_t fi, const uint32_t di)
   {
      IsoState &s = m.s;
      double sampleRate = m.sampleRate;
      double frequencyFactor = fi_table(fi);
      double baudRateFactor = di_table(di);
      s.clockFrequency = clockFrequency;
      s.frequencyFactor = (uint32_t) (int32_t) frequencyFactor;
      s.baudRateFactor = (uint32_t) (int32_t) baudRateFactor;
      s.frequencyFactorIndex = fi;
      s.baudRateFactorIndex = di;
      if (clockFrequency > 0)
      {
         s.elementaryTime = sampleRate * frequencyFactor / (baudRateFactor * clockFrequency);
         s.elementaryHalfTime = s.elementaryTime / 2;
         s.elementaryTimeUnit = s.elementaryTime * m.sampleTime;
         s.characterGuardTime = iso_d2u(round(s.elementaryTime * s.characterGuardTimeUnits));
         s.characterWaitingTime = iso_d2u(round(s.elementaryTime * s.characterWaitingTimeUnits));
         s.blockGuardTime = iso_d2u(round(s.elementaryTime * s.blockGuardTimeUnits));
         s.blockWaitingTime = iso_d2u(round(s.elementaryTime * s.blockWaitingTimeUnits));
         s.extraGuardTime = iso_d2u(round(s.elementaryTime * s.extraGuardTimeUnits));
         s.guardTime = iso_d2u(s.characterGuardTime - 0.5 * s.elementaryTime);
         s.waitingTime = iso_d2u(s.characterWaitingTime + 0.5 * s.elementaryTime);
         s.symbolRate = iso_d2u(1.0f / s.elementaryTimeUnit);
      }
      else
      {
         s.elementaryTime = 0;
         s.elementaryHalfTime = 0;
         s.elementaryTimeUnit = 0;
         s.characterGuardTime = 0;
         s.characterWaitingTime = 0;
         s.blockGuardTime = 0;
         s.blockWaitingTime = 0;
         s.extraGuardTime = 0;
      }
      s.protocolParametersChange = 0;
   }

   // Iso7816.cpp:1330-1373
   ISO_HD void resetModulation()
   {
      const uint32_t loop = m.s.loop, frames = m.s.frames;
      m.s = IsoState {};
      m.s.loop = loop;
      m.s.frames = frames;
      m.clockEdgeTime = 0;
      m.clockCounter = 0;
      m.clockFrequencyMod = 0;
      m.s.maximumInformationSize = IFSC_DEF;
      m.s.characterGuardTimeUnits = CGT_DEF;
      m.s.characterWaitingTimeUnits = CWT_DEF;
      m.s.extraGuardTimeUnits = EGT_DEF;
      m.s.blockGuardTimeUnits = BGT_DEF;
      m.s.blockWaitingTimeUnits = BWT_DEF;
      updateProtocol(0, FI_DEF, DI_DEF);
      m.s.frameType = ATR_FRAME;
      m.s.guardTime = m.s.characterGuardTime;
      m.s.waitingTime = m.s.characterWaitingTime;
   }

   ISO_HD void clearModulation() // modulationStatus = {}
   {
      m.s.searchModeState = m.s.searchStartTime = m.s.searchEndTime = m.s.searchSyncTime = m.s.syncStartTime = m.s.syncEndTime = 0;
      m.clockEdgeTime = 0;
      m.clockCounter = 0;
      m.clockFrequencyMod = 0;
   }

   ISO_HD void clearCharacter()
   {
      m.s.chrBits = m.s.chrData = m.s.chrFlags = m.s.chrParity = 0;
      m.s.chrStart = m.s.chrEnd = 0;
   }

   ISO_HD void appendByte(uint32_t v)
   {
      if (m.s.frameSize < FRAME_BYTES)
         m.frameData[m.s.frameSize] = (uint8_t) v;
      m.s.frameSize++;
   }

   ISO_HD void emitLine(uint32_t type)
   {
      IsoFrameOut o = {};
      o.techType = TECH_ISO_ANY;
      o.frameType = type;
      o.framePhase = ISO_ANY_PHASE;
      o.sampleStart = clock;
      o.sampleEnd = clock;
      o.timeStart = (double) clock / (double) m.sampleRate;
      o.timeEnd = (double) clock / (double) m.sampleRate;
      o.dateTime = m.streamTime + o.timeStart;
      o.data = m.frameData;
      m.s.frames++;
      sink.frame(o);
   }

   // Iso7816.cpp:271-307
   ISO_HD void detectLines()
   {
      if (f & F_VCC_CHG)
         emitLine((f & F_VCC_NEG) ? VCC_LOW : VCC_HIGH);
      if (f & F_RST_CHG)
         emitLine((f & F_RST_NEG) ? RST_LOW : RST_HIGH);
   }

   // Iso7816.cpp:312-344
   ISO_HD void detectClock()
   {
      if (f & F_CLK_FALL)
      {
         if (++m.clockCounter == 10)
         {
            double clockValue = (double) (m.sampleRate * m.clockCounter) / (double) (clock - m.clockEdgeTime);
            double clockDrift = fabs(clockValue - m.clockFrequencyMod) / m.clockFrequencyMod;
            m.clockCounter = 0;
            m.clockEdgeTime = clock;
            m.clockFrequencyMod = clockValue;
            if (clockDrift < 0.05 && m.s.clockFrequency > 0)
            {
               clockDrift = fabs(m.clockFrequencyMod - m.s.clockFrequency) / m.s.clockFrequency;
               if (clockDrift > 0.05)
                  updateProtocol(m.clockFrequencyMod, m.s.frequencyFactorIndex, m.s.baudRateFactorIndex);
            }
         }
      }
   }

   // Iso7816.cpp:349-362
   ISO_HD bool detectReset()
   {
      if ((f & F_VCC_HIGH) && (f & F_RST_POS) && clock > 2)
      {
         m.s.searchModeState = MODE_SYNC;
         m.s.searchStartTime = clock;
      }
      return false;
   }

   // Iso7816.cpp:367-437
   ISO_HD bool detectSync()
   {
      IsoState &s = m.s;
      if ((f & F_VCC_NEG) || (f & F_RST_NEG))
      {
         resetModulation();
         return false;
      }
      if (clock < s.searchStartTime)
         return false;
      if (!s.syncStartTime)
      {
         if (f & F_IO_NEG)
            s.syncStartTime = clock;
         return false;
      }
      if (!s.syncEndTime)
      {
         if (f & F_IO_NEG)
            s.syncEndTime = clock;
         return false;
      }
      s.chrStart = s.syncStartTime;
      s.chrEnd = 0;
      s.chrBits = 3;
      s.chrData = 3;
      s.chrFlags = 0;
      s.chrParity = 0;
      s.symbolConvention = DIRECT;
      const double etuSamples = (s.syncEndTime - s.syncStartTime) / 3.0;
      const double clockFrequency = (m.sampleRate / etuSamples) * (fi_table(FI_DEF) / di_table(DI_DEF));
      updateProtocol(clockFrequency, FI_DEF, DI_DEF);
      s.guardTime = iso_d2u(s.characterGuardTime - 0.5 * s.elementaryTime);
      s.waitingTime = iso_d2u(s.characterWaitingTime + 0.5 * s.elementaryTime);
      s.searchModeState = MODE_TS;
      s.searchSyncTime = iso_d2u((double) s.chrStart + s.elementaryTime * 3 + s.elementaryHalfTime);
      s.searchStartTime = 0;
      s.searchEndTime = 0;
      return false;
   }

   // Iso7816.cpp:442-489
   ISO_HD bool detectTS()
   {
      IsoState &s = m.s;
      if (decodeCharacter() == SYM_FULL)
      {
         switch (s.chrData)
         {
            case 0x3B:
               s.symbolConvention = DIRECT;
               break;
            case 0x03:
               s.chrData = 0x3F;
               s.chrParity = !s.chrParity;
               s.symbolConvention = INVERSE;
               break;
            default:
               resetModulation();
               return false;
         }
         s.searchModeState = MODE_ATR;
         s.frameType = ATR_FRAME;
         s.frameStart = (uint32_t) s.chrStart;
         s.frameEnd = (uint32_t) s.chrEnd;
         s.frameFlags = 0;
         s.frameSize = 0;
         appendByte(s.chrData);
         s.symbolRate = iso_d2u(1.0f / s.elementaryTimeUnit);
         clearCharacter();
      }
      return false;
   }

   // RawFrame of an ATR / T=0 / T=1 frame: date_time is set while time_start is still 0 (Iso7816.cpp:529-530)
   ISO_HD void buildFrame(IsoFrameOut &o, uint32_t type)
   {
      const IsoState &s = m.s;
      o = IsoFrameOut {};
      o.techType = TECH_ISO7816;
      o.frameType = type;
      o.frameRate = s.symbolRate;
      o.sampleStart = s.frameStart;
      o.sampleEnd = s.frameEnd;
      o.frameFlags = s.frameFlags | (s.frameSize > FRAME_BYTES ? FLAG_TRUNCATED : 0u);
      o.dateTime = m.streamTime + 0.0;
      o.timeStart = (double) s.frameStart / (double) m.sampleRate;
      o.timeEnd = (double) s.frameEnd / (double) m.sampleRate;
      o.length = s.frameSize;
      o.data = m.frameData;
   }

   ISO_HD void emit(IsoFrameOut &o)
   {
      m.s.frames++;
      sink.frame(o);
   }

   // Iso7816.cpp:494-559
   ISO_HD bool detectATR()
   {
      IsoState &s = m.s;
      int result = RES_INVALID;
      const int c = decodeCharacter();
      if (c == SYM_FULL)
      {
         s.frameEnd = (uint32_t) s.chrEnd;
         s.frameFlags |= s.chrFlags;
         appendByte(s.chrData);
         clearCharacter();
      }
      if (c == SYM_FULL || c == SYM_TIMEOUT)
      {
         if ((result = isATR()) == RES_SUCCESS)
         {
            IsoFrameOut o;
            buildFrame(o, ATR_FRAME);
            process(o);
            emit(o);
            s.locked = 1;
            return true;
         }
      }
      if (result == RES_FAILED)
         resetModulation();
      return false;
   }

   // Iso7816.cpp:705-754
   ISO_HD bool decodeFrameT0()
   {
      IsoState &s = m.s;
      int result;
      if ((result = decodeCharacter()) == SYM_FULL)
      {
         if (!s.frameStart)
            s.frameStart = (uint32_t) s.chrStart;
         s.frameEnd = (uint32_t) s.chrEnd;
         s.frameFlags |= s.chrFlags;
         appendByte(s.chrData);
         clearCharacter();
         if (isPPS() == RES_SUCCESS)
         {
            s.frameType = s.protocolParametersChange ? RESPONSE_FRAME : REQUEST_FRAME;
            return true;
         }
         if (isTPDU() == RES_SUCCESS)
         {
            s.frameType = EXCHANGE_FRAME;
            return true;
         }
         else
            s.searchEndTime = 0;
         if (s.frameSize == s.maximumInformationSize)
            return true;
         return false;
      }
      return result == SYM_TIMEOUT;
   }

   // Iso7816.cpp:759-796
   ISO_HD bool decodeFrameT1()
   {
      IsoState &s = m.s;
      int result;
      if ((result = decodeCharacter()) == SYM_FULL)
      {
         if (!s.frameStart)
            s.frameStart = (uint32_t) s.chrStart;
         s.frameEnd = (uint32_t) s.chrEnd;
         s.frameFlags |= s.chrFlags;
         appendByte(s.chrData);
         clearCharacter();
         if (isPPS() == RES_SUCCESS)
            return true;
         if (isBlock() == RES_SUCCESS)
            return true;
         if (s.frameSize >= s.maximumInformationSize + 3 + (s.errorCodeType == 0 ? 1u : 2u))
            return true;
         return false;
      }
      return result == SYM_TIMEOUT;
   }

   // one iteration of decodeStreamT0 / T1 (Iso7816.cpp:588-687): true when the stream function returns
   ISO_HD bool decodeStream(bool t1)
   {
      IsoState &s = m.s;
      if (t1 ? decodeFrameT1() : decodeFrameT0())
      {
         if (s.frameSize == 0)
         {
            const uint32_t loop = s.loop, frames = s.frames, locked = s.locked;
            // frameStatus = {.frameType = IsoExchangeFrame}; modulationStatus = {}; characterStatus = {}
            s.frameType = EXCHANGE_FRAME;
            s.symbolRate = s.frameStart = s.frameEnd = s.frameFlags = s.guardTime = s.waitingTime = s.frameSize = 0;
            clearModulation();
            clearCharacter();
            s.loop = loop;
            s.frames = frames;
            s.locked = locked;
            return true;
         }
         IsoFrameOut o;
         buildFrame(o, s.frameType);
         process(o);
         emit(o);
         return true;
      }
      return false;
   }

   // Iso7816.cpp:801-887
   ISO_HD int decodeCharacter()
   {
      IsoState &s = m.s;
      switch (decodeSymbol())
      {
         case SYM_FULL:
         {
            if (s.chrBits == 0)
            {
               s.chrData = 0;
               s.chrStart = s.symStart;
            }
            else if (s.chrBits < 9)
            {
               s.chrData |= s.symbolConvention == DIRECT ? s.symData << (s.chrBits - 1) : s.symData << (8 - s.chrBits);
            }
            else if (s.chrBits == 9)
            {
               s.chrEnd = s.symEnd;
               s.chrParity = s.symData;
               s.chrFlags |= checkParity(s.chrData, s.chrParity) ? FLAG_PARITY : 0u;
            }
            if (s.chrBits >= 9)
            {
               if (s.protocolType == 0)
               {
                  if (s.chrBits == 10)
                  {
                     s.searchStartTime = (uint32_t) (s.chrStart + s.guardTime);
                     s.searchEndTime = (uint32_t) (s.chrStart + s.waitingTime);
                     s.searchSyncTime = 0;
                     if (s.symValue)
                        return SYM_FULL;
                     clearCharacter();
                     return SYM_INCOMPLETE;
                  }
               }
               else if (s.protocolType == 1)
               {
                  s.searchStartTime = (uint32_t) (s.chrStart + s.guardTime);
                  s.searchEndTime = (uint32_t) (s.chrStart + s.waitingTime);
                  s.searchSyncTime = 0;
                  return SYM_FULL;
               }
            }
            s.chrBits++;
            s.searchSyncTime = iso_d2u((double) s.chrStart + s.elementaryTime * s.chrBits + s.elementaryHalfTime);
            return SYM_INCOMPLETE;
         }
         case SYM_RESET_LOW:
            return SYM_RESET_LOW;
         case SYM_TIMEOUT:
            return SYM_TIMEOUT;
      }
      return SYM_INCOMPLETE;
   }

   // Iso7816.cpp:892-947
   ISO_HD int decodeSymbol()
   {
      IsoState &s = m.s;
      const bool dataValue = (f & F_IO_HIGH) != 0;
      if (f & F_VCC_NEG)
      {
         resetModulation();
         return SYM_POWER_LOW;
      }
      if (f & F_RST_NEG)
      {
         resetModulation();
         return SYM_RESET_LOW;
      }
      if (s.searchStartTime && clock < s.searchStartTime)
         return SYM_INCOMPLETE;
      if (s.searchEndTime && clock >= s.searchEndTime)
         return SYM_TIMEOUT;
      if (!s.searchSyncTime && (f & F_IO_NEG))
      {
         s.searchStartTime = 0;
         s.searchEndTime = 0;
         s.searchSyncTime = iso_d2u(clock + s.elementaryHalfTime);
      }
      if (!s.searchSyncTime || clock < s.searchSyncTime)
         return SYM_INCOMPLETE;
      s.symValue = dataValue;
      s.symSync = s.searchSyncTime;
      s.symStart = iso_d2ul(s.searchSyncTime - s.elementaryHalfTime);
      s.symEnd = iso_d2ul(s.searchSyncTime + s.elementaryHalfTime);
      s.symData = s.symbolConvention == DIRECT ? dataValue : !dataValue;
      return SYM_FULL;
   }

   // Iso7816.cpp:952-1023 (`o` is the frame about to be emitted; its bytes are frameData)
   ISO_HD void process(IsoFrameOut &o)
   {
      IsoState &s = m.s;
      do
      {
         if (processATR(o))
            break;
         if (processPPS(o))
            break;
         if (processTPDU(o))
            break;
         if (processBlock(o, 0x80, 0x00)) // I-block: bit 8 clear
            break;
         if (processBlock(o, 0xC0, 0x80)) // R-block
            break;
         if (processBlock(o, 0xC0, 0xC0)) // S-block
            break;
      }
      while (false);
      if (s.protocolType == 1)
      {
         if (o.frameType == REQUEST_FRAME)
            s.frameType = RESPONSE_FRAME;
         else if (o.frameType == RESPONSE_FRAME)
            s.frameType = REQUEST_FRAME;
      }
      if (s.extraGuardTimeUnits == 255)
      {
         if (s.protocolType == 0)
            s.guardTime = iso_d2u((12 - 0.5) * s.elementaryTime);
         else
            s.guardTime = iso_d2u((11 - 0.5) * s.elementaryTime);
      }
      else
         s.guardTime = iso_d2u(s.characterGuardTime - 0.5 * s.elementaryTime);
      s.waitingTime = iso_d2u(s.characterWaitingTime + 0.5 * s.elementaryTime);
      s.searchStartTime = 0;
      s.searchEndTime = 0;
      s.searchSyncTime = 0;
      s.frameStart = 0;
      s.frameEnd = 0;
      s.frameFlags = 0;
      s.frameSize = 0;
      s.symbolRate = iso_d2u(1.0f / s.elementaryTimeUnit);
   }

   // Iso7816.cpp:1028-1169; frame bytes are frameData[0 .. o.length), frameSize is cleared only after process()
   ISO_HD bool processATR(IsoFrameOut &o)
   {
      IsoState &s = m.s;
      if (o.frameType != ATR_FRAME)
         return false;
      bool updateParameters = false;
      uint32_t i = 1, n = 2, k = 1, c = 0;
      do
      {
         if (byte(i) & 0x10)
         {
            uint32_t ta = byte(n++);
            if (k == 3)
               s.maximumInformationSize = ta;
         }
         if (byte(i) & 0x20)
         {
            uint32_t tb = byte(n++);
            if (k == 3)
            {
               updateParameters = true;
               s.blockWaitingTimeUnits = 11 + bwt_table(tb >> 4);
               s.characterWaitingTimeUnits = 11 + cwt_table(tb & 0x0f);
            }
         }
         if (byte(i) & 0x40)
         {
            uint32_t tc = byte(n++);
            uint32_t dn = di_table(s.baudRateFactorIndex);
            if (k == 1)
            {
               updateParameters = true;
               s.extraGuardTimeUnits = tc;
            }
            else if (k == 2)
            {
               updateParameters = true;
               s.characterWaitingTimeUnits = tc > 0 ? tc * 960 * dn : CWT_DEF;
            }
         }
         if (!(byte(i) & 0x80))
            break;
         k++;
         i = n++;
         c |= byte(i) & 0x0f;
      }
      while (n < o.length);
      if (c)
         o.frameFlags |= !checkLrc(o.length) ? FLAG_CRC : 0u;
      if (updateParameters)
         updateProtocol(s.clockFrequency, s.frequencyFactorIndex, s.baudRateFactorIndex);
      return true;
   }

   // Iso7816.cpp:1174-1230
   ISO_HD bool processPPS(IsoFrameOut &o)
   {
      IsoState &s = m.s;
      (void) o;
      if (byte(0) != 0xFF)
         return false;
      uint32_t i = 1;
      uint32_t pps0 = byte(i++);
      if (pps0 & 0x10)
      {
         uint32_t pps1 = byte(i++);
         uint32_t fi = pps1 >> 4;
         uint32_t di = pps1 & 0x0f;
         if (s.protocolParametersChange)
         {
            s.protocolType = pps0 & 0x0f;
            s.frameType = s.protocolType == 0 ? EXCHANGE_FRAME : REQUEST_FRAME;
            updateProtocol(s.clockFrequency, fi, di);
         }
         else
            s.protocolParametersChange = 1;
      }
      return true;
   }

   // Iso7816.cpp:1235-1248
   ISO_HD bool processTPDU(IsoFrameOut &o)
   {
      if (o.frameType != EXCHANGE_FRAME)
         return false;
      if (o.length < 5 || o.length > 255)
         return false;
      if (byte(0) == 0xFF)
         return false;
      return true;
   }

   // Iso7816.cpp:1253-1325: I / R / S block by the PCB's top bits, then the LRC or CRC check
   ISO_HD bool processBlock(IsoFrameOut &o, uint32_t mask, uint32_t value)
   {
      if (o.frameType != REQUEST_FRAME && o.frameType != RESPONSE_FRAME)
         return false;
      if ((byte(1) & mask) != value)
         return false;
      if (m.s.errorCodeType == 0)
         o.frameFlags |= !checkLrc(o.length) ? FLAG_CRC : 0u;
      else if (m.s.errorCodeType == 1)
         o.frameFlags |= !checkCrc(o.length) ? FLAG_CRC : 0u;
      return true;
   }

   // Iso7816.cpp:1440-1475
   ISO_HD int isATR() const
   {
      const uint32_t size = m.s.frameSize;
      if (size < 2)
         return RES_INVALID;
      if (size > 32)
         return RES_FAILED;
      uint32_t i = 1, n = 1, c = 0;
      uint32_t hb = byte(n++) & 0x0f;
      do
      {
         if (byte(i) & 0x10) n++;
         if (byte(i) & 0x20) n++;
         if (byte(i) & 0x40) n++;
         if (!(byte(i) & 0x80))
            break;
         i = n++;
         c |= byte(i) & 0x0f;
      }
      while (n < size);
      if (size < n + hb + (c ? 1 : 0))
         return RES_INVALID;
      return RES_SUCCESS;
   }

   // Iso7816.cpp:1480-1506
   ISO_HD int isPPS() const
   {
      const uint32_t size = m.s.frameSize;
      if (size < 3 || size > 6)
         return RES_INVALID;
      if (byte(0) != 0xFF)
         return RES_INVALID;
      uint32_t n = 3, ck = 0;
      if (byte(1) & 0x10) n++;
      if (byte(1) & 0x20) n++;
      if (byte(1) & 0x40) n++;
      if (size != n)
         return RES_INVALID;
      for (uint32_t i = 0; i < size; i++)
         ck ^= byte(i);
      return !ck ? RES_SUCCESS : RES_FAILED;
   }

   // Iso7816.cpp:1511-1544
   ISO_HD int isTPDU() const
   {
      const uint32_t size = m.s.frameSize;
      if (size < 5)
         return RES_INVALID;
      if (byte(0) == 0xFF)
         return RES_INVALID;
      if ((byte(1) & 0xf0) == 0x60 || (byte(1) & 0xf0) == 0x90)
         return RES_INVALID;
      for (uint32_t offset = 5; offset < size; offset++)
      {
         if (byte(offset) == 0x60)
            continue;
         if ((byte(offset) & 0xF0) == 0x60 || (byte(offset) & 0xF0) == 0x90)
            return size == offset + 2 ? RES_SUCCESS : RES_INVALID;
         if (byte(offset) == byte(1))
            offset += byte(4);
         else if (byte(offset) == (byte(1) ^ 0xFF))
            offset++;
      }
      return RES_INVALID;
   }

   // Iso7816.cpp:1549-1565
   ISO_HD int isBlock() const
   {
      const uint32_t size = m.s.frameSize;
      const uint32_t epilogue = m.s.errorCodeType == 0 ? 1 : 2;
      if (size < 3 + epilogue)
         return RES_INVALID;
      if (byte(0) == 0xFF)
         return RES_INVALID;
      if (size != 3 + byte(2) + epilogue)
         return RES_INVALID;
      return RES_SUCCESS;
   }

   ISO_HD static bool checkParity(uint32_t value, uint32_t parity)
   {
      for (uint32_t i = 0; i < 8; i++)
         if ((value & (1u << i)) != 0)
            parity = parity ^ 1;
      return parity;
   }

   ISO_HD bool checkLrc(uint32_t size) const
   {
      uint32_t rc = 0;
      for (uint32_t i = 1; i < size; i++)
         rc ^= byte(i);
      return !rc;
   }

   // ISO/IEC 13239 CRC (lab-data Crc.cpp:96-113, reflected CCITT, init 0xFFFF), inverted
   ISO_HD bool checkCrc(uint32_t size) const
   {
      if (size < 3)
         return false;
      uint32_t crc = 0xFFFF;
      for (uint32_t i = 0; i + 2 < size; i++)
      {
         crc ^= byte(i);
         for (int b = 0; b < 8; b++)
            crc = (crc & 1) ? (crc >> 1) ^ 0x8408 : crc >> 1;
      }
      crc = ~crc & 0xFFFF;
      const uint32_t res = byte(size - 2) | byte(size - 1) << 8;
      return res == crc;
   }

   // Iso7816.cpp:244-266
   ISO_HD bool detect()
   {
      detectLines();
      detectClock();
      switch (m.s.searchModeState)
      {
         case MODE_RESET:
            return detectReset();
         case MODE_SYNC:
            return detectSync();
         case MODE_TS:
            return detectTS();
         case MODE_ATR:
            return detectATR();
      }
      return false;
   }

   ISO_HD uint32_t decodeLoop() const
   {
      return m.s.protocolType == 0 ? LOOP_T0 : m.s.protocolType == 1 ? LOOP_T1 : LOOP_TX;
   }

   // one sample of IsoDecoder::Impl::nextFrames (IsoDecoder.cpp:184-208) in whichever loop runs
   ISO_HD void run()
   {
      switch (m.s.loop)
      {
         case LOOP_DETECT:
            if (detect())
               m.s.loop = decodeLoop();
            break;
         case LOOP_T0:
         case LOOP_T1:
            detectLines();
            detectClock();
            if (decodeStream(m.s.loop == LOOP_T1))
               m.s.loop = m.s.locked ? decodeLoop() : LOOP_DETECT;
            break;
         default:
            detectLines();
            detectClock();
            break;
      }
   }
};

// IsoDecoder::Impl::initialize (IsoDecoder.cpp:123-156) at the first buffer of a capture
ISO_HD void iso_init(IsoMachine &m, uint32_t sampleRate, uint32_t streamTime)
{
   struct NoSink
   {
      ISO_HD void frame(const IsoFrameOut &) {}
   } none;
   m.s = IsoState {};
   m.sampleRate = sampleRate;
   m.streamTime = streamTime;
   m.sampleTime = 1.0 / (double) sampleRate;
   IsoStep<NoSink> st {m, none, 0, 0};
   st.resetModulation();
   m.s.loop = LOOP_DETECT;
}

// where iso_walk() stops at the end of one buffer of a capture and picks up at the next: the walk's own locals.  CLK falling
// edges passed since the last step are in clockCounter already (none of them was the 10th, or the walk would have stepped
// there), so only these two are left
struct IsoCarry
{
   uint64_t wake;   // next sample where a step without edges may act (absolute); ~0 when no timer is pending
   uint32_t levels; // F_IO_HIGH / F_VCC_HIGH of the last sample (the sample before the first is 0)
   uint32_t unused;
};

ISO_HD IsoCarry iso_carry_init()
{
   return IsoCarry {~0ull, 0, 0};
}

// a decoder between two buffers of one capture
struct IsoStreamState
{
   IsoMachine m;
   IsoCarry c;
};

// the start of a later nextFrames() call at the same sample rate (IsoDecoder.cpp:184-200): its loop is chosen afresh --
// detect unless an ATR locked the protocol (`if (!decoder.bitrate)`), then decode()'s switch on the protocol type -- so a
// buffer that ends inside decodeStreamT0 after a reset cleared the protocol (IsoState::loop) resumes in detect.  A changed
// loop is a changed state: the first sample of the buffer is stepped.
ISO_HD void iso_resume(IsoMachine &m, IsoCarry &c, uint32_t base)
{
   const uint32_t p = m.s.protocolType;
   const uint32_t loop = m.s.locked ? (p == 0 ? LOOP_T0 : p == 1 ? LOOP_T1 : LOOP_TX) : LOOP_DETECT;
   if (loop != m.s.loop)
   {
      m.s.loop = loop;
      c.wake = base < c.wake ? base : c.wake;
   }
}

// a buffer at another sample rate (IsoDecoder.cpp:172-178 -> initialize(), :123-156): the clock restarts at 0 and
// Iso7816::initialize's resetModulation clears every status the machine holds; the last sample survives (IsoTech.cpp:43
// never reloads it), and with it the levels
ISO_HD void iso_restart(IsoMachine &m, IsoCarry &c, uint32_t sampleRate, uint32_t streamTime)
{
   iso_init(m, sampleRate, streamTime);
   c.wake = ~0ull;
}

// earliest timer after `t` (NONE when there is none)
ISO_HD uint64_t next_timer(const IsoState &s, uint32_t t)
{
   uint64_t w = ~0ull;
   if (s.searchStartTime > t && s.searchStartTime < w) w = s.searchStartTime;
   if (s.searchEndTime > t && s.searchEndTime < w) w = s.searchEndTime;
   if (s.searchSyncTime > t && s.searchSyncTime < w) w = s.searchSyncTime;
   return w;
}

/*
 * Walk one capture, or one buffer of it, up to the sample `end` (absolute: a buffer's first sample is the number of samples
 * before it since the last (re)start).  Ev supplies the events in sample order, at absolute samples:
 *   line_peek()        sample of the next line event (IO / RST / VCC edge) or NONE;  line_pop() its flags
 *   clk_nth(k)         sample of the k-th (from 0) CLK falling edge not yet consumed, or NONE;  clk_pop() consumes one,
 *                      clk_skip(k) consumes k
 * CLK falling edges are consumed as the walk passes them.  `c` holds the walk's state from the end of the previous buffer
 * and receives it at the end of this one.
 */
template <class Ev, class Sink>
ISO_HD void iso_walk(IsoMachine &m, IsoCarry &c, Ev &ev, uint32_t end, Sink &sink)
{
   uint32_t levels = c.levels; // IO / VCC above 0 since the last line event
   uint64_t wake = c.wake;     // next sample where a step without edges may act
   while (true)
   {
      const uint64_t tl = ev.line_peek();
      const uint64_t tc = ev.clk_nth(9 - m.clockCounter);
      uint64_t t = tl < tc ? tl : tc;
      t = wake < t ? wake : t;
      if (t >= end)
         break;
#ifdef __CUDA_ARCH__
      // on the device the walk runs on a whole warp, every lane with the same state: clock measurements that only update
      // the clock fields (no line event, no timer and no protocol update before them) are evaluated 32 at a time, lane j
      // taking the j-th measurement from here, in detectClock's arithmetic
      if (t == tc && tc != tl && tc != wake)
      {
         const uint32_t lane = threadIdx.x & 31;
         const uint64_t tj = ev.clk_nth(9 - m.clockCounter + 10 * lane);
         const uint32_t up = __shfl_up_sync(~0u, (uint32_t) tj, 1);
         const uint32_t prev = lane ? up : m.clockEdgeTime;
         const double v = (double) (m.sampleRate * 10u) / (double) ((uint32_t) tj - prev);
         const double vup = __shfl_up_sync(~0u, v, 1);
         const double vprev = lane ? vup : m.clockFrequencyMod;
         const double P = m.s.clockFrequency;
         const bool acts = fabs(v - vprev) / vprev < 0.05 && P > 0 && fabs(v - P) / P > 0.05;
         const uint64_t limit = tl < wake ? tl : wake;
         const uint32_t stop = __ballot_sync(~0u, acts || tj >= limit || tj >= end);
         const uint32_t take = stop ? __ffs(stop) - 1 : 32;
         if (take > 0)
         {
            ev.clk_skip(10 - m.clockCounter + 10 * (take - 1));
            m.clockCounter = 0;
            m.clockEdgeTime = __shfl_sync(~0u, (uint32_t) tj, take - 1);
            m.clockFrequencyMod = __shfl_sync(~0u, v, take - 1);
            continue;
         }
      }
#endif
      // CLK falling edges before t only count: none of them is the 10th
      while (ev.clk_nth(0) < t)
      {
         ev.clk_pop();
         m.clockCounter++;
      }
      uint32_t f = levels;
      if (tl == t)
      {
         f = ev.line_pop();
         levels = f & F_LEVELS;
      }
      if (ev.clk_nth(0) == t)
      {
         ev.clk_pop();
         f |= F_CLK_FALL;
      }
      const IsoState before = m.s;
      IsoStep<Sink> st {m, sink, (uint32_t) t, f};
      st.run();
      wake = state_equal(before, m.s) ? next_timer(m.s, (uint32_t) t) : t + 1;
   }
   // CLK falling edges between the last step and the end only count
   while (ev.clk_nth(0) < end)
   {
      ev.clk_pop();
      m.clockCounter++;
   }
   c.levels = levels;
   c.wake = wake;
}

// a whole capture from its first sample
template <class Ev, class Sink>
ISO_HD void iso_walk(IsoMachine &m, Ev &ev, uint32_t n, Sink &sink)
{
   IsoCarry c = iso_carry_init();
   iso_walk(m, c, ev, n, sink);
}

} // namespace iso7816

#endif
