/*
 * nfc_spectrum.cuh -- the reference's FFT spectrum of IQ (lab::FourierProcessTask::process, FourierProcessTask.cpp:223-352)
 * at every hop of every stream of a batch.
 *
 * One spectrum frame of a buffer that starts at sample b (sample rate fs):
 *   decimation  d = fs / 625000 in unsigned division                                           (:239, bandwidth :49)
 *   selection   window position k takes sample b + 4 d (k / 4) + k % 4: runs of 4 consecutive samples, one run every
 *               4 d samples.  This is what the x86 build's SSE2 loop (:250-263, enabled by lab-tasks/CMakeLists.txt:17-19)
 *               reads: 8 floats from data + i * d with i counting floats.  It is the reference's behaviour, not a
 *               uniform decimation (its scalar branch, :266-272, would take runs of 2).
 *   window      w[k] = float(pow(sin(float(M_PI k / 1024)), 2)), the default Hamming case (:87, :126-127), one float
 *               multiply on I and on Q
 *   transform   1024-point complex forward FFT, unnormalised (mufft MUFFT_FORWARD, :96, :276)
 *   magnitude   sqrt(re * re + im * im): multiply, multiply, add, IEEE sqrt (:280-329)
 *   bin order   negative frequencies first: mag[512..1023], mag[0..511] (:345)
 *
 * The FFT is a radix-8 x 8 x 8 x 2 Stockham transform (natural order in, natural order out).  The arithmetic -- selection,
 * window, butterflies, twiddle products, magnitude -- is __host__ __device__ code with a fixed operation order; the library
 * is built with -fmad=false and the host build (tests/native/spectrum_host.cpp) with -ffp-contract=off, so both give the
 * same bits.  Twiddles and window are computed on the host (spectrum_tables) and uploaded: device sinf / cos differ from
 * glibc in the last bits.
 *
 * Device layout: one CTA of 128 threads per frame, grid-striding over the (stream, frame) pairs of a launch.  Thread j
 * gathers window positions j + 128 r (r = 0..7), so four neighbouring threads read one run of 4 samples: one 32-byte
 * sector of float2 IQ, 16 bytes of int16 IQ.  The first radix-8 pass runs on those registers, the two further radix-8
 * passes exchange through a padded shared-memory frame, and the radix-2 pass writes the shifted magnitudes to global
 * memory, coalesced.
 */
#ifndef NFCB200_SPECTRUM_CUH
#define NFCB200_SPECTRUM_CUH

#include <stdint.h>

#include <cmath>

#if defined(__CUDACC__)
#define SPEC_HD __host__ __device__ __forceinline__
#else
#define SPEC_HD inline
#endif

namespace nfcb200 {

// SPEC_BLOCKS_PER_SM: resident CTAs the launch bound asks for (80 registers, no spills; 8 would spill)
enum { SPEC_LEN = 1024, SPEC_BANDWIDTH = 625000, SPEC_THREADS = 128, SPEC_BLOCKS_PER_SM = 6 };

struct SpecCx
{
   float x, y;
};

// ---------------------------------------------------------------------------------------------------------------------
// geometry (host)
// ---------------------------------------------------------------------------------------------------------------------

// decimation (:239) and frames of a stream: frame f covers samples [f * hop, f * hop + span), span = 1024 d (:242)
inline uint32_t spectrum_decimation(uint32_t sample_rate)
{
   return sample_rate / (uint32_t) SPEC_BANDWIDTH;
}

inline uint64_t spectrum_frames(uint64_t n_samples, uint32_t decimation, uint64_t hop)
{
   const uint64_t span = (uint64_t) SPEC_LEN * decimation;
   return n_samples < span ? 0 : (n_samples - span) / hop + 1;
}

// twiddles exp(-2 pi i k / 1024) in double rounded to float, and the window exactly as FourierProcessTask::start computes it
// (:126-127; std::sin of a float is glibc sinf, std::pow of a float and an int is the double pow)
inline void spectrum_tables(SpecCx *tw, float *win)
{
   for (int k = 0; k < SPEC_LEN; k++)
   {
      const double a = -2.0 * M_PI * k / SPEC_LEN;
      tw[k].x = (float) std::cos(a);
      tw[k].y = (float) std::sin(a);
   }
   for (int n = 0; n < SPEC_LEN; ++n)
      win[n] = static_cast<float>(std::pow(std::sin(static_cast<float>(M_PI * n / SPEC_LEN)), 2));
}

// ---------------------------------------------------------------------------------------------------------------------
// arithmetic shared by the kernel and the host build
// ---------------------------------------------------------------------------------------------------------------------

// offset of window position k from the frame's first sample (the SSE2 selection, see the top of this file)
SPEC_HD uint64_t spec_offset(uint32_t k, uint32_t decimation)
{
   return (uint64_t) 4 * decimation * (k >> 2) + (k & 3);
}

// one IQ sample times the window; int16 IQ enters as s / 32768.f (RecordDevice.cpp:281-311)
SPEC_HD SpecCx spec_windowed(float I, float Q, float w)
{
   return SpecCx{I * w, Q * w};
}

SPEC_HD SpecCx spec_windowed_s16(short I, short Q, float w)
{
   return spec_windowed((float) I / 32768.0f, (float) Q / 32768.0f, w);
}

SPEC_HD SpecCx cx_add(SpecCx a, SpecCx b)
{
   return SpecCx{a.x + b.x, a.y + b.y};
}

SPEC_HD SpecCx cx_sub(SpecCx a, SpecCx b)
{
   return SpecCx{a.x - b.x, a.y - b.y};
}

SPEC_HD SpecCx cx_mul(SpecCx a, SpecCx w)
{
   return SpecCx{a.x * w.x - a.y * w.y, a.x * w.y + a.y * w.x};
}

// a * (-i)
SPEC_HD SpecCx cx_mul_mi(SpecCx a)
{
   return SpecCx{a.y, -a.x};
}

SPEC_HD void bfly2(SpecCx &a, SpecCx &b)
{
   const SpecCx t = a;
   a = cx_add(t, b);
   b = cx_sub(t, b);
}

// forward DFT of 4 points in place, natural order out
SPEC_HD void dft4(SpecCx &v0, SpecCx &v1, SpecCx &v2, SpecCx &v3)
{
   bfly2(v0, v2);
   bfly2(v1, v3);
   v3 = cx_mul_mi(v3);
   bfly2(v0, v1);
   bfly2(v2, v3);
   const SpecCx t = v1; // (v0, v1, v2, v3) now hold X0, X2, X1, X3
   v1 = v2;
   v2 = t;
}

// forward DFT of 8 points in place, natural order out (one decimation-in-frequency step, then two DFT-4)
SPEC_HD void dft8(SpecCx *v)
{
   const float r = 0.70710678118654752440f;
   for (int k = 0; k < 4; k++)
      bfly2(v[k], v[k + 4]);
   v[5] = SpecCx{(v[5].x + v[5].y) * r, (v[5].y - v[5].x) * r}; // W8^1 = (1 - i) / sqrt 2
   v[6] = cx_mul_mi(v[6]);                                      // W8^2 = -i
   v[7] = SpecCx{(v[7].y - v[7].x) * r, -(v[7].x + v[7].y) * r}; // W8^3 = (-1 - i) / sqrt 2
   dft4(v[0], v[1], v[2], v[3]); // X0 X2 X4 X6
   dft4(v[4], v[5], v[6], v[7]); // X1 X3 X5 X7
   const SpecCx e1 = v[1], e2 = v[2], e3 = v[3], o0 = v[4], o1 = v[5], o2 = v[6];
   v[1] = o0;
   v[2] = e1;
   v[3] = o1;
   v[4] = e2;
   v[5] = o2;
   v[6] = e3;
}

// Stockham pass of radix R over butterfly j with Ns = product of the earlier radices: input r of the butterfly is element
// j + r * 1024 / R, scaled by exp(-2 pi i r (j % Ns) / (Ns R)) = tw[r (j % Ns) 1024 / (Ns R)]; output r goes to element
// (j / Ns) Ns R + j % Ns + r Ns.  The first pass (Ns = 1) has no twiddles.
SPEC_HD void spec_twiddle8(SpecCx *v, const SpecCx *tw, uint32_t j, uint32_t ns)
{
   const uint32_t step = (j % ns) * (SPEC_LEN / (ns * 8));
   for (uint32_t r = 1; r < 8; r++)
      v[r] = cx_mul(v[r], tw[r * step]);
}

SPEC_HD uint32_t spec_dest(uint32_t j, uint32_t ns, uint32_t radix, uint32_t r)
{
   return (j / ns) * ns * radix + j % ns + r * ns;
}

// the last pass (radix 2, Ns = 512) and the magnitudes: a + b w goes to bin j, a - b w to bin j + 512
SPEC_HD void spec_last(SpecCx a, SpecCx b, SpecCx w, float &mag_j, float &mag_j512)
{
   b = cx_mul(b, w);
   bfly2(a, b);
   mag_j = sqrtf(a.x * a.x + a.y * a.y);
   mag_j512 = sqrtf(b.x * b.x + b.y * b.y);
}

// ---------------------------------------------------------------------------------------------------------------------
// kernel
// ---------------------------------------------------------------------------------------------------------------------
#if defined(__CUDACC__)

// frame element i of the shared exchange buffer, padded by one float2 every 8 so that the radix-8 stores do not conflict
__device__ __forceinline__ uint32_t spec_pad(uint32_t i)
{
   return i + (i >> 3);
}

struct SpecLaunch
{
   const void *samples;   // first sample of stream `s0`
   uint64_t n_samples;    // samples per stream
   uint64_t hop;
   uint64_t n_frames;     // frames per stream
   uint64_t g0;           // first (stream, frame) pair of this launch, flattened as stream * n_frames + frame
   uint64_t count;        // pairs of this launch
   uint32_t s0;
   uint32_t decimation;
   const SpecCx *tw;      // spectrum_tables, in device memory
   const float *win;
   float *out;            // [count][1024] magnitudes of pairs g0 .. g0 + count
};

template <bool S16>
__global__ void __launch_bounds__(SPEC_THREADS, SPEC_BLOCKS_PER_SM) spectrum_kernel(const SpecLaunch L)
{
   __shared__ SpecCx sTw[SPEC_LEN];
   __shared__ float sWin[SPEC_LEN];
   __shared__ SpecCx sX[SPEC_LEN + SPEC_LEN / 8];

   const uint32_t j = threadIdx.x;
   for (uint32_t i = j; i < SPEC_LEN; i += SPEC_THREADS)
   {
      sTw[i] = L.tw[i];
      sWin[i] = L.win[i];
   }
   __syncthreads();

   for (uint64_t g = blockIdx.x; g < L.count; g += gridDim.x)
   {
      const uint64_t pair = L.g0 + g;
      const uint64_t s = pair / L.n_frames, f = pair - s * L.n_frames;
      const uint64_t base = (s - L.s0) * L.n_samples + f * L.hop;

      SpecCx v[8];
#pragma unroll
      for (uint32_t r = 0; r < 8; r++)
      {
         const uint32_t k = j + r * (SPEC_LEN / 8);
         const uint64_t idx = base + spec_offset(k, L.decimation);
         if (S16)
         {
            const short2 q = __ldg((const short2 *) L.samples + idx);
            v[r] = spec_windowed_s16(q.x, q.y, sWin[k]);
         }
         else
         {
            const float2 q = __ldg((const float2 *) L.samples + idx);
            v[r] = spec_windowed(q.x, q.y, sWin[k]);
         }
      }

      // pass 1 (Ns = 1) on the gathered registers
      dft8(v);
      __syncthreads(); // the previous frame's last pass has read sX
#pragma unroll
      for (uint32_t r = 0; r < 8; r++)
         sX[spec_pad(spec_dest(j, 1, 8, r))] = v[r];
      __syncthreads();

      // passes 2 and 3 (Ns = 8, 64)
#pragma unroll
      for (uint32_t ns = 8; ns <= 64; ns *= 8)
      {
#pragma unroll
         for (uint32_t r = 0; r < 8; r++)
            v[r] = sX[spec_pad(j + r * (SPEC_LEN / 8))];
         spec_twiddle8(v, sTw, j, ns);
         dft8(v);
         __syncthreads();
#pragma unroll
         for (uint32_t r = 0; r < 8; r++)
            sX[spec_pad(spec_dest(j, ns, 8, r))] = v[r];
         __syncthreads();
      }

      // pass 4 (radix 2, Ns = 512) and the shifted magnitudes: bin b lands at (b + 512) % 1024
      float *o = L.out + g * SPEC_LEN;
#pragma unroll
      for (uint32_t q = 0; q < 4; q++)
      {
         const uint32_t jj = j + q * SPEC_THREADS;
         float m0, m1;
         spec_last(sX[spec_pad(jj)], sX[spec_pad(jj + SPEC_LEN / 2)], sTw[jj], m0, m1);
         __stcs(o + jj + SPEC_LEN / 2, m0);
         __stcs(o + jj, m1);
      }
   }
}

#endif

} // namespace nfcb200

#endif
