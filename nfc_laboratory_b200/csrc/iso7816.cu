/*
 * iso7816.cu -- ISO 7816 contact smart-card traffic from logic captures of 4-8 channels (lab::IsoDecoder, iso_decode.cuh):
 * nfcb200_iso7816_decode_batch(_ch) for whole captures, nfcb200_iso7816_stream_* for one capture pushed buffer by buffer.
 * All run the same dense pass and the same walk.
 */
#include <numeric>

#include "host.h"
#include "iso_decode.cuh"

using namespace nfcb200;

// bytes of one channel of a logic sample
static uint32_t iso_elem_bytes(int sigtype)
{
   return sigtype == NFCB200_SIG_LOGIC_F32 ? 4 : sigtype == NFCB200_SIG_LOGIC_S16 ? 2 : 1;
}

// one dense pass over sc streams of `channels` channels at dSamples: float32 / int16 at stride 4 aligned to the sample and
// 8-bit at stride 4 aligned to 16 bytes load samples directly, everything else is staged in shared memory (iso_decode.cuh)
static void launch_edges(cudaStream_t st, int sigtype, uint32_t channels, uint32_t sc, const IsoEdgesArgs &E)
{
   const dim3 grid(E.n_tiles, sc);
   const uintptr_t at = (uintptr_t) E.samples;
   const uint32_t bps = channels * iso_elem_bytes(sigtype);
   if (channels == 4 && sigtype != NFCB200_SIG_LOGIC_U8 && at % bps == 0)
   {
      if (sigtype == NFCB200_SIG_LOGIC_S16)
         iso_edges_kernel<true><<<grid, ISO_THREADS, 0, st>>>(E);
      else
         iso_edges_kernel<false><<<grid, ISO_THREADS, 0, st>>>(E);
   }
   else if (channels == 4 && at % 16 == 0 && (sc == 1 || E.n_samples % 4 == 0))
      iso_edges_u8x4_kernel<<<grid, ISO_THREADS, 0, st>>>(E);
   else if (sigtype == NFCB200_SIG_LOGIC_F32)
      iso_edges_staged_kernel<float><<<grid, ISO_THREADS, iso_stage_bytes<float>(bps), st>>>(E, channels);
   else if (sigtype == NFCB200_SIG_LOGIC_S16)
      iso_edges_staged_kernel<int16_t><<<grid, ISO_THREADS, iso_stage_bytes<int16_t>(bps), st>>>(E, channels);
   else
      iso_edges_staged_kernel<uint8_t><<<grid, ISO_THREADS, iso_stage_bytes<uint8_t>(bps), st>>>(E, channels);
}

// the dense pass over sc streams at dSamples, again with room for a line event and a CLK falling edge at every sample
// when a tile overflows the first try's slots; E holds the slots the walk reads
static int edge_pass(cudaStream_t st, int sigtype, uint32_t channels, const void *dSamples, uint32_t sc, uint64_t n_samples, float4 last,
                     nfcb200_handle::IsoEvents &B, uint32_t *overflow, IsoEdgesArgs &E)
{
   const uint32_t nTiles = (uint32_t) ((n_samples + ISO_TILE - 1) / ISO_TILE);
   int rc;
   if ((rc = B.clkCount.reserve((uint64_t) sc * nTiles * 4)) || (rc = B.lineCount.reserve((uint64_t) sc * nTiles * 4)))
      return rc;
   E = {};
   E.samples = dSamples;
   E.n_samples = n_samples;
   E.n_tiles = nTiles;
   E.line_count = B.lineCount.as<uint32_t>();
   E.clk_count = B.clkCount.as<uint32_t>();
   E.overflow = overflow;
   E.last = last;
   for (E.line_cap = ISO_LINE_CAP, E.clk_cap = ISO_CLK_CAP;; E.line_cap = E.clk_cap = ISO_TILE)
   {
      if ((rc = B.line.reserve((uint64_t) sc * nTiles * E.line_cap * 4)) || (rc = B.clk.reserve((uint64_t) sc * nTiles * E.clk_cap * sizeof(uint16_t))))
         return rc;
      E.line = B.line.as<uint32_t>();
      E.clk = B.clk.as<uint16_t>();
      CUDA_TRY(cudaMemsetAsync(E.overflow, 0, 4, st));
      launch_edges(st, sigtype, channels, sc, E);
      CUDA_TRY(cudaGetLastError());
      uint32_t over = 0;
      CUDA_TRY(cudaMemcpyAsync(&over, E.overflow, 4, cudaMemcpyDeviceToHost, st));
      CUDA_TRY(cudaStreamSynchronize(st));
      if (!over || E.line_cap == ISO_TILE)
         return 0;
   }
}

// the walk of sc streams over the slots of E, again with a larger pool when the frames did not fit (W's decoder state is
// read from `resume` and written elsewhere, so a walk can run again); *count = frames in the pool
static int walk_pass(cudaStream_t st, const IsoEdgesArgs &E, IsoWalkArgs &W, uint32_t sc, DevBuf &pool, uint32_t &poolCap, uint32_t &count)
{
   W.n_streams = sc;
   W.n_samples = (uint32_t) E.n_samples;
   W.n_tiles = E.n_tiles;
   W.line_cap = E.line_cap;
   W.clk_cap = E.clk_cap;
   W.line = E.line;
   W.line_count = E.line_count;
   W.clk = E.clk;
   W.clk_count = E.clk_count;
   while (true)
   {
      W.pool = pool.as<nfcb200_frame>();
      W.pool_cap = poolCap;
      CUDA_TRY(cudaMemsetAsync(W.pool_count, 0, 4, st));
      if (W.resume)
         iso_walk_kernel<true><<<sc, 32, 0, st>>>(W);
      else
         iso_walk_kernel<false><<<sc, 32, 0, st>>>(W);
      CUDA_TRY(cudaGetLastError());
      CUDA_TRY(cudaMemcpyAsync(&count, W.pool_count, 4, cudaMemcpyDeviceToHost, st));
      CUDA_TRY(cudaStreamSynchronize(st));
      if (count <= poolCap)
         return 0;
      poolCap = count;
      if (int rc = pool.reserve((uint64_t) poolCap * sizeof(nfcb200_frame)))
         return rc;
   }
}

static bool is_logic(int sigtype)
{
   return sigtype == NFCB200_SIG_LOGIC_F32 || sigtype == NFCB200_SIG_LOGIC_S16 || sigtype == NFCB200_SIG_LOGIC_U8;
}

// channels outside 4-8: below 4 the reference reads channels the buffer does not have, above 8 it writes past its 8-channel
// sample (IsoTech.cpp:37-58)
static int check_channels(uint32_t channels)
{
   if (channels < 4 || channels > 8)
      return fail(NFCB200_ERR_INVALID, "%u channels: logic samples have 4 to 8", channels);
   return 0;
}

// the batch decode of both entry points; `align`: the alignment device samples must have
static int iso_batch(nfcb200_handle *h, const void *samples, int samples_on_device, int sigtype, uint32_t channels, uint32_t align, uint32_t n_streams,
                     uint64_t n_samples, uint32_t sample_rate, nfcb200_frame *out, uint64_t cap, uint64_t *n_out)
{
   if (sample_rate == 0)
      return fail(NFCB200_ERR_INVALID, "sample rate of 0");
   if (!samples || n_streams == 0 || n_samples == 0)
      return fail(NFCB200_ERR_INVALID, "empty batch");
   if (cap && !out)
      return fail(NFCB200_ERR_INVALID, "null frame buffer");
   if (n_samples >= 0xFFFFFFFFull)
      return fail(NFCB200_ERR_UNSUPPORTED, "streams of 2^32 - 1 samples or more exceed the 32-bit sample clock of the reference (IsoTech.h:221)");
   const uint64_t bs = (uint64_t) channels * iso_elem_bytes(sigtype);
   if (samples_on_device && ((uintptr_t) samples % align))
      return fail(NFCB200_ERR_INVALID, "device samples not aligned to %u bytes", align);

   CUDA_TRY(cudaSetDevice(h->device));
   cudaStream_t st = h->stream;
   auto &I = h->iso;
   int rc;

   uint32_t poolCap = (uint32_t) std::max<uint64_t>(1024, I.pool.cap / sizeof(nfcb200_frame));
   if ((rc = I.ctr.reserve(8)) || (rc = I.pool.reserve((uint64_t) poolCap * sizeof(nfcb200_frame))))
      return rc;

   uint64_t nf = 0; // frames of the groups so far
   auto group = [&](uint32_t s0, uint32_t sc, const void *dSamples) -> int {
      if ((rc = I.streamCount.reserve((uint64_t) sc * 4)) || (rc = I.first.reserve((uint64_t) sc * 8)))
         return rc;
      IsoEdgesArgs E;
      if ((rc = edge_pass(st, sigtype, channels, dSamples, sc, n_samples, make_float4(0, 0, 0, 0), I.ev, I.ctr.as<uint32_t>() + 1, E)))
         return rc;
      IsoWalkArgs W = {};
      W.stream0 = s0;
      W.sample_rate = sample_rate;
      W.stream_time = h->cfg.stream_time;
      W.pool_count = I.ctr.as<uint32_t>();
      W.stream_count = I.streamCount.as<uint32_t>();
      uint32_t count = 0;
      if ((rc = walk_pass(st, E, W, sc, I.pool, poolCap, count)))
         return rc;
      // (stream, rank in the stream): the order the reference returns each capture's frames in
      if (count && nf < cap)
      {
         std::vector<uint32_t> streamCount(sc);
         std::vector<uint64_t> first(sc);
         CUDA_TRY(cudaMemcpy(streamCount.data(), W.stream_count, (uint64_t) sc * 4, cudaMemcpyDeviceToHost));
         std::exclusive_scan(streamCount.begin(), streamCount.end(), first.begin(), (uint64_t) 0);
         if ((rc = I.ordered.reserve((uint64_t) count * sizeof(nfcb200_frame))))
            return rc;
         CUDA_TRY(cudaMemcpyAsync(I.first.ptr, first.data(), (uint64_t) sc * 8, cudaMemcpyHostToDevice, st));
         const uint32_t blocks = (uint32_t) std::min<uint64_t>((count + 7) / 8, (uint64_t) h->smCount * 16);
         iso_gather_kernel<<<blocks, 256, 0, st>>>(W.pool, count, I.first.as<uint64_t>(), s0, I.ordered.as<nfcb200_frame>());
         CUDA_TRY(cudaGetLastError());
         CUDA_TRY(cudaMemcpyAsync(out + nf, I.ordered.ptr, std::min<uint64_t>(count, cap - nf) * sizeof(nfcb200_frame), cudaMemcpyDeviceToHost, st));
         CUDA_TRY(cudaStreamSynchronize(st));
      }
      nf += count;
      return 0;
   };
   // a group's streams are the edge pass's grid.y
   if ((rc = for_each_stream_group(samples, samples_on_device, n_streams, n_samples * bs, 65535, I.in, st, group)))
      return rc;

   if (n_out)
      *n_out = nf;
   if (nf > cap)
      return fail(NFCB200_ERR_CAPACITY, "%llu frames decoded but room for %llu only", (unsigned long long) nf, (unsigned long long) cap);
   return 0;
}

extern "C" int nfcb200_iso7816_decode_batch(nfcb200_handle *h, const void *samples, int samples_on_device, int sigtype, uint32_t n_streams,
                                            uint64_t n_samples, uint32_t sample_rate, nfcb200_frame *out, uint64_t cap, uint64_t *n_out)
{
   if (!h)
      return fail(NFCB200_ERR_INVALID, "null handle");
   if (n_out)
      *n_out = 0;
   if (sigtype != NFCB200_SIG_LOGIC_F32 && sigtype != NFCB200_SIG_LOGIC_S16)
      return fail(NFCB200_ERR_INVALID, "signal type %d is not a 4-channel logic format", sigtype);
   return iso_batch(h, samples, samples_on_device, sigtype, 4, sigtype == NFCB200_SIG_LOGIC_S16 ? 8 : 16, n_streams, n_samples, sample_rate, out, cap,
                    n_out);
}

extern "C" int nfcb200_iso7816_decode_batch_ch(nfcb200_handle *h, const void *samples, int samples_on_device, int sigtype, uint32_t channels,
                                               uint32_t n_streams, uint64_t n_samples, uint32_t sample_rate, nfcb200_frame *out, uint64_t cap,
                                               uint64_t *n_out)
{
   if (!h)
      return fail(NFCB200_ERR_INVALID, "null handle");
   if (n_out)
      *n_out = 0;
   if (!is_logic(sigtype))
      return fail(NFCB200_ERR_INVALID, "signal type %d is not a logic format", sigtype);
   if (int rc = check_channels(channels))
      return rc;
   return iso_batch(h, samples, samples_on_device, sigtype, channels, iso_elem_bytes(sigtype), n_streams, n_samples, sample_rate, out, cap, n_out);
}

// ---------------------------------------------------------------------------------------------------------------------
// streaming: one capture, buffer by buffer
// ---------------------------------------------------------------------------------------------------------------------
extern "C" int nfcb200_iso7816_stream_reset(nfcb200_handle *h)
{
   if (!h)
      return fail(NFCB200_ERR_INVALID, "null handle");
   auto &S = h->isoStream;
   S.init = false;
   S.rate = 0;
   S.clock = 0;
   std::fill(S.last, S.last + 4, 0.f);
   S.pending.clear();
   return 0;
}

extern "C" int nfcb200_iso7816_stream_pending(nfcb200_handle *h, nfcb200_frame *out, uint64_t cap, uint64_t *n_out, uint64_t *n_left)
{
   if (!h)
      return fail(NFCB200_ERR_INVALID, "null handle");
   auto &S = h->isoStream;
   const uint64_t deliver = std::min<uint64_t>(S.pending.size(), out ? cap : 0);
   std::copy(S.pending.begin(), S.pending.begin() + (size_t) deliver, out);
   S.pending.erase(S.pending.begin(), S.pending.begin() + (size_t) deliver);
   if (n_out)
      *n_out = deliver;
   if (n_left)
      *n_left = S.pending.size();
   return 0;
}

// the push of both entry points (sigtype and channels checked)
static int iso_push(nfcb200_handle *h, const void *samples, int sigtype, uint32_t channels, uint64_t n, uint32_t sample_rate, nfcb200_frame *out,
                    uint64_t cap, uint64_t *n_out)
{
   if (cap && !out)
      return fail(NFCB200_ERR_INVALID, "null frame buffer");
   auto &S = h->isoStream;

   // n == 0 is nextFrames({}): an invalid buffer gives the decoder no sample (IsoTech.cpp:31-32), so it decodes nothing and
   // the next buffer picks its loop afresh anyway; only frames still pending are delivered
   if (n)
   {
      if (!samples)
         return fail(NFCB200_ERR_INVALID, "null samples");
      if (sample_rate == 0)
         return fail(NFCB200_ERR_INVALID, "sample rate of 0");
      // a buffer at another sample rate restarts the decoder's clock at 0 (IsoDecoder.cpp:172-178)
      const bool restart = !S.init || S.rate != sample_rate;
      const uint64_t base = restart ? 0 : S.clock;
      if (base + n >= 0xFFFFFFFFull)
         return fail(NFCB200_ERR_UNSUPPORTED, "stream position would pass 2^32 - 1 samples, the 32-bit sample clock of the reference (IsoTech.h:221): "
                                              "call nfcb200_iso7816_stream_reset");
      const uint64_t bs = (uint64_t) channels * iso_elem_bytes(sigtype);

      CUDA_TRY(cudaSetDevice(h->device));
      cudaStream_t st = h->stream;
      int rc;
      uint32_t poolCap = (uint32_t) std::max<uint64_t>(1024, S.pool.cap / sizeof(nfcb200_frame));
      if ((rc = S.ctr.reserve(8)) || (rc = S.pool.reserve((uint64_t) poolCap * sizeof(nfcb200_frame))) || (rc = S.streamCount.reserve(4)) ||
          (rc = S.state.reserve(2 * sizeof(iso7816::IsoStreamState))) || (rc = S.in.reserve(n * bs)))
         return rc;
      CUDA_TRY(cudaMemcpyAsync(S.in.ptr, samples, n * bs, cudaMemcpyHostToDevice, st));
      auto *state = S.state.as<iso7816::IsoStreamState>();
      if (!S.init) // the levels of the sample before the first are 0, like that sample
         CUDA_TRY(cudaMemsetAsync(state + S.cur, 0, sizeof(iso7816::IsoStreamState), st));

      IsoEdgesArgs E;
      if ((rc = edge_pass(st, sigtype, channels, S.in.ptr, 1, n, make_float4(S.last[0], S.last[1], S.last[2], S.last[3]), S.ev, S.ctr.as<uint32_t>() + 1, E)))
         return rc;
      IsoWalkArgs W = {};
      W.sample_rate = sample_rate;
      W.stream_time = h->cfg.stream_time;
      W.pool_count = S.ctr.as<uint32_t>();
      W.stream_count = S.streamCount.as<uint32_t>();
      W.resume = state + S.cur;
      W.state_out = state + (S.cur ^ 1);
      W.base = (uint32_t) base;
      W.restart = restart;
      uint32_t count = 0;
      if ((rc = walk_pass(st, E, W, 1, S.pool, poolCap, count)))
         return rc;
      // one stream's frames lie in the pool in decode order
      if (count)
      {
         const size_t old = S.pending.size();
         S.pending.resize(old + count);
         CUDA_TRY(cudaMemcpyAsync(S.pending.data() + old, W.pool, (uint64_t) count * sizeof(nfcb200_frame), cudaMemcpyDeviceToHost, st));
         CUDA_TRY(cudaStreamSynchronize(st));
         for (size_t i = old; i < S.pending.size(); i++)
            S.pending[i].reserved = 0;
      }

      S.cur ^= 1;
      S.init = true;
      S.rate = sample_rate;
      S.clock = (uint32_t) (base + n);
      // channels 0-3 of the last sample, as the decoder read them
      const unsigned char *tail = (const unsigned char *) samples + (n - 1) * bs;
      for (int c = 0; c < 4; c++)
         S.last[c] = sigtype == NFCB200_SIG_LOGIC_S16 ? ((const int16_t *) tail)[c] / 32768.f
                     : sigtype == NFCB200_SIG_LOGIC_U8 ? tail[c] / 255.f
                                                       : ((const float *) tail)[c];
   }

   const uint64_t nf = S.pending.size();
   uint64_t deliver = 0;
   nfcb200_iso7816_stream_pending(h, out, cap, &deliver, nullptr);
   if (n_out)
      *n_out = deliver;
   if (nf > cap)
      return fail(NFCB200_ERR_CAPACITY, "%llu frames decoded but room for %llu only: the rest waits in nfcb200_iso7816_stream_pending",
                  (unsigned long long) nf, (unsigned long long) cap);
   return 0;
}

extern "C" int nfcb200_iso7816_stream_push(nfcb200_handle *h, const void *samples, int sigtype, uint64_t n, uint32_t sample_rate, nfcb200_frame *out,
                                           uint64_t cap, uint64_t *n_out)
{
   if (!h)
      return fail(NFCB200_ERR_INVALID, "null handle");
   if (n_out)
      *n_out = 0;
   if (n && sigtype != NFCB200_SIG_LOGIC_F32 && sigtype != NFCB200_SIG_LOGIC_S16)
      return fail(NFCB200_ERR_INVALID, "signal type %d is not a 4-channel logic format", sigtype);
   return iso_push(h, samples, sigtype, 4, n, sample_rate, out, cap, n_out);
}

extern "C" int nfcb200_iso7816_stream_push_ch(nfcb200_handle *h, const void *samples, int sigtype, uint32_t channels, uint64_t n, uint32_t sample_rate,
                                              nfcb200_frame *out, uint64_t cap, uint64_t *n_out)
{
   if (!h)
      return fail(NFCB200_ERR_INVALID, "null handle");
   if (n_out)
      *n_out = 0;
   if (n && !is_logic(sigtype))
      return fail(NFCB200_ERR_INVALID, "signal type %d is not a logic format", sigtype);
   if (n)
      if (int rc = check_channels(channels))
         return rc;
   return iso_push(h, samples, sigtype, channels, n, sample_rate, out, cap, n_out);
}
