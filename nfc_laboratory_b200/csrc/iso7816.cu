/*
 * iso7816.cu -- nfcb200_iso7816_decode_batch: ISO 7816 contact smart-card traffic from 4-channel logic captures
 * (lab::IsoDecoder, iso_decode.cuh).
 */
#include <numeric>

#include "host.h"
#include "iso_decode.cuh"

using namespace nfcb200;

extern "C" int nfcb200_iso7816_decode_batch(nfcb200_handle *h, const void *samples, int samples_on_device, int sigtype, uint32_t n_streams,
                                            uint64_t n_samples, uint32_t sample_rate, nfcb200_frame *out, uint64_t cap, uint64_t *n_out)
{
   if (!h)
      return fail(NFCB200_ERR_INVALID, "null handle");
   if (n_out)
      *n_out = 0;
   if (sigtype != NFCB200_SIG_LOGIC_F32 && sigtype != NFCB200_SIG_LOGIC_S16)
      return fail(NFCB200_ERR_INVALID, "signal type %d is not a 4-channel logic format", sigtype);
   if (sample_rate == 0)
      return fail(NFCB200_ERR_INVALID, "sample rate of 0");
   if (!samples || n_streams == 0 || n_samples == 0)
      return fail(NFCB200_ERR_INVALID, "empty batch");
   if (cap && !out)
      return fail(NFCB200_ERR_INVALID, "null frame buffer");
   if (n_samples >= 0xFFFFFFFFull)
      return fail(NFCB200_ERR_UNSUPPORTED, "streams of 2^32 - 1 samples or more exceed the 32-bit sample clock of the reference (IsoTech.h:221)");
   const bool s16 = sigtype == NFCB200_SIG_LOGIC_S16;
   const uint64_t bs = s16 ? 8 : 16;
   if (samples_on_device && ((uintptr_t) samples % bs))
      return fail(NFCB200_ERR_INVALID, "device samples not aligned to %u bytes", (unsigned) bs);

   CUDA_TRY(cudaSetDevice(h->device));
   cudaStream_t st = h->stream;
   auto &I = h->iso;
   int rc;

   const uint32_t nTiles = (uint32_t) ((n_samples + ISO_TILE - 1) / ISO_TILE);
   uint32_t poolCap = (uint32_t) std::max<uint64_t>(1024, I.pool.cap / sizeof(nfcb200_frame));
   if ((rc = I.ctr.reserve(8)) || (rc = I.pool.reserve((uint64_t) poolCap * sizeof(nfcb200_frame))))
      return rc;

   uint64_t nf = 0; // frames of the groups so far
   auto group = [&](uint32_t s0, uint32_t sc, const void *dSamples) -> int {
      if ((rc = I.clkCount.reserve((uint64_t) sc * nTiles * 4)) || (rc = I.lineCount.reserve((uint64_t) sc * nTiles * 4)) ||
          (rc = I.streamCount.reserve((uint64_t) sc * 4)) || (rc = I.first.reserve((uint64_t) sc * 8)))
         return rc;
      IsoEdgesArgs E = {};
      E.samples = dSamples;
      E.n_samples = n_samples;
      E.n_tiles = nTiles;
      E.line_count = I.lineCount.as<uint32_t>();
      E.clk_count = I.clkCount.as<uint32_t>();
      E.overflow = I.ctr.as<uint32_t>() + 1;
      // the dense pass, again with room for a line event and a CLK falling edge at every sample when a tile overflows
      // the first try's slots
      for (E.line_cap = ISO_LINE_CAP, E.clk_cap = ISO_CLK_CAP;; E.line_cap = E.clk_cap = ISO_TILE)
      {
         if ((rc = I.line.reserve((uint64_t) sc * nTiles * E.line_cap * 4)) || (rc = I.clk.reserve((uint64_t) sc * nTiles * E.clk_cap * sizeof(uint16_t))))
            return rc;
         E.line = I.line.as<uint32_t>();
         E.clk = I.clk.as<uint16_t>();
         CUDA_TRY(cudaMemsetAsync(E.overflow, 0, 4, st));
         const dim3 grid(nTiles, sc);
         if (s16)
            iso_edges_kernel<true><<<grid, ISO_THREADS, 0, st>>>(E);
         else
            iso_edges_kernel<false><<<grid, ISO_THREADS, 0, st>>>(E);
         CUDA_TRY(cudaGetLastError());
         uint32_t overflow = 0;
         CUDA_TRY(cudaMemcpyAsync(&overflow, E.overflow, 4, cudaMemcpyDeviceToHost, st));
         CUDA_TRY(cudaStreamSynchronize(st));
         if (!overflow || E.line_cap == ISO_TILE)
            break;
      }
      // the walk, again with a larger pool when the frames did not fit
      IsoWalkArgs W = {};
      W.n_streams = sc;
      W.stream0 = s0;
      W.n_samples = (uint32_t) n_samples;
      W.n_tiles = nTiles;
      W.line_cap = E.line_cap;
      W.clk_cap = E.clk_cap;
      W.sample_rate = sample_rate;
      W.stream_time = h->cfg.stream_time;
      W.line = E.line;
      W.line_count = E.line_count;
      W.clk = E.clk;
      W.clk_count = E.clk_count;
      W.pool_count = I.ctr.as<uint32_t>();
      W.stream_count = I.streamCount.as<uint32_t>();
      uint32_t count = 0;
      while (true)
      {
         W.pool = I.pool.as<nfcb200_frame>();
         W.pool_cap = poolCap;
         CUDA_TRY(cudaMemsetAsync(W.pool_count, 0, 4, st));
         iso_walk_kernel<<<sc, 32, 0, st>>>(W);
         CUDA_TRY(cudaGetLastError());
         CUDA_TRY(cudaMemcpyAsync(&count, W.pool_count, 4, cudaMemcpyDeviceToHost, st));
         CUDA_TRY(cudaStreamSynchronize(st));
         if (count <= poolCap)
            break;
         poolCap = count;
         if ((rc = I.pool.reserve((uint64_t) poolCap * sizeof(nfcb200_frame))))
            return rc;
      }
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
