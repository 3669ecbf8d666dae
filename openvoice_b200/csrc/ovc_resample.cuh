// Batched, ragged, windowable polyphase resampler (ovc_resample, include/ovc.h); arithmetic in ovc_resample.h.
//
// Grid (output tiles, items).  A CTA stages the input span of its tile's valid outputs in shared memory with
// coalesced loads (samples outside [0, len) or outside the supplied row read as 0), then one thread per output sample
// runs output_at over the staged samples.  Outputs at or past n_out(len) are written as 0, so a row is ready for the
// spectrogram, which expects zero padding.  The fp64 bank ([up][K], 52 KB at 48 kHz -> 22.05 kHz, 206 KB from
// 192 kHz) is read through the read-only data cache: each thread walks K consecutive taps of its phase.
//
// The staged samples are converted to fp64 once (S = double): converting in the tap loop would run at a quarter of
// the FP64 FMA rate.  Only pairs whose single-output support overflows shared memory as doubles (up = 1 and
// down > ~1450, e.g. 2048 Hz -> 1 Hz) stage fp32 (S = float); the sum is the same either way.
#pragma once
#include "ovc_resample.h"

namespace ovc {

// staged input samples a tile of `tile` outputs needs, whatever its first output
inline int64_t resample_stage_len(const ovc_rs::Plan& p, int64_t tile) {
  return ((tile - 1) * p.down + p.taps - 1) / p.up + 2;
}

template <class S>
__global__ void __launch_bounds__(256) resample_kernel(ovc_rs::Plan p, const double* __restrict__ bank,
                                                       const float* __restrict__ in, int64_t in_pitch, int64_t in_start,
                                                       const int64_t* __restrict__ in_lengths, float* __restrict__ out,
                                                       int64_t out_pitch, int64_t out_start, int tile) {
  extern __shared__ __align__(16) unsigned char rs_smem[];
  S* xs = reinterpret_cast<S*>(rs_smem);
  const int b = blockIdx.y;
  const int64_t len = in_lengths[b] > 0 ? in_lengths[b] : 0;
  const int64_t nout = ovc_rs::n_out(p, len);
  const int64_t r0 = (int64_t)blockIdx.x * tile;
  const int64_t r1 = min(r0 + (int64_t)tile, out_pitch);
  const int64_t m0 = out_start + r0;
  const int64_t mv = min(out_start + r1, nout);        // valid outputs of the tile: [m0, mv)
  int64_t s0 = 0, s1 = 0;
  if (mv > m0) ovc_rs::span(p, m0, mv, &s0, &s1);
  const float* row = in + (int64_t)b * in_pitch;
  for (int64_t j = s0 + threadIdx.x; j < s1; j += blockDim.x) {
    const int64_t k = j - in_start;
    xs[j - s0] = (S)((j >= 0 && j < len && k >= 0 && k < in_pitch) ? row[k] : 0.f);
  }
  __syncthreads();
  for (int64_t r = r0 + threadIdx.x; r < r1; r += blockDim.x) {
    const int64_t m = out_start + r;
    out[(int64_t)b * out_pitch + r] = m < nout ? (float)ovc_rs::output_at(p, bank, (const S*)xs, s0, m) : 0.f;
  }
}

}  // namespace ovc
