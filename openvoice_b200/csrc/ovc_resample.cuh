// Batched, ragged, windowable polyphase resampler (ovc_resample, include/ovc.h) and its ring form for live streams
// (ovc_resample_rings); arithmetic in ovc_resample.h.
//
// Grid (output tiles, items).  A CTA stages the input span of its tile's valid outputs in shared memory with
// coalesced loads (samples outside [0, len) or outside what the caller holds read as 0), then one thread per output
// sample runs output_at over the staged samples.  Outputs at or past n_out(len) are written as 0, so a row is ready for
// the spectrogram, which expects zero padding.  The fp64 bank ([up][K], 52 KB at 48 kHz -> 22.05 kHz, 206 KB from
// 192 kHz) is read through the read-only data cache: each thread walks K consecutive taps of its phase.
//
// The staged samples are converted to fp64 once (S = double): converting in the tap loop would run at a quarter of
// the FP64 FMA rate.  Only pairs whose single-output support overflows shared memory as doubles (up = 1 and
// down > ~1450, e.g. 2048 Hz -> 1 Hz) stage fp32 (S = float); the sum is the same either way.
//
// resample_kernel (one plan, rows of a [B, pitch] array) and resample_ring_kernel (a plan per item, ring rows in, ring
// rows or a packed buffer out) share the tile body, resample_tile; only the loader and the storer differ.
#pragma once
#include "ovc_resample.h"

namespace ovc {

// staged input samples a tile of `tile` outputs needs, whatever its first output
inline int64_t resample_stage_len(const ovc_rs::Plan& p, int64_t tile) {
  return ((tile - 1) * p.down + p.taps - 1) / p.up + 2;
}

// Outputs [m0, m0 + n) of plan p, the ones at or past nout written as 0.  load(j) returns input sample j (0 where the
// caller holds none); store(i, v) writes output m0 + i.  Every thread of the CTA calls it (one __syncthreads).
template <class S, class Load, class Store>
__device__ __forceinline__ void resample_tile(const ovc_rs::Plan& p, const double* __restrict__ bank, S* xs, int64_t m0,
                                              int64_t n, int64_t nout, Load load, Store store) {
  const int64_t mv = min(m0 + n, nout);                // valid outputs of the tile: [m0, mv)
  int64_t s0 = 0, s1 = 0;
  if (mv > m0) ovc_rs::span(p, m0, mv, &s0, &s1);
  for (int64_t j = s0 + threadIdx.x; j < s1; j += blockDim.x) xs[j - s0] = (S)load(j);
  __syncthreads();
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const int64_t m = m0 + i;
    store(i, m < nout ? (float)ovc_rs::output_at(p, bank, (const S*)xs, s0, m) : 0.f);
  }
}

template <class S>
__global__ void __launch_bounds__(256) resample_kernel(ovc_rs::Plan p, const double* __restrict__ bank,
                                                       const float* __restrict__ in, int64_t in_pitch, int64_t in_start,
                                                       const int64_t* __restrict__ in_lengths, float* __restrict__ out,
                                                       int64_t out_pitch, int64_t out_start, int tile) {
  extern __shared__ __align__(16) unsigned char rs_smem[];
  const int b = blockIdx.y;
  const int64_t len = in_lengths[b] > 0 ? in_lengths[b] : 0;
  const int64_t r0 = (int64_t)blockIdx.x * tile;
  const int64_t r1 = min(r0 + (int64_t)tile, out_pitch);
  const float* row = in + (int64_t)b * in_pitch;
  float* orow = out + (int64_t)b * out_pitch + r0;
  resample_tile<S>(
      p, bank, reinterpret_cast<S*>(rs_smem), out_start + r0, r1 - r0, ovc_rs::n_out(p, len),
      [&](int64_t j) {
        const int64_t k = j - in_start;
        return (j >= 0 && j < len && k >= 0 && k < in_pitch) ? row[k] : 0.f;
      },
      [&](int64_t i, float v) { orow[i] = v; });
}

// one entry of a context's plan table (ovc_resample_plan)
struct RsRingPlan {
  ovc_rs::Plan p;
  const double* bank;
  int dbl;                      // stage fp64 (the rule of ovc_resample), else fp32
};

// Item b: outputs [m0, m0 + count) of plan[b], input sample j at in[in_row * in_cap + j mod in_cap] (0 outside
// [0, in_len)), output m at out[out_row * out_cap + (out_off + m - m0) mod out_cap]; descriptors clamped by
// ovc_rs::ring_item.  CTA (x, b) computes the item's outputs [x tile, (x + 1) tile) below its count.
__global__ void __launch_bounds__(256) resample_ring_kernel(
    const RsRingPlan* __restrict__ plans, int n_plans, const int32_t* __restrict__ plan, const float* __restrict__ in,
    int64_t in_rows, int64_t in_cap, const int64_t* __restrict__ in_row, const int64_t* __restrict__ in_len,
    const int64_t* __restrict__ m0, const int64_t* __restrict__ count, float* __restrict__ out, int64_t out_rows,
    int64_t out_cap, const int64_t* __restrict__ out_row, const int64_t* __restrict__ out_off, int64_t max_count,
    int tile) {
  extern __shared__ __align__(16) unsigned char rs_smem[];
  const int b = blockIdx.y;
  const ovc_rs::RingItem it = ovc_rs::ring_item(plan[b], in_row[b], in_len[b], m0[b], count[b], out_row[b], out_off[b],
                                                n_plans, in_rows, out_rows, out_cap, max_count);
  const int64_t r0 = (int64_t)blockIdx.x * tile;
  if (r0 >= it.count) return;                          // the whole CTA: before the tile's barrier
  const int64_t n = min((int64_t)tile, it.count - r0);
  const RsRingPlan P = plans[it.plan];
  const int64_t nout = ovc_rs::n_out(P.p, it.in_len);
  auto load = [&](int64_t j) {
    const int64_t k = ovc_rs::ring_in_at(it, j, in_cap);
    return k >= 0 ? in[k] : 0.f;
  };
  auto store = [&](int64_t i, float v) { out[ovc_rs::ring_out_at(it, r0 + i, out_cap)] = v; };
  if (P.dbl)
    resample_tile<double>(P.p, P.bank, reinterpret_cast<double*>(rs_smem), it.m0 + r0, n, nout, load, store);
  else
    resample_tile<float>(P.p, P.bank, reinterpret_cast<float*>(rs_smem), it.m0 + r0, n, nout, load, store);
}

}  // namespace ovc
