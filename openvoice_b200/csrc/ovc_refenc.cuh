// ovc_refenc.cuh -- the tone-colour (speaker) embedding extractor of extract_se, row f2 of SURVEY.md section 8:
// ReferenceEncoder.forward (openvoice/models.py:339-359) = LayerNorm over frequency, 6 x (Conv2d 3x3 stride 2
// pad 1 + ReLU), GRU(1152 -> 128) last hidden state, Linear(128 -> gin).  ~1 GFLOP per 10 s clip and run once
// per reference speaker, so these are plain direct kernels -- correctness and "no PyTorch module on the path",
// not throughput, are the point.
//
// Ragged batches: every kernel takes an optional `lengths` [N] (frames, device).  Item n's limit at layer 0 is
// h0 = clamp(lengths[n], 1, T0) (the clamp keeps a bad device value inside the buffers) and each stride-2 conv maps a
// limit h to (h - 1) / 2 + 1, the host's H[] formula.  Rows at or past an item's limit are never read (a conv tap
// there is skipped exactly like a tap past Hi, not multiplied by zero) and never computed, so row n gets the fmaf
// sequence of a solo call at its own length, bit for bit, whatever the padding holds.  Grids and row pitches are
// sized by T0; threads past a limit return.  lengths == nullptr: every item is T0 frames.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "ovc_refenc_stream.h"
#include "ovc_small.cuh"

namespace ovc {

// limit (valid rows) of item n after `layer` stride-2 convs
__device__ __forceinline__ int refenc_limit(const int64_t* __restrict__ lengths, int n, int T0, int layer) {
  int h = T0;
  if (lengths) {
    const int64_t l = lengths[n];
    h = l < 1 ? 1 : (l > T0 ? T0 : (int)l);
  }
  for (int i = 0; i < layer; ++i) h = (h - 1) / 2 + 1;
  return h;
}

// The per-element bodies below are shared by the whole-clip kernels and refenc_stream_kernel, so a streamed row gets
// the same fmaf sequence as a clip.

// LayerNorm of one frame: s[f * stride], f < F -> o[f]; one warp, every lane calls it
__device__ __forceinline__ void refenc_ln_row(const float* __restrict__ s, size_t stride, const float* __restrict__ gamma,
                                              const float* __restrict__ beta, float* __restrict__ o_, int F, int lane) {
  float sum = 0.f;
  for (int f = lane; f < F; f += 32) sum += s[(size_t)f * stride];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / F;
  float var = 0.f;
  for (int f = lane; f < F; f += 32) { const float d = s[(size_t)f * stride] - mean; var += d * d; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) var += __shfl_xor_sync(0xffffffffu, var, o);
  const float rstd = rsqrtf(var / F + 1e-5f);   // nn.LayerNorm default eps, biased variance
  for (int f = lane; f < F; f += 32) o_[f] = (s[(size_t)f * stride] - mean) * rstd * gamma[f] + beta[f];
}

// one output element of Conv2d(3x3, stride 2, padding 1) + ReLU: row(ci, hi) points at input row hi of channel ci
// (Wi floats); taps outside [0, hin) x [0, Wi) are skipped
template <class Row>
__device__ __forceinline__ float refenc_conv_point(const Row& row, const float* __restrict__ w, const float* __restrict__ bias,
                                                   int Cin, int Wi, int co, int ho, int wo, int hin) {
  float acc = bias[co];
  const float* wc = w + (size_t)co * Cin * 9;
  for (int ci = 0; ci < Cin; ++ci) {
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int hi = 2 * ho - 1 + kh;
      if (hi < 0 || hi >= hin) continue;
      const float* xr = row(ci, hi);
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int wi = 2 * wo - 1 + kw;
        if (wi < 0 || wi >= Wi) continue;
        acc = fmaf(wc[ci * 9 + kh * 3 + kw], xr[wi], acc);
      }
    }
  }
  return acc > 0.f ? acc : 0.f;
}

// W_ih[j,:] . feat over K inputs, lane-strided then reduced by the xor butterfly (every lane gets the sum)
template <class Feat>
__device__ __forceinline__ float refenc_gru_in_dot(const float* __restrict__ wr, const Feat& feat, int K, int lane) {
  float s = 0.f;
  for (int k = lane; k < K; k += 32) s = fmaf(wr[k], feat(k), s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}

// one GRU step of hidden unit j (gate order r, z, n like torch.nn.GRU): g = the step's input projections [384],
// h = the hidden state [128]; returns the new h[j]
__device__ __forceinline__ float refenc_gru_cell(const float* __restrict__ g, const float* h, const float* __restrict__ w_hh,
                                                 const float* __restrict__ b_hh, int j) {
  float gr = b_hh[j], gz = b_hh[128 + j], gn = b_hh[256 + j];
  for (int k = 0; k < 128; ++k) {
    const float hk = h[k];
    gr = fmaf(w_hh[(size_t)j * 128 + k], hk, gr);
    gz = fmaf(w_hh[(size_t)(128 + j) * 128 + k], hk, gz);
    gn = fmaf(w_hh[(size_t)(256 + j) * 128 + k], hk, gn);
  }
  const float r = 1.f / (1.f + expf(-(g[j] + gr)));
  const float z = 1.f / (1.f + expf(-(g[128 + j] + gz)));
  const float c = tanhf(g[256 + j] + r * gn);
  return (1.f - z) * c + z * h[j];
}

// output o of the final Linear(128 -> gin) on the hidden state h
__device__ __forceinline__ float refenc_proj(const float* __restrict__ pw, const float* __restrict__ pb, const float* h, int o) {
  float s = pb[o];
  for (int k = 0; k < 128; ++k) s = fmaf(pw[(size_t)o * 128 + k], h[k], s);
  return s;
}

// LayerNorm(spec_channels) on the [N][F][T] spectrogram, written as the conv stack's [N][1][T][F] input
// (the reference feeds y.transpose(1,2).view(N,1,T,F), api.py:130 / models.py:342-344).  One warp per (n, t).
__global__ void __launch_bounds__(256) refenc_layernorm_kernel(const float* __restrict__ spec, const float* __restrict__ gamma,
                                                               const float* __restrict__ beta, float* __restrict__ out, int N,
                                                               int F, int T, const int64_t* __restrict__ lengths) {
  const int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (wid >= N * T) return;
  const int n = wid / T, t = wid % T;
  if (t >= refenc_limit(lengths, n, T, 0)) return;   // warp-uniform
  refenc_ln_row(spec + (size_t)n * F * T + t, T, gamma, beta, out + ((size_t)n * T + t) * F, F, lane);
}

// Conv2d(3x3, stride 2, padding 1) + ReLU, NCHW, one thread per output element; `layer` (0..5) is the conv's index
// in the stack and T0 the layer-0 row count, for the per-item limits
__global__ void __launch_bounds__(256) refenc_conv_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                          const float* __restrict__ bias, float* __restrict__ y, int N, int Cin,
                                                          int Hi, int Wi, int Cout, int Ho, int Wo,
                                                          const int64_t* __restrict__ lengths, int T0, int layer) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)N * Cout * Ho * Wo;
  if (idx >= total) return;
  const int wo = (int)(idx % Wo), ho = (int)((idx / Wo) % Ho), co = (int)((idx / ((long long)Wo * Ho)) % Cout);
  const int n = (int)(idx / ((long long)Wo * Ho * Cout));
  const int hin = refenc_limit(lengths, n, T0, layer);
  if (ho >= (hin - 1) / 2 + 1) return;
  const auto row = [&](int ci, int hi) { return x + ((size_t)n * Cin + ci) * Hi * Wi + (size_t)hi * Wi; };
  y[idx] = refenc_conv_point(row, w, bias, Cin, Wi, co, ho, wo, hin);
}

// GRU input projections for every step at once: gi[n][t][j] = b_ih[j] + W_ih[j,:] . feat[n][t][:], where
// feat[n][t][c*Wf + w] = conv6[n][c][t][w] (out.transpose(1,2).view(N,T,-1), models.py:351-354).  One warp per output.
__global__ void __launch_bounds__(256) refenc_gru_in_kernel(const float* __restrict__ conv, const float* __restrict__ w_ih,
                                                            const float* __restrict__ b_ih, float* __restrict__ gi, int N, int C,
                                                            int Tq, int Wf, int G, const int64_t* __restrict__ lengths, int T0) {
  const int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (wid >= N * Tq * G) return;
  const int j = wid % G, t = (wid / G) % Tq, n = wid / (G * Tq);
  if (t >= refenc_limit(lengths, n, T0, 6)) return;   // warp-uniform
  const int K = C * Wf;
  const float* wr = w_ih + (size_t)j * K;
  const auto feat = [&](int k) {
    const int c = k / Wf, wf = k % Wf;
    return conv[(((size_t)n * C + c) * Tq + t) * Wf + wf];
  };
  const float s = refenc_gru_in_dot(wr, feat, K, lane);
  if (lane == 0) gi[wid] = s + b_ih[j];
}

// GRU recurrence (gate order r, z, n like torch.nn.GRU) over the item's own h6 steps + the final Linear; one CTA of
// 128 threads per item
__global__ void __launch_bounds__(128) refenc_gru_kernel(const float* __restrict__ gi, const float* __restrict__ w_hh,
                                                         const float* __restrict__ b_hh, const float* __restrict__ pw,
                                                         const float* __restrict__ pb, float* __restrict__ out, int Tq, int gin,
                                                         const int64_t* __restrict__ lengths, int T0) {
  __shared__ float h[128];
  const int n = blockIdx.x, j = threadIdx.x;
  const int steps = refenc_limit(lengths, n, T0, 6);
  h[j] = 0.f;
  __syncthreads();
  for (int t = 0; t < steps; ++t) {
    const float hn = refenc_gru_cell(gi + ((size_t)n * Tq + t) * 384, h, w_hh, b_hh, j);
    __syncthreads();
    h[j] = hn;
    __syncthreads();
  }
  for (int o = j; o < gin; o += 128) out[(size_t)n * gin + o] = refenc_proj(pw, pb, h, o);
}

// ---------------------------------------------------------------------------------------------
// ovc_reference_encoder_stream: the encoder advanced with live streams held in audio rings, state rows as laid out by
// ovc_re::geom (ovc_refenc_stream.h).  Item b of a call is descriptor desc[4 b ..] = (state_row, ring_row, n_adv,
// n_snap), clamped by ovc_re::item.  Two launches: stft_refenc_kernel writes the item's new final frames [c0, a2) into
// columns [0, a2 - c0) of spec[b] and its snapshot tail frames [a1, a1 + tail) (reflected at n_snap) after them, then
// refenc_stream_kernel (one CTA per item) runs LayerNorm, the six convs and the GRU on those rows, layer by layer.
// ---------------------------------------------------------------------------------------------
struct RefencWeights {
  const float* ln_g;
  const float* ln_b;
  const float* conv_w[6];
  const float* conv_b[6];
  const float *w_ih, *b_ih, *w_hh, *b_hh, *pw, *pb;
};

__device__ __forceinline__ ovc_re::Item refenc_stream_item(const float* state, int state_rows, long long state_floats,
                                                           const int64_t* d, int ring_rows, int max_new, int hop) {
  const int64_t row = ovc_re::clamp64(d[0], 0, state_rows - 1);
  const int64_t c0 = *reinterpret_cast<const int64_t*>(state + row * state_floats);
  return ovc_re::item(d, c0, state_rows, ring_rows, max_new, hop, STFT_N);
}

__global__ void __launch_bounds__(256) stft_refenc_kernel(const float* __restrict__ rings, long long cap, int ring_rows,
                                                          const float* __restrict__ state, int state_rows,
                                                          long long state_floats, const int64_t* __restrict__ desc,
                                                          int max_new, int hop, float* __restrict__ spec, int Tcols,
                                                          const float2* __restrict__ tw, const float* __restrict__ win) {
  const int b = blockIdx.y, t0 = blockIdx.x * STFT_FR;
  const ovc_re::Item it = refenc_stream_item(state, state_rows, state_floats, desc + 4 * b, ring_rows, max_new, hop);
  const int nadv = (int)(it.a2 - it.c0), T = nadv + it.tail;
  if (t0 >= T) return;   // block-uniform; columns past T are never read
  const float* ring = rings + it.ring_row * cap;
  const auto load = [&](int t, int n) {
    return t < nadv ? ring_frame_sample(ring, cap, RING_OPEN, it.c0 + t, n, hop)
                    : ring_frame_sample(ring, cap, it.n_snap, it.a1 + (t - nadv), n, hop);
  };
  stft_block(load, T, t0, spec + (size_t)b * (STFT_N / 2 + 1) * Tcols, Tcols, Tcols, tw, win);
}

__global__ void __launch_bounds__(256) refenc_stream_kernel(const RefencWeights P, const float* __restrict__ spec, int Tcols,
                                                            float* __restrict__ state, int state_rows,
                                                            const int64_t* __restrict__ desc, int ring_rows, int max_new,
                                                            int hop, int F, int gin, float* __restrict__ ws,
                                                            long long ws_item, float* __restrict__ out) {
  __shared__ float h[128], hs[128];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const ovc_re::Geom G = ovc_re::geom(F);
  const ovc_re::Item it = refenc_stream_item(state, state_rows, G.floats, desc + 4 * b, ring_rows, max_new, hop);
  float* st = state + it.state_row * G.floats;
  const float* sp = spec + (size_t)b * F * Tcols;
  float* nb[ovc_re::LAYERS + 1];   // rows of layer l from the layer's first non-carry row on
  {
    float* p = ws + (size_t)b * ws_item;
#pragma unroll
    for (int l = 0; l <= ovc_re::LAYERS; ++l) {
      nb[l] = p;
      p += ovc_re::ws_rows(max_new, l) * ovc_re::filt(l) * G.W[l];
    }
  }
  float* gi = nb[ovc_re::LAYERS] + ovc_re::ws_rows(max_new, ovc_re::LAYERS) * ovc_re::filt(ovc_re::LAYERS) * G.W[ovc_re::LAYERS];
  const int K = ovc_re::filt(ovc_re::LAYERS) * G.W[ovc_re::LAYERS];
  if (tid < 128) h[tid] = st[G.h + tid];

  // LayerNorm of frames [t0, t0 + n) from spec columns col0 .. into nb[0]
  const auto layernorm = [&](int col0, int n) {
    for (int t = warp; t < n; t += nwarps) refenc_ln_row(sp + col0 + t, Tcols, P.ln_g, P.ln_b, nb[0] + (size_t)t * F, F, lane);
    __syncthreads();
  };
  // rows [o0, o1) of layer l + 1 into nb[l + 1]: input rows below cin from the carry (slot row & 1), rows from cin on
  // from nb[l]; taps at or past hin are skipped
  const auto conv = [&](int l, int cin, int hin, int o0, int o1) {
    const int Cin = ovc_re::filt(l), Wi = G.W[l], Co = ovc_re::filt(l + 1), Wo = G.W[l + 1];
    const float* carry = st + G.carry[l];
    const float* in = nb[l];
    const auto row = [&](int ci, int hi) {
      return (hi < cin ? carry + (size_t)(hi & 1) * Cin * Wi : in + (size_t)(hi - cin) * Cin * Wi) + (size_t)ci * Wi;
    };
    const int total = (o1 - o0) * Co * Wo;
    for (int e = tid; e < total; e += blockDim.x) {
      const int wo = e % Wo, co = (e / Wo) % Co, r = e / (Wo * Co);
      nb[l + 1][e] = refenc_conv_point(row, P.conv_w[l], P.conv_b[l], Cin, Wi, co, o0 + r, wo, hin);
    }
    __syncthreads();
  };
  // GRU steps [s0, s1) on hh, reading their inputs from nb[6]
  const auto gru = [&](int s0, int s1, float* hh) {
    const int n = s1 - s0;
    if (n <= 0) return;   // block-uniform
    for (int e = warp; e < n * 384; e += nwarps) {
      const int t = e / 384, j = e % 384;
      const float* x = nb[ovc_re::LAYERS] + (size_t)t * K;
      const float s = refenc_gru_in_dot(P.w_ih + (size_t)j * K, [&](int k) { return x[k]; }, K, lane);
      if (lane == 0) gi[e] = s + P.b_ih[j];
    }
    __syncthreads();
    for (int t = 0; t < n; ++t) {
      float hn = 0.f;
      if (tid < 128) hn = refenc_gru_cell(gi + (size_t)t * 384, hh, P.w_hh, P.b_hh, tid);
      __syncthreads();
      if (tid < 128) hh[tid] = hn;
      __syncthreads();
    }
  };
  // advance the row from cA to cB final frames, whose spectrogram starts at column col0
  const auto advance = [&](int cA, int cB, int col0) {
    if (cB <= cA) return;   // block-uniform
    layernorm(col0, cB - cA);
#pragma unroll
    for (int l = 0; l < ovc_re::LAYERS; ++l) conv(l, cA >> l, cB >> l, cA >> (l + 1), cB >> (l + 1));
    gru(cA >> ovc_re::LAYERS, cB >> ovc_re::LAYERS, h);
#pragma unroll
    for (int l = 0; l < ovc_re::LAYERS; ++l) {   // the carry: rows [max(c, carry_lo(c')), c') of nb[l]
      const int c = cA >> l, c1 = cB >> l, Cw = ovc_re::filt(l) * G.W[l];
      const int r0 = max(c, (int)ovc_re::carry_lo(c1));
      for (int e = tid; e < (c1 - r0) * Cw; e += blockDim.x) {
        const int r = r0 + e / Cw;
        st[G.carry[l] + (size_t)(r & 1) * Cw + e % Cw] = nb[l][(size_t)(r - c) * Cw + e % Cw];
      }
    }
    __syncthreads();
  };

  __syncthreads();
  advance((int)it.c0, (int)it.a1, 0);
  if (it.snap_ok) {   // the snapshot's tail rows [c_l, limit_l) from the carry, its final hidden state and the Linear
    const int a = (int)it.a1;
    int lim = (int)it.T;
    layernorm((int)(it.a2 - it.c0), it.tail);
#pragma unroll
    for (int l = 0; l < ovc_re::LAYERS; ++l) {
      const int lim1 = (lim - 1) / 2 + 1;
      conv(l, a >> l, lim, a >> (l + 1), lim1);
      lim = lim1;
    }
    if (tid < 128) hs[tid] = h[tid];
    __syncthreads();
    gru(a >> ovc_re::LAYERS, lim, hs);
    for (int o = tid; o < gin; o += blockDim.x) out[(size_t)b * gin + o] = refenc_proj(P.pw, P.pb, hs, o);
  } else if (it.snap) {
    for (int o = tid; o < gin; o += blockDim.x) out[(size_t)b * gin + o] = __int_as_float(0x7fc00000);
  }
  advance((int)it.a1, (int)it.a2, (int)(it.a1 - it.c0));
  if (tid < 128) st[G.h + tid] = h[tid];
  if (tid == 0) *reinterpret_cast<int64_t*>(st) = it.a2;
}

}  // namespace ovc
