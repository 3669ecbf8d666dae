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

// LayerNorm(spec_channels) on the [N][F][T] spectrogram, written as the conv stack's [N][1][T][F] input
// (the reference feeds y.transpose(1,2).view(N,1,T,F), api.py:130 / models.py:342-344).  One warp per (n, t).
__global__ void __launch_bounds__(256) refenc_layernorm_kernel(const float* __restrict__ spec, const float* __restrict__ gamma,
                                                               const float* __restrict__ beta, float* __restrict__ out, int N,
                                                               int F, int T, const int64_t* __restrict__ lengths) {
  const int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (wid >= N * T) return;
  const int n = wid / T, t = wid % T;
  if (t >= refenc_limit(lengths, n, T, 0)) return;   // warp-uniform
  const float* s = spec + (size_t)n * F * T + t;
  float sum = 0.f;
  for (int f = lane; f < F; f += 32) sum += s[(size_t)f * T];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / F;
  float var = 0.f;
  for (int f = lane; f < F; f += 32) { const float d = s[(size_t)f * T] - mean; var += d * d; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) var += __shfl_xor_sync(0xffffffffu, var, o);
  const float rstd = rsqrtf(var / F + 1e-5f);   // nn.LayerNorm default eps, biased variance
  float* o_ = out + ((size_t)n * T + t) * F;
  for (int f = lane; f < F; f += 32) o_[f] = (s[(size_t)f * T] - mean) * rstd * gamma[f] + beta[f];
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
  float acc = bias[co];
  const float* wc = w + (size_t)co * Cin * 9;
  for (int ci = 0; ci < Cin; ++ci) {
    const float* xc = x + ((size_t)n * Cin + ci) * Hi * Wi;
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int hi = 2 * ho - 1 + kh;
      if (hi < 0 || hi >= hin) continue;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int wi = 2 * wo - 1 + kw;
        if (wi < 0 || wi >= Wi) continue;
        acc = fmaf(wc[ci * 9 + kh * 3 + kw], xc[(size_t)hi * Wi + wi], acc);
      }
    }
  }
  y[idx] = acc > 0.f ? acc : 0.f;
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
  float s = 0.f;
  for (int k = lane; k < K; k += 32) {
    const int c = k / Wf, wf = k % Wf;
    s = fmaf(wr[k], conv[(((size_t)n * C + c) * Tq + t) * Wf + wf], s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
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
    const float* g = gi + ((size_t)n * Tq + t) * 384;
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
    const float hn = (1.f - z) * c + z * h[j];
    __syncthreads();
    h[j] = hn;
    __syncthreads();
  }
  for (int o = j; o < gin; o += 128) {
    float s = pb[o];
    for (int k = 0; k < 128; ++k) s = fmaf(pw[(size_t)o * 128 + k], h[k], s);
    out[(size_t)n * gin + o] = s;
  }
}

}  // namespace ovc
