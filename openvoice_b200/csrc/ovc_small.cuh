// ovc_small.cuh -- the non-GEMM kernels of the hot path: speaker-conditioning mat-vec,
// conv_post (+leaky_relu 0.01, tanh), latent copy-out.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ovc {

// ---------------------------------------------------------------------------------------------
// cond_kernel: every 1x1 conv the reference applies to the [B, gin, 1] speaker embedding
// (WN.cond_layer of enc_q and of the 4 couplings, modules.py:189-190; Generator.cond,
// models.py:274-275) is a mat-vec.  All of them run in ONE launch: row `i` of the stacked,
// pre-permuted matrix dotted with g_src / g_tgt / zeros (zero_g) of batch item b.  The bias of
// the conv that consumes the result (in_layer / conv_pre) is pre-added on the host, so the conv
// epilogues add a single per-(batch,row) vector.  One warp per output, warp-shuffle reduction.
// ---------------------------------------------------------------------------------------------
struct CondArgs {
  const float* w;        // [rows_w][gin]
  const float* bias;     // [rows_out]
  const int* w_row;      // [rows_out] matrix row feeding output row i
  const int* sel;        // [rows_out] 0 = zeros, 1 = g_src, 2 = g_tgt
  const float* g_src; const float* g_tgt;   // [B][gin]
  float* out;            // [B][rows_out]
  int rows_out; int gin;
};

__global__ void __launch_bounds__(256) cond_kernel(const CondArgs a) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.y;
  if (warp >= a.rows_out) return;
  const int sel = a.sel[warp];
  float s = 0.f;
  if (sel != 0) {
    const float* g = (sel == 1 ? a.g_src : a.g_tgt) + (size_t)b * a.gin;
    const float* w = a.w + (size_t)a.w_row[warp] * a.gin;
    for (int c = lane; c < a.gin; c += 32) s = fmaf(w[c], g[c], s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  }
  if (lane == 0) a.out[(size_t)b * a.rows_out + warp] = s + a.bias[warp];
}

// ---------------------------------------------------------------------------------------------
// conv_post_kernel: y[b, t] = tanh( sum_{ci<C, k<7} w[ci,k] * lrelu_0.01(x[b, ci, t+k-3]) )
// (models.py:287-289; conv_post has no bias, models.py:266).  3.4 FLOP/B -> HBM-bound: every
// thread produces 4 consecutive samples from aligned 16-byte loads; neighbouring threads'
// halo vectors hit L1.
// ---------------------------------------------------------------------------------------------
template <int C>
__global__ void __launch_bounds__(256) conv_post_kernel(const float* __restrict__ x, long long x_bs, int x_pitch,
                                                        const float* __restrict__ w, float* __restrict__ y,
                                                        long long y_bs, int y_len, const long long* lens, int tmax,
                                                        int mul) {
  __shared__ float ws[C * 7];
  for (int i = threadIdx.x; i < C * 7; i += blockDim.x) ws[i] = w[i];
  __syncthreads();
  const int b = blockIdx.y;
  const int lim = (lens ? (int)min((long long)tmax, lens[b]) : tmax) * mul;
  const int t = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (t >= y_len) return;
  float* yp = y + (size_t)b * y_bs + t;
  if (t >= lim) {
    *reinterpret_cast<float4*>(yp) = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  const float* xb = x + (size_t)b * x_bs;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
  for (int ci = 0; ci < C; ++ci) {
    const float* xr = xb + (size_t)ci * x_pitch;
    float win[12];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const int tt = t - 4 + 4 * i;
      float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
      if (tt >= 0 && tt < lim) q = *reinterpret_cast<const float4*>(xr + tt);
      const float e[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float v = (tt + j < lim) ? e[j] : 0.f;
        win[4 * i + j] = v > 0.f ? v : 0.01f * v;
      }
    }
#pragma unroll
    for (int k = 0; k < 7; ++k) {
      const float wk = ws[ci * 7 + k];
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[j] = fmaf(wk, win[1 + k + j], acc[j]);
    }
  }
  float o[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) o[j] = (t + j < lim) ? tanhf(acc[j]) : 0.f;
  *reinterpret_cast<float4*>(yp) = make_float4(o[0], o[1], o[2], o[3]);
}

// latent copy-out: internal [B][C][pitch] -> caller [B][C][tmax], zero past the length (the
// reference returns masked latents, models.py:220 and modules.py:449,454)
__global__ void __launch_bounds__(256) copy_latent_kernel(const float* __restrict__ src, int pitch, float* __restrict__ dst,
                                                          int tmax, int C, const long long* lens) {
  const int b = blockIdx.z, c = blockIdx.y;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= tmax) return;
  const int len = (int)min((long long)tmax, lens[b]);
  const float v = t < len ? src[((size_t)b * C + c) * pitch + t] : 0.f;
  dst[((size_t)b * C + c) * tmax + t] = v;
}


// ---------------------------------------------------------------------------------------------
// stft_mag_kernel: the linear-spectrogram front end of convert (mel_processing.py:40-75):
// reflect-pad (n_fft-hop)/2 = 384 at BOTH ends of each utterance's own length, periodic hann,
// 1024-point DFT, centre=False, sqrt(re^2 + im^2 + 1e-6).  One CTA transforms 8 consecutive
// frames (radix-4 Stockham FFT in shared memory, twiddles and window from host-computed
// double-precision tables) and writes a [513][8] block so rows are stored 32 B at a time.
// Frames past an utterance's T = L / hop are written as zeros.
// ---------------------------------------------------------------------------------------------
constexpr int STFT_N = 1024, STFT_FR = 8;

// The per-CTA body both STFT kernels instantiate: columns [t0, t0 + 8) of one item, column t < T transformed from the
// samples load(t, n), n < 1024 (window applied here), columns T .. Tmax-1 written as zeros.
template <class Load>
__device__ __forceinline__ void stft_block(const Load& load, int T, int t0, float* __restrict__ sp, int spec_pitch, int Tmax,
                                           const float2* __restrict__ tw, const float* __restrict__ win) {
  __shared__ float2 buf[2][STFT_N];
  __shared__ float mag[STFT_N / 2 + 1][STFT_FR + 1];
  __shared__ float2 tws[STFT_N];
  const int tid = threadIdx.x;
  for (int i = tid; i < STFT_N; i += 256) tws[i] = tw[i];
  for (int fr = 0; fr < STFT_FR; ++fr) {
    const int t = t0 + fr;
    if (t < T) {   // block-uniform
      for (int n = tid; n < STFT_N; n += 256) buf[0][n] = make_float2(load(t, n) * win[n], 0.f);
      __syncthreads();
      int src = 0;
#pragma unroll
      for (int Ns = 1; Ns < STFT_N; Ns *= 4) {
        const float2* in = buf[src];
        float2* out = buf[src ^ 1];
        const int k = tid & (Ns - 1);
        const int j0 = ((tid - k) << 2) + k;
        const int tstep = k * (256 / Ns);
        float2 u0 = in[tid], u1 = in[tid + 256], u2 = in[tid + 512], u3 = in[tid + 768];
        const float2 w1 = tws[tstep], w2 = tws[2 * tstep], w3 = tws[3 * tstep];
        u1 = make_float2(u1.x * w1.x - u1.y * w1.y, u1.x * w1.y + u1.y * w1.x);
        u2 = make_float2(u2.x * w2.x - u2.y * w2.y, u2.x * w2.y + u2.y * w2.x);
        u3 = make_float2(u3.x * w3.x - u3.y * w3.y, u3.x * w3.y + u3.y * w3.x);
        const float2 v0 = make_float2(u0.x + u2.x, u0.y + u2.y), v1 = make_float2(u0.x - u2.x, u0.y - u2.y);
        const float2 v2 = make_float2(u1.x + u3.x, u1.y + u3.y);
        const float2 d = make_float2(u1.x - u3.x, u1.y - u3.y);
        const float2 v3 = make_float2(d.y, -d.x);   // (u1 - u3) * (-i)
        out[j0] = make_float2(v0.x + v2.x, v0.y + v2.y);
        out[j0 + Ns] = make_float2(v1.x + v3.x, v1.y + v3.y);
        out[j0 + 2 * Ns] = make_float2(v0.x - v2.x, v0.y - v2.y);
        out[j0 + 3 * Ns] = make_float2(v1.x - v3.x, v1.y - v3.y);
        src ^= 1;
        __syncthreads();
      }
      for (int f = tid; f <= STFT_N / 2; f += 256) {
        const float2 c = buf[src][f];
        mag[f][fr] = sqrtf(c.x * c.x + c.y * c.y + 1e-6f);
      }
    } else {
      for (int f = tid; f <= STFT_N / 2; f += 256) mag[f][fr] = 0.f;
    }
    __syncthreads();
  }
  for (int e = tid; e < (STFT_N / 2 + 1) * STFT_FR; e += 256) {
    const int f = e / STFT_FR, fr = e % STFT_FR;
    if (t0 + fr < Tmax) sp[(size_t)f * spec_pitch + t0 + fr] = mag[f][fr];
  }
}

__global__ void __launch_bounds__(256) stft_mag_kernel(const float* __restrict__ wav, long long wav_bs,
                                                       const long long* __restrict__ wav_len, int hop,
                                                       float* __restrict__ spec, long long spec_bs, int spec_pitch,
                                                       int Tmax, const float2* __restrict__ tw,
                                                       const float* __restrict__ win, long long* __restrict__ frames_out) {
  const int b = blockIdx.y, t0 = blockIdx.x * STFT_FR;
  const int L = (int)wav_len[b];
  const int T = min(Tmax, L / hop);
  if (blockIdx.x == 0 && threadIdx.x == 0 && frames_out) frames_out[b] = T;
  const float* w = wav + (size_t)b * wav_bs;
  const int pad = (STFT_N - hop) / 2;
  const auto load = [&](int t, int n) {
    int idx = t * hop + n - pad;
    if (idx < 0) idx = -idx;
    if (idx >= L) idx = 2 * (L - 1) - idx;
    idx = max(0, min(idx, L - 1));   // (callers guarantee L > 384; never read out of bounds regardless)
    return w[idx];
  };
  stft_block(load, T, t0, spec + (size_t)b * spec_bs, spec_pitch, Tmax, tw, win);
}

// ---------------------------------------------------------------------------------------------
// stft_ring_kernel: stft_mag_kernel's frames read straight from per-stream audio rings, so many
// live streams' window spectrograms come from one launch.  Sample s of the stream in row r lives
// at rings[r * cap + s % cap].  Item b writes frames [lo[b], lo[b] + frames[b]) of row[b] into
// columns 0 .. frames[b]-1 of spec[b] (zeros up to Tmax): the padded batch voice conversion reads.
// Frame t reads samples t*hop + n - pad; negative indices reflect at the stream start, indices
// at or past len[b] reflect at the stream end only once the stream has ended (len[b] !=
// RING_OPEN).  Per-item values are clamped, so no read leaves the rings whatever they hold.
// ---------------------------------------------------------------------------------------------
constexpr long long RING_OPEN = 0x7fffffffffffffffLL;

__global__ void __launch_bounds__(256) stft_ring_kernel(const float* __restrict__ rings, long long cap, int rows,
                                                        const long long* __restrict__ row, const long long* __restrict__ lo,
                                                        const long long* __restrict__ frames,
                                                        const long long* __restrict__ len, int hop, float* __restrict__ spec,
                                                        int Tmax, const float2* __restrict__ tw,
                                                        const float* __restrict__ win) {
  const int b = blockIdx.y, t0 = blockIdx.x * STFT_FR;
  const long long r = max(0LL, min(row[b], (long long)rows - 1));
  const long long f0 = max(0LL, min(lo[b], 1LL << 40));
  const int T = (int)max(0LL, min(frames[b], (long long)Tmax));
  const long long L = len[b] == RING_OPEN ? RING_OPEN : max(1LL, min(len[b], 1LL << 50));
  const float* ring = rings + r * cap;
  const long long pad = (STFT_N - hop) / 2;
  const auto load = [&](int t, int n) {
    long long idx = (f0 + t) * hop + n - pad;
    if (idx < 0) idx = -idx;
    if (L != RING_OPEN) {
      if (idx >= L) idx = 2 * (L - 1) - idx;
      idx = min(idx, L - 1);
    }
    return ring[max(idx, 0LL) % cap];
  };
  stft_block(load, T, t0, spec + (size_t)b * (STFT_N / 2 + 1) * Tmax, Tmax, Tmax, tw, win);
}

}  // namespace ovc
