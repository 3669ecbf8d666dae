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
// epilogues add a single per-(batch,row) vector.
//
// Frames: an embedding may vary over time (reference: sid_src / sid_tgt of shape [B, gin, T]).
// Side s of item b at frame f is g_s[b * bs + c * cs + f * fs] (fs = 0: one embedding per item),
// and output column i of frame f goes to out[b * out_bs + f * out_fs + i].  A per-item call is the
// one-frame case.  Every (frame, row) output is the same arithmetic whatever the call: lane l
// accumulates fmaf over c = l, l + 32, ... from 0, then the 32 partials are summed by the xor
// butterfly, plus the bias -- so a frame whose embedding equals a per-item one gets the bit-identical
// vector.  A warp holds the 8 weights per lane of COND_RW rows in registers and sweeps the CTA's
// frames, staged COND_FT at a time in shared memory; its COND_RW x COND_FW partial sums are reduced
// in one transposed butterfly (each step exchanges half of the remaining values, lane l ends with
// sum l, and every sum gets the additions of the plain xor tree, in the same pairing).
// ---------------------------------------------------------------------------------------------
constexpr int COND_GIN_MAX = 256;   // 8 weights per lane and row
constexpr int COND_RW = 4, COND_FW = 8;   // COND_RW * COND_FW == 32 sums per butterfly
constexpr int COND_ROWS = 8 * COND_RW;    // output columns of one CTA (8 warps); each CTA reads one side
constexpr int COND_FT = 32;               // frames staged per pass
constexpr int COND_FCHUNK = 256;          // frames of one CTA (blockIdx.z)
static_assert(COND_RW * COND_FW == 32, "one butterfly reduces 32 sums");

struct CondArgs {
  const float* w;        // [rows_w][gin]
  const float* bias;     // [rows] of the stacked list
  const int* w_row;      // [rows] matrix row feeding stacked row i
  const int* sel;        // [rows] 0 = zeros, 1 = g_src, 2 = g_tgt; uniform over aligned blocks of COND_ROWS outputs
  const int* cols;       // [n_out] stacked row of output column i; NULL = identity
  const float* g_src; const float* g_tgt;   // a NULL side reads as zeros (the caller does not use its columns)
  long long src_bs, src_cs, src_fs, tgt_bs, tgt_cs, tgt_fs;
  float* out; long long out_bs, out_fs;
  int n_out; int gin; int frames;
};

// one step of the transposed butterfly: of the 2H sums a lane holds, it keeps half (the upper half when lane bit H is
// set) and adds its xor-H partner's partial of each kept sum
template <int H>
__device__ __forceinline__ void cond_fold(float (&acc)[32], int lane) {
  const bool up = lane & H;
#pragma unroll
  for (int p = 0; p < H; ++p) {
    const float got = __shfl_xor_sync(0xffffffffu, up ? acc[p] : acc[p + H], H);
    acc[p] = (up ? acc[p + H] : acc[p]) + got;
  }
}

__global__ void __launch_bounds__(256) cond_kernel(const CondArgs a) {
  __shared__ float gsm[COND_FT][COND_GIN_MAX + 1];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.y;
  const int i_blk = blockIdx.x * COND_ROWS;
  const int i0 = i_blk + warp * COND_RW;
  const int sel = a.sel[a.cols ? a.cols[i_blk] : i_blk];   // block-uniform (host-checked)
  const float* g = sel == 1 ? a.g_src : sel == 2 ? a.g_tgt : nullptr;
  const bool live = g != nullptr;                           // block-uniform
  const long long gcs = sel == 1 ? a.src_cs : a.tgt_cs, gfs = sel == 1 ? a.src_fs : a.tgt_fs;
  if (live) g += (size_t)b * (sel == 1 ? a.src_bs : a.tgt_bs);
  float w[COND_RW][COND_GIN_MAX / 32];
#pragma unroll
  for (int r = 0; r < COND_RW; ++r) {
    const int i = min(i0 + r, a.n_out - 1);
    const float* wr = a.w + (size_t)a.w_row[a.cols ? a.cols[i] : i] * a.gin;
#pragma unroll
    for (int k = 0; k < COND_GIN_MAX / 32; ++k) w[r][k] = (live && lane + 32 * k < a.gin) ? wr[lane + 32 * k] : 0.f;
  }
  const int fz0 = blockIdx.z * COND_FCHUNK, fz1 = min(a.frames, fz0 + COND_FCHUNK);
  for (int f0 = fz0; f0 < fz1; f0 += COND_FT) {
    const int nf = min(COND_FT, fz1 - f0);
    const int nfp = (nf + COND_FW - 1) / COND_FW * COND_FW;
    __syncthreads();
    if (live)
      for (int e = threadIdx.x; e < nfp * a.gin; e += blockDim.x) {
        const int c = e / nfp, f = e % nfp;   // consecutive threads: consecutive frames of one channel
        gsm[f][c] = f < nf ? g[(size_t)c * gcs + (size_t)(f0 + f) * gfs] : 0.f;
      }
    __syncthreads();
    for (int fb = 0; fb < nf; fb += COND_FW) {
      float acc[32];   // sum r * COND_FW + f
#pragma unroll
      for (int r = 0; r < COND_RW; ++r)
#pragma unroll
        for (int f = 0; f < COND_FW; ++f) {
          float s = 0.f;
#pragma unroll
          for (int k = 0; k < COND_GIN_MAX / 32; ++k)
            if (live && lane + 32 * k < a.gin) s = fmaf(w[r][k], gsm[fb + f][lane + 32 * k], s);
          acc[r * COND_FW + f] = s;
        }
      cond_fold<16>(acc, lane);
      cond_fold<8>(acc, lane);
      cond_fold<4>(acc, lane);
      cond_fold<2>(acc, lane);
      cond_fold<1>(acc, lane);
      const int i = i0 + lane / COND_FW, f = f0 + fb + lane % COND_FW;
      if (i < a.n_out && f < f0 + nf)
        a.out[(size_t)b * a.out_bs + (size_t)f * a.out_fs + i] = acc[0] + a.bias[a.cols ? a.cols[i] : i];
    }
  }
}

// ---------------------------------------------------------------------------------------------
// tone_track_kernel: per-frame embeddings from keyframe tracks.  Track b has keys [key0[b], key0[b] + nkeys[b]) of
// (key_frame, key_se [gin]); out[b][c][t] = g_b(frame0[b] + t) for t < frames[b], zeros up to Tmax, where
//   g(t) = se_0 before the first key, se_last from the last key on, and
//   se_k + ((t - f_k) / (f_{k+1} - f_k)) * (se_{k+1} - se_k) for f_k <= t < f_{k+1}
// in fp32 with every operation rounded on its own (no contraction), so a host statement of the rule reproduces it
// bit for bit; of two keys at the same frame the later one holds from that frame on.  Descriptors are clamped here, so
// no read leaves the key arrays whatever they hold.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float tone_track_at(const long long* kf, const float* kse, int n, int gin, int c, long long t) {
  int lo = 0, hi = n;   // first key with frame > t
  while (lo < hi) {
    const int m = (lo + hi) >> 1;
    if (kf[m] <= t) lo = m + 1; else hi = m;
  }
  if (lo == 0) return kse[c];
  if (lo == n) return kse[(size_t)(n - 1) * gin + c];
  const long long f0 = kf[lo - 1], f1 = kf[lo];
  const float a = kse[(size_t)(lo - 1) * gin + c], d = __fsub_rn(kse[(size_t)lo * gin + c], a);
  const float u = __fdiv_rn((float)(t - f0), (float)(f1 - f0));
  return __fadd_rn(a, __fmul_rn(u, d));
}

__global__ void __launch_bounds__(256) tone_track_kernel(const long long* __restrict__ key_frame,
                                                         const float* __restrict__ key_se, long long n_keys,
                                                         const long long* __restrict__ key0,
                                                         const long long* __restrict__ nkeys,
                                                         const long long* __restrict__ frame0,
                                                         const long long* __restrict__ frames, int gin, int Tmax,
                                                         float* __restrict__ out) {
  const int b = blockIdx.z, c = blockIdx.y;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= Tmax || n_keys < 1) return;
  const long long k0 = max(0LL, min(key0[b], n_keys - 1));
  const int n = (int)max(1LL, min(nkeys[b], n_keys - k0));
  const long long T = max(0LL, min(frames[b], (long long)Tmax));
  const long long at = max(0LL, min(frame0[b], 1LL << 40)) + t;
  out[((size_t)b * gin + c) * Tmax + t] = t < T ? tone_track_at(key_frame + k0, key_se + (size_t)k0 * gin, n, gin, c, at) : 0.f;
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

// latent copy-in, the inverse: caller [B][C][tmax] -> internal [B][C][pitch] (pitch >= tmax), zero from the length on,
// so the generator reads a caller's z_hat exactly as it reads the one the flow left in the workspace
__global__ void __launch_bounds__(256) latent_in_kernel(const float* __restrict__ src, int tmax, float* __restrict__ dst,
                                                        int pitch, int C, const long long* lens) {
  const int b = blockIdx.z, c = blockIdx.y;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= pitch) return;
  const int len = (int)max(0LL, min((long long)tmax, lens[b]));
  dst[((size_t)b * C + c) * pitch + t] = t < len ? src[((size_t)b * C + c) * tmax + t] : 0.f;
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

// sample n of frame t of the stream in `ring` (cap samples), L samples long (RING_OPEN: not ended)
__device__ __forceinline__ float ring_frame_sample(const float* __restrict__ ring, long long cap, long long L, long long t,
                                                   int n, int hop) {
  const long long pad = (STFT_N - hop) / 2;
  long long idx = t * hop + n - pad;
  if (idx < 0) idx = -idx;
  if (L != RING_OPEN) {
    if (idx >= L) idx = 2 * (L - 1) - idx;
    idx = min(idx, L - 1);
  }
  return ring[max(idx, 0LL) % cap];
}

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
  const auto load = [&](int t, int n) { return ring_frame_sample(ring, cap, L, f0 + t, n, hop); };
  stft_block(load, T, t0, spec + (size_t)b * (STFT_N / 2 + 1) * Tmax, Tmax, Tmax, tw, win);
}

}  // namespace ovc
