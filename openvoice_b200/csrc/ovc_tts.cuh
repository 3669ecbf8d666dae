// CUDA wrappers of the TTS element functions (ovc_tts_ops.h): one thread per output element / row.
// Text-side tensors are channels-last [B][T][C]; `lens` = token counts (x_lengths, models.py:467); threads at or
// past an utterance's length do nothing (the reference's x_mask).  The 1x1 channel contractions between these kernels
// (QKV / attention-out / stats projections, SDP pre / proj, DDSConv 1x1) run on the tensor-core conv (ovc_tcconv.cuh);
// the four k = 3 convs with long contractions (FFN, DurationPredictor) stay in fp32 on the CUDA cores (tts_dense_kernel).
#pragma once
#include <cuda_runtime.h>

#include "ovc_conv.cuh"
#include "ovc_tts_ops.h"

namespace ovc {

__device__ __forceinline__ int tts_len(const long long* lens, int b, int T) {
  const long long l = lens[b];
  return l < 0 ? 0 : (l > T ? T : (int)l);
}

// grid (ceil(T*H/256), B)
__global__ void tts_embed_kernel(const long long* tokens, const long long* lens, const float* emb, int n_vocab, int T, int H,
                                 float scale, float* out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (idx >= T * H) return;
  const int t = idx / H, c = idx % H;
  const int len = tts_len(lens, b, T);
  float v = 0.f;
  if (t < len) {
    long long tok = tokens[(size_t)b * T + t];
    tok = tok < 0 ? 0 : (tok >= n_vocab ? n_vocab - 1 : tok);   // ids are validated on the host; never index outside the table
    v = emb[(size_t)tok * H + c] * scale;
  }
  out[((size_t)b * T + t) * H + c] = v;
}

// grid (ceil(T/64), B), 64 threads: one row per thread
__global__ void tts_ln_kernel(const float* a, const float* r, const float* res, const float* gamma, const float* beta,
                              const long long* lens, int T, int C, int pre, int post, float* out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (t >= tts_len(lens, b, T)) return;
  const size_t o = ((size_t)b * T + t) * C;
  ovc_tts::layer_norm_row(a + o, r ? r + o : nullptr, res ? res + o : nullptr, gamma, beta, C, pre, post, out + o);
}

// Warp-per-row LayerNorm (same math as ovc_tts::layer_norm_row; lanes stride over channels, coalesced, shuffle
// reductions).  grid (ceil(T/4), B), 128 threads = 4 rows.  In-place safe (a == out, res == out).
__global__ void tts_ln_warp_kernel(const float* a, const float* r, const float* res, const float* gamma, const float* beta,
                                   const long long* lens, int T, int C, int pre, int post, float* out) {
  const int t = blockIdx.x * 4 + (threadIdx.x >> 5), b = blockIdx.y, lane = threadIdx.x & 31;
  if (t >= tts_len(lens, b, T)) return;
  const size_t o = ((size_t)b * T + t) * C;
  auto val = [&](int c) {
    float v = a[o + c] + (r ? r[o + c] : 0.f);
    if (pre == 1) v = v > 0.f ? v : 0.f;
    return v;
  };
  float sum = 0.f;
  for (int c = lane; c < C; c += 32) sum += val(c);
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, m);
  const float mean = sum / (float)C;
  float sq = 0.f;
  for (int c = lane; c < C; c += 32) { const float d = val(c) - mean; sq += d * d; }
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, m);
  const float rstd = 1.f / sqrtf(sq / (float)C + 1e-5f);
  for (int c = lane; c < C; c += 32) {
    float y = (val(c) - mean) * rstd * gamma[c] + beta[c];
    if (post == 1) y = ovc_tts::gelu_erf(y);
    out[o + c] = y + (res ? res[o + c] : 0.f);
  }
}

// Fused relative-position self-attention (attentions.py:272-324), same math as ovc_tts::attn_score / attn_out:
// one CTA = 8 queries of one (utterance, head); logits and probabilities live in shared memory.
// grid (ceil(T/8), heads, B), 128 threads, dynamic smem = (8 * T + 8 * dk) floats.  dk % 4 == 0.
constexpr int TTS_ATT_Q = 8;
__global__ void tts_attention_kernel(const float* qkv, const long long* lens, const float* rel_k, const float* rel_v, int T,
                                     int H, int heads, int window, float* out) {
  extern __shared__ float att_smem[];
  const int b = blockIdx.z, h = blockIdx.y, i0 = blockIdx.x * TTS_ATT_Q;
  const int len = tts_len(lens, b, T);
  if (i0 >= len) return;
  const int dk = H / heads, ld = 3 * H, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  float* sq = att_smem;                    // [8][dk]   queries, pre-scaled by 1/sqrt(dk)
  float* sp = att_smem + TTS_ATT_Q * dk;   // [8][T]    logits, then probabilities
  const float* base = qkv + (size_t)b * T * ld;
  const float inv = 1.f / sqrtf((float)dk);
  const int nq = min(TTS_ATT_Q, len - i0);
  for (int e = tid; e < TTS_ATT_Q * dk; e += blockDim.x) {
    const int qi = e / dk, d = e % dk;
    sq[e] = qi < nq ? base[(size_t)(i0 + qi) * ld + h * dk + d] * inv : 0.f;
  }
  __syncthreads();
  // logits: thread <- key j; the key row streams through registers four channels at a time
  for (int j = tid; j < len; j += blockDim.x) {
    const float* kr = base + (size_t)j * ld + H + h * dk;
    float acc[TTS_ATT_Q];
#pragma unroll
    for (int qi = 0; qi < TTS_ATT_Q; ++qi) acc[qi] = 0.f;
    for (int d = 0; d < dk; d += 4) {
      const float4 kv = *reinterpret_cast<const float4*>(kr + d);
#pragma unroll
      for (int qi = 0; qi < TTS_ATT_Q; ++qi) {
        const float* q = sq + qi * dk + d;
        acc[qi] += q[0] * kv.x + q[1] * kv.y + q[2] * kv.z + q[3] * kv.w;
      }
    }
#pragma unroll
    for (int qi = 0; qi < TTS_ATT_Q; ++qi) {
      const int rel = j - (i0 + qi);
      float s = acc[qi];
      if (qi < nq && rel >= -window && rel <= window) {                 // relative-key logits (attentions.py:282-291)
        const float* e = rel_k + (size_t)(rel + window) * dk;
        const float* q = sq + qi * dk;
        float sl = 0.f;
        for (int d = 0; d < dk; ++d) sl += q[d] * e[d];
        s += sl;
      }
      sp[qi * T + j] = s;
    }
  }
  __syncthreads();
  // softmax over keys: warp w owns queries 2w, 2w + 1
  for (int qi = warp * 2; qi < warp * 2 + 2; ++qi) {
    if (qi >= nq) continue;
    float* row = sp + qi * T;
    float m = -3.4e38f;
    for (int j = lane; j < len; j += 32) m = fmaxf(m, row[j]);
#pragma unroll
    for (int k = 16; k > 0; k >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, k));
    float den = 0.f;
    for (int j = lane; j < len; j += 32) { const float e = expf(row[j] - m); row[j] = e; den += e; }
#pragma unroll
    for (int k = 16; k > 0; k >>= 1) den += __shfl_xor_sync(0xffffffffu, den, k);
    const float rden = 1.f / den;
    for (int j = lane; j < len; j += 32) row[j] *= rden;
  }
  __syncthreads();
  // value mix: thread <- channel d (coalesced value rows), 8 queries at once; then the relative-value term
  for (int d = tid; d < dk; d += blockDim.x) {
    float acc[TTS_ATT_Q];
#pragma unroll
    for (int qi = 0; qi < TTS_ATT_Q; ++qi) acc[qi] = 0.f;
    const float* vcol = base + 2 * H + h * dk + d;
    for (int j = 0; j < len; ++j) {
      const float v = vcol[(size_t)j * ld];
#pragma unroll
      for (int qi = 0; qi < TTS_ATT_Q; ++qi) acc[qi] += sp[qi * T + j] * v;
    }
    for (int qi = 0; qi < nq; ++qi) {
      const int i = i0 + qi;
      float a = acc[qi];
      for (int rel = -window; rel <= window; ++rel) {
        const int j = i + rel;
        if (j >= 0 && j < len) a += sp[qi * T + j] * rel_v[(size_t)(rel + window) * dk + d];
      }
      out[((size_t)b * T + i) * H + h * dk + d] = a;
    }
  }
}

// grid (ceil(T*T/256), heads, B): scores [B][heads][T][T]
__global__ void tts_scores_kernel(const float* qkv, const long long* lens, const float* rel_k, int T, int H, int heads,
                                  int window, float* scores) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int len = tts_len(lens, b, T);
  if (idx >= T * T) return;
  const int i = idx / T, j = idx % T;
  if (i >= len || j >= len) return;
  scores[(((size_t)b * heads + h) * T + i) * T + j] =
      ovc_tts::attn_score(qkv + (size_t)b * T * 3 * H, 3 * H, H, H / heads, h, i, j, len, rel_k, window);
}

// grid (ceil(T*H/256), B): out [B][T][H]
__global__ void tts_attn_out_kernel(const float* scores, const float* qkv, const long long* lens, const float* rel_v, int T,
                                    int H, int heads, int window, float* out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (idx >= T * H) return;
  const int i = idx / H, ch = idx % H;
  const int len = tts_len(lens, b, T);
  if (i >= len) return;
  const int dk = H / heads, h = ch / dk, d = ch % dk;
  out[((size_t)b * T + i) * H + ch] = ovc_tts::attn_out(scores + (((size_t)b * heads + h) * T + i) * T, qkv + (size_t)b * T * 3 * H,
                                                          3 * H, H, dk, h, i, d, len, rel_v, window);
}

// fp32 dense 'same' conv (FFN / DurationPredictor k = 3 layers), w [K][Cin][N]      grid (ceil(T*N/256), B)
__global__ void tts_dense_kernel(const float* x, const long long* lens, const float* w, const float* bias, int T, int Cin,
                                 int K, int N, int relu_in, float* out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (idx >= T * N) return;
  const int t = idx / N, n = idx % N;
  const int len = tts_len(lens, b, T);
  if (t >= len) return;
  out[((size_t)b * T + t) * N + n] = ovc_tts::dense_at(x + (size_t)b * T * Cin, w, bias, Cin, K, N, t, n, len, relu_in);
}

// channels-last rows -> the [C][P] layout of the FFMA conv kernels (ovc_conv.cuh) and back; P = T rounded up to 4.
// grid (ceil(P/32), ceil(C/32), B), block (32, 8): 32x32 tiles through shared memory, both sides coalesced
__global__ void tts_to_ct_kernel(const float* x, const long long* lens, int T, int C, int P, float* out) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int len = tts_len(lens, b, T);
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int t = t0 + i, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (t < len && c < C) ? x[((size_t)b * T + t) * C + c] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int c = c0 + i, t = t0 + threadIdx.x;
    if (c < C && t < P) out[((size_t)b * C + c) * P + t] = tile[threadIdx.x][i];
  }
}
__global__ void tts_from_ct_kernel(const float* in, const long long* lens, int T, int C, int P, float* out) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int len = tts_len(lens, b, T);
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int c = c0 + i, t = t0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && t < len) ? in[((size_t)b * C + c) * P + t] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int t = t0 + i, c = c0 + threadIdx.x;
    if (t < len && c < C) out[((size_t)b * T + t) * C + c] = tile[threadIdx.x][i];
  }
}

// grid (ceil(T*C/256), B)
__global__ void tts_dwconv_kernel(const float* x, const long long* lens, const float* w, const float* bias, int T, int C,
                                  int dil, float* out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (idx >= T * C) return;
  const int t = idx / C, c = idx % C;
  const int len = tts_len(lens, b, T);
  if (t >= len) return;
  out[((size_t)b * T + t) * C + c] = ovc_tts::dwconv_at(x + (size_t)b * T * C, w, bias, C, t, c, len, dil);
}

// out[b][r] = bias[r] + W[r][:] . g[b][:]  (the cond 1x1 convs on [B,gin,1]; models.py:89, 139)    grid (ceil(rows/128), B)
__global__ void tts_lin_kernel(const float* g, const float* W, const float* bias, int in_dim, int rows, float* out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (r >= rows) return;
  float acc = bias[r];
  for (int i = 0; i < in_dim; ++i) acc += W[(size_t)r * in_dim + i] * g[(size_t)b * in_dim + i];
  out[(size_t)b * rows + r] = acc;
}

// Per-token conditioning of the duration predictors (models.py:89-92, 139-141 with g [B, gin, T]):
// out[b][t][r] = x[b][t][r] + (bias[r] + W[r][:] . g[b][:][t]) for t < lens[b]; in place safe (x == out).  Each sum is
// the fmaf chain of tts_lin_kernel in the same order, then the add of tts_add_rowvec_kernel, so a token whose vector
// equals the row vector gets bit-identical values.  A CTA takes 128 output rows of TTS_TOK_T tokens: g's columns are
// staged in shared memory and each weight is read once per TTS_TOK_T tokens.  g [B][in_dim][T]; dynamic smem
// in_dim * TTS_TOK_T floats.  grid (ceil(rows/128), ceil(T/TTS_TOK_T), B), 128 threads
constexpr int TTS_TOK_T = 8;
__global__ void __launch_bounds__(128) tts_cond_tok_kernel(const float* x, const float* __restrict__ g,
                                                           const float* __restrict__ W, const float* __restrict__ bias,
                                                           const long long* lens, int T, int in_dim, int rows, float* out) {
  extern __shared__ float sg[];   // [in_dim][TTS_TOK_T]
  const int r = blockIdx.x * blockDim.x + threadIdx.x, t0 = blockIdx.y * TTS_TOK_T, b = blockIdx.z;
  const int nt = min(TTS_TOK_T, tts_len(lens, b, T) - t0);
  if (nt <= 0) return;
  for (int e = threadIdx.x; e < in_dim * TTS_TOK_T; e += blockDim.x) {
    const int i = e / TTS_TOK_T, k = e % TTS_TOK_T;
    sg[e] = k < nt ? g[((size_t)b * in_dim + i) * T + t0 + k] : 0.f;
  }
  __syncthreads();
  if (r >= rows) return;
  float acc[TTS_TOK_T];
  const float b0 = bias[r];
#pragma unroll
  for (int k = 0; k < TTS_TOK_T; ++k) acc[k] = b0;
  const float* wr = W + (size_t)r * in_dim;
  for (int i = 0; i < in_dim; ++i) {
    const float w = wr[i];
#pragma unroll
    for (int k = 0; k < TTS_TOK_T; ++k) acc[k] = fmaf(w, sg[i * TTS_TOK_T + k], acc[k]);
  }
#pragma unroll
  for (int k = 0; k < TTS_TOK_T; ++k) {
    if (k < nt) {
      const size_t o = ((size_t)b * T + t0 + k) * rows + r;
      out[o] = x[o] + acc[k];
    }
  }
}

// emb_g(sid)                                                                     models.py:470        grid (ceil(dim/128), B)
__global__ void tts_speaker_kernel(const float* table, const long long* sid, int n_rows, int dim, float* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (i >= dim) return;
  long long s = sid[b];
  s = s < 0 ? 0 : (s >= n_rows ? n_rows - 1 : s);
  out[(size_t)b * dim + i] = table[(size_t)s * dim + i];
}

// out = x + v[b]                                                                 grid (ceil(T*C/256), B)
__global__ void tts_add_rowvec_kernel(const float* x, const float* v, const long long* lens, int T, int C, float* out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (idx >= T * C) return;
  if (idx / C >= tts_len(lens, b, T)) return;
  out[(size_t)b * T * C + idx] = x[(size_t)b * T * C + idx] + v[(size_t)b * C + idx % C];
}

// ConvFlow.pre (1 -> C, 1x1) + conditioning: h = z0 * w + bias + g               modules.py:486-487, 116-117
__global__ void tts_cf_pre_kernel(const float* z0, const float* w, const float* bias, const float* g, const long long* lens,
                                  int T, int C, float* out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (idx >= T * C) return;
  const int t = idx / C, c = idx % C;
  if (t >= tts_len(lens, b, T)) return;
  const size_t o = (size_t)b * T * C + idx;
  out[o] = z0[(size_t)b * T + t] * w[c] + bias[c] + g[o];
}

// ConvFlow tail: proj (C -> 29) + inverse spline on z1, in place                 grid (ceil(T/64), B)
__global__ void tts_cf_tail_kernel(const float* h, const long long* lens, const float* pw, const float* pb, float* z1, int T,
                                   int C, float bound) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (t >= tts_len(lens, b, T)) return;
  const size_t o = (size_t)b * T + t;
  z1[o] = ovc_tts::convflow_tail(h + o * C, pw, pb, C, z1[o], bound);
}

// z = noise_w * noise_scale_w (explicit) or Philox normals                       models.py:173        grid (ceil(T/128), B)
// it.seed / it.stream / it.noise_scale_w, when set, replace the call's seed, stream b and scale for item b
__global__ void tts_noise_w_kernel(const float* noise_w, unsigned long long seed, float scale, int T, float* z0, float* z1,
                                   ItemParams it) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (t >= T) return;
  const size_t o = (size_t)b * T + t;
  if (it.seed) seed = it.seed[b];
  const uint32_t stream = it.stream ? (uint32_t)it.stream[b] : (uint32_t)b;
  if (it.noise_scale_w) scale = it.noise_scale_w[b];
  z0[o] = (noise_w ? noise_w[((size_t)b * 2 + 0) * T + t] : philox_normal(seed, stream, 0x7700u, (uint32_t)t)) * scale;
  z1[o] = (noise_w ? noise_w[((size_t)b * 2 + 1) * T + t] : philox_normal(seed, stream, 0x7701u, (uint32_t)t)) * scale;
}

// DurationPredictor.proj (C -> 1) or ElementwiseAffine^-1 on the SDP output      models.py:99, modules.py:398-399
// mode 0: out = bias + w . x_row;  mode 1: out = (z - m) * exp(-logs)  (w = {m, logs})
__global__ void tts_logw_kernel(const float* x, const long long* lens, const float* w, const float* bias, int T, int C,
                                int mode, float* out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (t >= T) return;
  const size_t o = (size_t)b * T + t;
  if (t >= tts_len(lens, b, T)) { out[o] = 0.f; return; }
  if (mode == 1) { out[o] = (x[o] - w[0]) * expf(-w[1]); return; }
  float acc = bias[0];
  for (int c = 0; c < C; ++c) acc += w[c] * x[o * C + c];
  out[o] = acc;
}

// one thread per utterance; it.sdp_ratio / it.length_scale, when set, replace the call's values  models.py:474-481
__global__ void tts_durations_kernel(const float* logw_sdp, const float* logw_dp, const long long* lens, float ratio,
                                     float length_scale, int B, int T, float* logw, float* w_ceil, int* cum,
                                     long long* y_len, ItemParams it) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const size_t o = (size_t)b * T;
  if (it.sdp_ratio) ratio = it.sdp_ratio[b];
  if (it.length_scale) length_scale = it.length_scale[b];
  y_len[b] = ovc_tts::durations_row(logw_sdp + o, logw_dp + o, ratio, length_scale, T, tts_len(lens, b, T), logw + o, w_ceil + o,
                                    cum + o);
}

// Fit groups of ovc_tts_encode_fit (include/ovc.h: ovc_tts_fit), all device arrays
struct TtsFit {
  const long long* row0;     // [G] first row of group g
  const long long* row1;     // [G] one past its last row
  const long long* target;   // [G] frames
  int G;
  float lo, hi;              // the scale range
  float* scale;              // [B] out: every row's length scale
};

// CTA g fits group g (ovc_tts::fit_* on the logw tts_durations_kernel wrote) and writes its scale to the group's rows;
// it also writes the unfitted rows between the previous group and this one (and the last CTA those after every
// group) with the scale they have without a fit.  Row ranges are clamped into [0, B), each to start at or after the
// previous group's end, so no two groups share a row; targets below 1 count as 1.  Warp w sums rows r0 + w, r0 + w + 8,
// ... with its lanes striding over the row's tokens, so a row may be longer than the CTA.  grid (G), 256 threads
constexpr int TTS_FIT_THREADS = 256;
__global__ void __launch_bounds__(TTS_FIT_THREADS) tts_fit_kernel(const float* __restrict__ logw, const long long* lens, int B,
                                                                  int T, TtsFit fit, float length_scale,
                                                                  const float* it_length_scale) {
  __shared__ long long s_part[TTS_FIT_THREADS / 32];
  __shared__ long long s_total;
  const int g = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  long long prev_end = 0, r0 = 0, r1 = 0;
  for (int k = 0; k <= g; ++k) {
    prev_end = r1;
    r0 = min(max(fit.row0[k], prev_end), (long long)B);
    r1 = min(max(fit.row1[k], r0), (long long)B);
  }
  for (long long b = prev_end + threadIdx.x; b < r0; b += blockDim.x)
    fit.scale[b] = it_length_scale ? it_length_scale[b] : length_scale;
  if (g == fit.G - 1)
    for (long long b = r1 + threadIdx.x; b < B; b += blockDim.x) fit.scale[b] = it_length_scale ? it_length_scale[b] : length_scale;
  const long long target = max(fit.target[g], 1LL);
  ovc_tts::FitSearch f = ovc_tts::fit_begin(fit.lo, fit.hi);
  while (!ovc_tts::fit_done(f)) {                    // f is the same in every thread: the loop is CTA-uniform
    const float s = ovc_tts::fit_probe(f);
    long long acc = 0;
    for (long long r = r0 + warp; r < r1; r += TTS_FIT_THREADS / 32) {
      const int len = tts_len(lens, (int)r, T);
      const float* lw = logw + r * T;
      long long n = 0;
      for (int t = lane; t < len; t += 32) n += ovc_tts::token_frames_int(expf(lw[t]), s);
#pragma unroll
      for (int m = 16; m > 0; m >>= 1) n += __shfl_xor_sync(0xffffffffu, n, m);
      acc += n < 1 ? 1 : n;
    }
    if (lane == 0) s_part[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      long long tot = 0;
      for (int w = 0; w < TTS_FIT_THREADS / 32; ++w) tot += s_part[w];
      s_total = tot;
    }
    __syncthreads();
    ovc_tts::fit_step(f, s_total >= target);
    __syncthreads();                                 // s_part / s_total are rewritten by the next step
  }
  const float s = ovc_tts::fit_result(f);
  for (long long b = r0 + threadIdx.x; b < r1; b += blockDim.x) fit.scale[b] = s;
}

// Windows of ovc_tts_decode_windows: output row w expands encoded row row[w] at absolute frames frame0[w] + t,
// t < len[w].  Every pointer NULL: output row b is encoded row b from frame 0 (the whole decode).
struct TtsWindows {
  const long long* row;      // [W], clamped into [0, N)
  const long long* frame0;   // [W]
  const long long* len;      // [W]
  int N;                     // encoded rows
};

// z_p[b][c][y] = m_p[tok(y)][c] + noise * exp(logs_p[tok(y)][c]) * noise_scale   models.py:484-487
// stats [B][T][2C] (m | logs), z_p [B][C][P]; frames at or past y_len are zero.  grid (ceil(Ty/128), C, B)
// it.seed / it.stream / it.noise_scale, when set, replace the call's seed, stream b and noise_scale for item b.
// With windows, row b reads encoded row r = row[b] at frame f = frame0[b] + y (token, Philox counter and y_len all
// at f) and is zero at or past len[b]; an explicit noise tensor is indexed by the output column y.
__global__ void tts_expand_kernel(const float* stats, const int* cum, const long long* y_len, const float* noise,
                                  long long noise_bs, int noise_pitch, unsigned long long seed, float noise_scale, int T,
                                  int C, int Ty, int P, float* z_p, ItemParams it, TtsWindows win) {
  const int y = blockIdx.x * blockDim.x + threadIdx.x, c = blockIdx.y, b = blockIdx.z;
  if (y >= P) return;
  const long long r = win.row ? min(max(win.row[b], 0LL), (long long)win.N - 1) : (long long)b;
  const long long f = win.frame0 ? win.frame0[b] + y : (long long)y;
  float v = 0.f;
  if (y < Ty && f >= 0 && f < y_len[r] && (!win.len || y < win.len[b])) {
    const int j = ovc_tts::frame_token(cum + (size_t)r * T, T, (int)f);
    const float* s = stats + ((size_t)r * T + j) * 2 * C;
    if (it.seed) seed = it.seed[b];
    const uint32_t stream = it.stream ? (uint32_t)it.stream[b] : (uint32_t)b;
    if (it.noise_scale) noise_scale = it.noise_scale[b];
    const float nz = noise ? noise[(size_t)b * noise_bs + (size_t)c * noise_pitch + y]
                           : philox_normal(seed, stream, (uint32_t)c, (uint32_t)f);
    v = s[c] + nz * expf(s[C + c]) * noise_scale;
  }
  z_p[((size_t)b * C + c) * P + y] = v;
}

// Per-window inputs of the flow and generator (ovc_tts_decode_windows): g_out[w] = g[row[w]], and lens[w] = the
// frames of window w that lie inside its row, clamp(min(len[w], y_len[row[w]] - frame0[w]), 0, Tmax).  grid (W), 128
__global__ void tts_window_rows_kernel(const float* g, const long long* y_len, int gin, TtsWindows win, int Tmax,
                                       float* g_out, long long* lens) {
  const int w = blockIdx.x;
  const long long r = min(max(win.row[w], 0LL), (long long)win.N - 1);
  for (int i = threadIdx.x; i < gin; i += blockDim.x) g_out[(size_t)w * gin + i] = g[(size_t)r * gin + i];
  if (threadIdx.x == 0) {
    const long long n = min(win.len[w], y_len[r] - win.frame0[w]);
    lens[w] = n < 0 ? 0 : (n > Tmax ? Tmax : n);
  }
}

// Per-token speaker vectors along the alignment path, as tts_expand_kernel expands m_p: g_out[b][i][y] = g[r][i][tok(f)]
// for frames f = frame0[b] + y the expansion fills (inside the row, below len[b]), 0 elsewhere.  g [N][gin][T] (the
// per-token encode's layout), g_out [B][gin][Ty].  One thread per frame finds its token once and writes every channel.
// grid (ceil(Ty/128), B), 128 threads
__global__ void tts_expand_g_kernel(const float* __restrict__ g, const int* __restrict__ cum, const long long* y_len, int T,
                                    int gin, int Ty, float* __restrict__ g_out, TtsWindows win) {
  const int y = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (y >= Ty) return;
  const long long r = win.row ? min(max(win.row[b], 0LL), (long long)win.N - 1) : (long long)b;
  const long long f = win.frame0 ? win.frame0[b] + y : (long long)y;
  float* dst = g_out + (size_t)b * gin * Ty + y;
  if (f >= 0 && f < y_len[r] && (!win.len || y < win.len[b])) {
    const int j = ovc_tts::frame_token(cum + (size_t)r * T, T, (int)f);
    const float* src = g + (size_t)r * gin * T + j;
    for (int i = 0; i < gin; ++i) dst[(size_t)i * Ty] = src[(size_t)i * T];
  } else {
    for (int i = 0; i < gin; ++i) dst[(size_t)i * Ty] = 0.f;
  }
}

// Encoded rows -> rows of a state pool (ovc_tts_encode_state_rows / ovc_tts_state_rows): source row b (B rows of T tokens)
// goes to pool row dst_row[b], clamped into [0, N), at token pitch Tp >= T.  Tokens T <= t < Tp get the padding a short
// row gets inside an encode: cum keeps its last value (durations_row), stats are 0.  One item per element of the
// destination row: Tp * C2 stats, Tp cum, gin g, one y_length.  grid (x: element blocks, y: rows), both strided.
__global__ void __launch_bounds__(256) tts_state_rows_kernel(const float* __restrict__ stats, const int* __restrict__ cum,
                                                             const float* __restrict__ g, const long long* __restrict__ y_len,
                                                             int B, int T, int C2, int gin, const long long* __restrict__ dst_row,
                                                             int N, int Tp, float* __restrict__ d_stats, int* __restrict__ d_cum,
                                                             float* __restrict__ d_g, long long* __restrict__ d_ylen) {
  const long long n_stats = (long long)Tp * C2, per_row = n_stats + Tp + gin + 1;
  for (int b = blockIdx.y; b < B; b += gridDim.y) {
    const long long r = min(max(dst_row[b], 0LL), (long long)N - 1);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < per_row; i += (long long)gridDim.x * blockDim.x) {
      if (i < n_stats) {
        const int t = (int)(i / C2), c = (int)(i - (long long)t * C2);
        d_stats[r * n_stats + i] = t < T ? stats[((size_t)b * T + t) * C2 + c] : 0.f;
      } else if (i < n_stats + Tp) {
        const int t = (int)(i - n_stats);
        d_cum[r * Tp + t] = cum[(size_t)b * T + min(t, T - 1)];
      } else if (i < n_stats + Tp + gin) {
        const int k = (int)(i - n_stats - Tp);
        d_g[r * gin + k] = g[(size_t)b * gin + k];
      } else {
        d_ylen[r] = y_len[b];
      }
    }
  }
}

// The per-token speaker vectors of encoded rows -> rows of a per-token state pool (ovc_tts_encode_state_rows_tokens /
// ovc_tts_state_rows_tokens): g [B][gin][T] -> d_g[dst_row[b]][gin][Tp], dst_row clamped into [0, N); tokens
// T <= t < Tp get 0, as the stats there.  The rest of each row is written by tts_state_rows_kernel.
// grid (x: element blocks, y: rows), both strided; 256 threads
__global__ void __launch_bounds__(256) tts_state_rows_g_kernel(const float* __restrict__ g, int B, int T, int gin,
                                                               const long long* __restrict__ dst_row, int N, int Tp,
                                                               float* __restrict__ d_g) {
  const long long per_row = (long long)gin * Tp;
  for (int b = blockIdx.y; b < B; b += gridDim.y) {
    const long long r = min(max(dst_row[b], 0LL), (long long)N - 1);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < per_row; i += (long long)gridDim.x * blockDim.x) {
      const int c = (int)(i / Tp), t = (int)(i - (long long)c * Tp);
      d_g[r * per_row + i] = t < T ? g[((size_t)b * gin + c) * T + t] : 0.f;
    }
  }
}

// out[c][t] = philox_normal(seed, stream, c0 + c, frame0 + t): the draws the kernels above make, as a tensor
// (ovc_philox_normals).  grid (ceil(T/128), C)
__global__ void philox_normals_kernel(unsigned long long seed, uint32_t stream, uint32_t c0, uint32_t frame0, int T,
                                      float* out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x, c = blockIdx.y;
  if (t >= T) return;
  out[(size_t)c * T + t] = philox_normal(seed, stream, c0 + (uint32_t)c, frame0 + (uint32_t)t);
}

}  // namespace ovc
