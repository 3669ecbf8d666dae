// Element functions of the V1 TTS front half (SynthesizerTrn.infer, openvoice/models.py:467-490): everything on the
// text side that is not a dense channel contraction (those run on the tensor-core conv kernel, ovc_tcconv.cuh).
//
// Text-side tensors are channels-last: [B][T][C] rows of C contiguous floats (T = padded token count); rows at or
// past an utterance's length are never read as data (the conv kernel zero-fills them, these functions test `len`),
// which is the reference's `* x_mask` (commons.sequence_mask, commons.py:121-125) without a mask tensor.
//
// Every function is plain C++ on raw pointers (OVC_HD = __host__ __device__ under nvcc, empty otherwise): the CUDA
// kernels in ovc_tts.cuh are one-thread-per-element wrappers around them, and tests/hostcheck compiles the same
// functions with g++ so that they can be checked on the CPU box without a GPU.  They do a few MFLOP per sentence (SURVEY.md
// section 8 rows a12/a13: "< 0.1 % of the decoder"), so clarity wins over speed here.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define OVC_HD __host__ __device__ __forceinline__
#else
#define OVC_HD inline
#endif

namespace ovc_tts {

constexpr int NB = 10;               // spline bins                          modules.py:466
constexpr int NP = 3 * NB - 1;       // parameters per element (10 + 10 + 9) modules.py:477
constexpr float MIN_BIN = 1e-3f;     // width / height / derivative floors   transforms.py:7-9

OVC_HD float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }   // F.gelu, modules.py:122,125

OVC_HD float softplus(float x) { return x > 20.f ? x : log1pf(expf(x)); }                       // F.softplus (threshold 20)

// ---- TextEncoder embedding: emb(tok) * sqrt(H), masked                       models.py:48-52
OVC_HD float embed_at(const long long* tokens, const float* emb, int H, float scale, int T, int b, int t, int c, int len) {
  if (t >= len) return 0.f;
  return emb[(size_t)tokens[(size_t)b * T + t] * H + c] * scale;
}

// ---- out = post(LN_C(pre(a + r))) * gamma + beta [+ res]                      modules.py:26-29
// pre: 0 none | 1 relu (DurationPredictor, models.py:92-93);  post: 0 none | 1 erf-GELU (DDSConv, modules.py:121-125)
OVC_HD void layer_norm_row(const float* a, const float* r, const float* res, const float* gamma, const float* beta, int C,
                           int pre, int post, float* out) {
  double sum = 0.0;                       // serial fp32 sums of C terms would cost ~5e-6; the rows are tiny
  for (int c = 0; c < C; ++c) {
    float v = a[c] + (r ? r[c] : 0.f);
    if (pre == 1) v = v > 0.f ? v : 0.f;
    sum += v;
  }
  const float mean = (float)(sum / C);
  double sq = 0.0;
  for (int c = 0; c < C; ++c) {
    float v = a[c] + (r ? r[c] : 0.f);
    if (pre == 1) v = v > 0.f ? v : 0.f;
    sq += (double)(v - mean) * (v - mean);
  }
  const float rstd = 1.f / sqrtf((float)(sq / C) + 1e-5f);
  for (int c = 0; c < C; ++c) {
    float v = a[c] + (r ? r[c] : 0.f);
    if (pre == 1) v = v > 0.f ? v : 0.f;
    float y = (v - mean) * rstd * gamma[c] + beta[c];
    if (post == 1) y = gelu_erf(y);
    out[c] = y + (res ? res[c] : 0.f);
  }
}

// ---- attention logits of one (query i, key j) pair of head h                  attentions.py:279-296
// qkv row layout: [q (H) | k (H) | v (H)], head h owns channels [h*dk, +dk).  rel_k [2w+1][dk] (heads share it).
OVC_HD float attn_score(const float* qkv_b, int ld, int H, int dk, int h, int i, int j, int len, const float* rel_k,
                        int window) {
  if (j >= len || i >= len) return -1e4f;                                  // masked_fill(mask == 0, -1e4)
  const float inv = 1.f / sqrtf((float)dk);
  const float* q = qkv_b + (size_t)i * ld + h * dk;
  const float* k = qkv_b + (size_t)j * ld + H + h * dk;
  float s = 0.f;
  for (int d = 0; d < dk; ++d) s += (q[d] * inv) * k[d];
  const int rel = j - i;
  if (rel >= -window && rel <= window) {
    const float* e = rel_k + (size_t)(rel + window) * dk;
    float sl = 0.f;
    for (int d = 0; d < dk; ++d) sl += (q[d] * inv) * e[d];
    s += sl;
  }
  return s;
}

// ---- softmax over keys + value mix of one output element (b, i, h, d)         attentions.py:307-323
// scores: row i of the [T][T] logits of this (b, h).  out = sum_j p_j v_j[d] + sum_{|j-i|<=w} p_j Ev[j-i+w][d]
// (keys at or past `len` carry -1e4 in the reference: exp underflows to exactly 0 in fp32, so they are skipped)
OVC_HD float attn_out(const float* scores_row, const float* qkv_b, int ld, int H, int dk, int h, int i, int d, int len,
                      const float* rel_v, int window) {
  float m = -3.4e38f;
  for (int j = 0; j < len; ++j) m = scores_row[j] > m ? scores_row[j] : m;
  float den = 0.f;
  for (int j = 0; j < len; ++j) den += expf(scores_row[j] - m);
  float acc = 0.f;
  for (int j = 0; j < len; ++j) {
    const float p = expf(scores_row[j] - m) / den;
    float v = qkv_b[(size_t)j * ld + 2 * H + h * dk + d];
    const int rel = j - i;
    if (rel >= -window && rel <= window) v += rel_v[(size_t)(rel + window) * dk + d];
    acc += p * v;
  }
  return acc;
}

// ---- dense 'same' conv, one output element, plain fp32 FMA chain               attentions.py:439-448, models.py:90-96
// The k = 3 convs of the FFN and the DurationPredictor contract over up to 3 * 768 terms; on the tensor cores the
// accumulator's truncating adds over that many terms cost far more than fp32 rounding, which the spline inverses of the
// SDP amplify into duration flips -- so these four layers stay on the CUDA cores.  w is stored [K][Cin][N] (n contiguous: a
// warp of consecutive n reads coalesced weights and one broadcast activation).  relu_in: relu on the input rows.
OVC_HD float dense_at(const float* x_b, const float* w, const float* bias, int Cin, int K, int N, int t, int n, int len,
                      int relu_in) {
  float acc = bias[n];
  const int pad = (K - 1) / 2;
  for (int k = 0; k < K; ++k) {
    const int tt = t + k - pad;
    if (tt < 0 || tt >= len) continue;
    const float* xr = x_b + (size_t)tt * Cin;
    const float* wk = w + (size_t)k * Cin * N + n;
    for (int c = 0; c < Cin; ++c) {
      float v = xr[c];
      if (relu_in) v = v > 0.f ? v : 0.f;
      acc += v * wk[(size_t)c * N];
    }
  }
  return acc;
}

// ---- DDSConv depthwise dilated conv, one output element                       modules.py:100-108,118
// x [T][C] rows (masked at len), w [C][3], 'same' padding = dilation
OVC_HD float dwconv_at(const float* x_b, const float* w, const float* bias, int C, int t, int c, int len, int dil) {
  float acc = bias[c];
  for (int k = 0; k < 3; ++k) {
    const int tt = t + (k - 1) * dil;
    if (tt >= 0 && tt < len) acc += w[c * 3 + k] * x_b[(size_t)tt * C + c];
  }
  return acc;
}

// ---- rational-quadratic spline, inverse branch, linear tails                  transforms.py:50-97, 100-176
// p[NP] = ConvFlow.proj outputs of this element: widths[NB], heights[NB] (both divided by `scale` = sqrt(filter
// channels), modules.py:497-500), derivatives[NB-1].  Identity outside [-bound, bound].
OVC_HD float rq_spline_inverse(float x, const float* p, float scale, float bound) {
  if (!(x >= -bound && x <= bound)) return x;
  float cw[NB + 1], chh[NB + 1], der[NB + 1];
  for (int pass = 0; pass < 2; ++pass) {
    const float* u = p + pass * NB;
    float* cum = pass == 0 ? cw : chh;
    float m = -3.4e38f;
    for (int i = 0; i < NB; ++i) { const float v = u[i] / scale; m = v > m ? v : m; }
    float den = 0.f;
    for (int i = 0; i < NB; ++i) den += expf(u[i] / scale - m);
    float run = 0.f;
    cum[0] = -bound;
    for (int i = 0; i < NB; ++i) {
      const float w = MIN_BIN + (1.f - MIN_BIN * NB) * (expf(u[i] / scale - m) / den);
      run += w;
      cum[i + 1] = 2.f * bound * run - bound;
    }
    cum[NB] = bound;
  }
  const float edge = 0.5397424172369522f;    // log(exp(1 - 1e-3) - 1): tails join with slope 1  (transforms.py:70-73)
  der[0] = MIN_BIN + softplus(edge);
  der[NB] = der[0];
  for (int i = 1; i < NB; ++i) der[i] = MIN_BIN + softplus(p[2 * NB + i - 1]);
  int bin = -1;                                     // searchsorted: #(x >= edge) - 1, last edge + 1e-6 (transforms.py:45-47)
  for (int i = 0; i <= NB; ++i) bin += (x >= (i == NB ? chh[NB] + 1e-6f : chh[i])) ? 1 : 0;
  bin = bin < 0 ? 0 : (bin > NB - 1 ? NB - 1 : bin);
  const float in_cw = cw[bin], in_w = cw[bin + 1] - cw[bin];
  const float in_ch = chh[bin], in_h = chh[bin + 1] - chh[bin];
  const float delta = in_h / in_w, d0 = der[bin], d1 = der[bin + 1];
  const float y = x - in_ch;
  const float s = d0 + d1 - 2.f * delta;
  const float qa = y * s + in_h * (delta - d0);
  const float qb = in_h * d0 - y * s;
  const float qc = -delta * y;
  const float root = (2.f * qc) / (-qb - sqrtf(qb * qb - 4.f * qa * qc));
  return root * in_w + in_cw;
}

// ---- ConvFlow tail, reverse, one (b, t): params = proj(h) (masked rows never get here), x1 <- spline^-1(x1)
// h_row [C]; pw [NP][C], pb [NP]                                               modules.py:488-516
OVC_HD float convflow_tail(const float* h_row, const float* pw, const float* pb, int C, float x1, float bound) {
  float p[NP];
  for (int n = 0; n < NP; ++n) p[n] = pb[n];
  for (int c = 0; c < C; ++c) {            // channel-outer: one read of h per channel, the NP weights are warp-uniform
    const float hv = h_row[c];
    for (int n = 0; n < NP; ++n) p[n] += pw[(size_t)n * C + c] * hv;
  }
  return rq_spline_inverse(x1, p, sqrtf((float)C), bound);
}

// ---- one token's frames at length scale s, from e = expf(logw)                models.py:477-478
OVC_HD float token_frames(float e, float s) { return ceilf(e * s); }

// ---- durations of one utterance (serial over tokens)                          models.py:474-481
// logw = sdp * ratio + dp * (1 - ratio);  w = exp(logw) * mask * length_scale;  w_ceil = ceil(w);
// cum[t] = inclusive prefix sum (commons.generate_path, commons.py:135);  returns y_length = max(1, sum)
OVC_HD long long durations_row(const float* logw_sdp, const float* logw_dp, float ratio, float length_scale, int T, int len,
                               float* logw, float* w_ceil, int* cum) {
  float total = 0.f;
  int run = 0;
  for (int t = 0; t < T; ++t) {
    float lw = 0.f, wc = 0.f;
    if (t < len) {
      lw = logw_sdp[t] * ratio + logw_dp[t] * (1.f - ratio);
      wc = token_frames(expf(lw), length_scale);
    }
    logw[t] = lw;
    w_ceil[t] = wc;
    total += wc;
    run += (int)wc;
    cum[t] = run;
  }
  const long long n = (long long)total;
  return n < 1 ? 1 : n;
}

// ---- duration fit (ovc_tts_encode_fit)
// A fit group is a run of rows [r0, r1) with a target of F* frames.  Its frames at scale s are
// F(s) = sum_r max(1, sum_{t < len_r} token_frames(expf(logw_r[t]), s)), durations_row's y_lengths at length_scale = s.
// The fitted scale is the smallest fp32 s in [lo, hi] with F(s) >= F*, or hi when there is none.  F is monotone
// non-decreasing in s (fp32 rounding of a product with a positive factor is monotone, and so is ceilf), and the bit
// patterns of positive floats are ordered as their values, so a bisection over the patterns in [lo, hi] finds s in
// about 25 steps.  Frames add up in integers, so the order of the sum cannot change it.
OVC_HD long long token_frames_int(float e, float s) {
  const float wc = token_frames(e, s);
  return wc < 1073741824.f ? (long long)wc : 1073741824LL;   // a NaN or a count past 2^30 saturates instead of overflowing
}

OVC_HD uint32_t fit_bits(float s) { uint32_t u; memcpy(&u, &s, sizeof u); return u; }
OVC_HD float fit_float(uint32_t u) { float s; memcpy(&s, &u, sizeof s); return s; }

struct FitSearch { uint32_t lo, hi; };   // the answer's bit pattern lies in [lo, hi]
OVC_HD FitSearch fit_begin(float scale_lo, float scale_hi) { return FitSearch{fit_bits(scale_lo), fit_bits(scale_hi)}; }
OVC_HD bool fit_done(const FitSearch& f) { return f.lo >= f.hi; }
OVC_HD float fit_probe(const FitSearch& f) { return fit_float(f.lo + (f.hi - f.lo) / 2); }
OVC_HD void fit_step(FitSearch& f, bool reached) {   // reached: F(fit_probe(f)) >= F*
  const uint32_t mid = f.lo + (f.hi - f.lo) / 2;
  if (reached) f.hi = mid; else f.lo = mid + 1;
}
OVC_HD float fit_result(const FitSearch& f) { return fit_float(f.lo); }

// F(s) of rows [r0, r1) of e = expf(logw) [rows][T], lens clamped into [0, T] (serial: the host statement of the rule)
OVC_HD long long fit_group_frames(const float* e, const long long* lens, int T, long long r0, long long r1, float s) {
  long long F = 0;
  for (long long r = r0; r < r1; ++r) {
    const int len = lens[r] < 0 ? 0 : (lens[r] > T ? T : (int)lens[r]);
    long long n = 0;
    for (int t = 0; t < len; ++t) n += token_frames_int(e[r * T + t], s);
    F += n < 1 ? 1 : n;
  }
  return F;
}

OVC_HD float fit_scale(const float* e, const long long* lens, int T, long long r0, long long r1, long long target,
                       float scale_lo, float scale_hi) {
  FitSearch f = fit_begin(scale_lo, scale_hi);
  while (!fit_done(f)) fit_step(f, fit_group_frames(e, lens, T, r0, r1, fit_probe(f)) >= target);
  return fit_result(f);
}

// ---- frame -> token: first token whose cumulative duration exceeds y          commons.py:136-141
OVC_HD int frame_token(const int* cum, int T, int y) {
  int lo = 0, hi = T - 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (cum[mid] > y) hi = mid; else lo = mid + 1;
  }
  return lo;
}

}  // namespace ovc_tts
