// Polyphase sample-rate conversion with the arithmetic of scipy.signal.resample_poly(x, up, down) at its defaults
// (window = ('kaiser', 5.0), padtype = 'constant'): the function _load_audio falls back to, and the one librosa's
// res_type='polyphase' calls.
//
//   g = gcd(sr_in, sr_out); up = sr_out / g; down = sr_in / g; M = max(up, down)
//   half = 10 M; N = 2 half + 1 taps; h = firwin(N, 1 / M, window=('kaiser', 5.0)) * up
//   pre_pad = down - half % down; pre_remove = (half + pre_pad) / down; n_out(L) = ceil(L up / down)
//   y[m] = sum_j x[j] h[t - j up],  t = (m + pre_remove) down - pre_pad,  0 <= t - j up < N
//
// Taps and accumulation are fp64 (fma, ascending j), rounded to fp32 once by the caller: that rounding equals
// float32(resample_poly(float64(x))) to within one ulp, and the sum does not depend on which samples a caller staged,
// so a windowed or streamed call gives the whole-clip result bit for bit, on the host (g++) and the device alike.
// Equal rates are the identity (one tap of 1), as resample_poly returns a copy.
//
// The design functions run on the host (the library builds one bank per rate pair and uploads it); the plan
// arithmetic and output_at are OVC_HD so that the kernel (ovc_resample.cuh) and tests/hostcheck share them.
#pragma once
#include <math.h>
#include <stdint.h>

#include <vector>

#ifndef OVC_HD
#if defined(__CUDACC__)
#define OVC_HD __host__ __device__ __forceinline__
#else
#define OVC_HD inline
#endif
#endif

namespace ovc_rs {

// Largest reduced max(up, down) accepted: every common rate from 8 kHz to 192 kHz fits (192 k <-> 22.05 k has
// M = 1280); a pair like 44 101 -> 22 050 (M = 44 101, an 882 k-tap filter) is refused.
constexpr int64_t MAX_M = 2048;
constexpr double KAISER_BETA = 5.0;
constexpr int64_t OPEN = INT64_MAX;   // length of a stream that has not ended
constexpr double PI = 3.14159265358979323846;

struct Plan {
  int64_t up = 1, down = 1;
  int64_t half = 0, taps = 1;   // filter half length and length N = 2 half + 1
  int64_t K = 1;                // taps per phase: ceil(N / up); bank is [up][K]
  int64_t pre_pad = 1, pre_remove = 1;
};

OVC_HD int64_t fdiv(int64_t a, int64_t b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }   // floor, b > 0
OVC_HD int64_t cdiv(int64_t a, int64_t b) { return -fdiv(-a, b); }                            // ceil,  b > 0

// 0 and *p filled, or -1 when a rate is not positive or the reduced max(up, down) exceeds MAX_M
OVC_HD int make_plan(int64_t sr_in, int64_t sr_out, Plan* p) {
  if (sr_in <= 0 || sr_out <= 0) return -1;
  int64_t a = sr_in, b = sr_out;
  while (b) { const int64_t r = a % b; a = b; b = r; }
  p->up = sr_out / a;
  p->down = sr_in / a;
  const int64_t M = p->up > p->down ? p->up : p->down;
  if (M > MAX_M) return -1;
  p->half = p->up == p->down ? 0 : 10 * M;
  p->taps = 2 * p->half + 1;
  p->K = (p->taps + p->up - 1) / p->up;
  p->pre_pad = p->down - p->half % p->down;
  p->pre_remove = (p->half + p->pre_pad) / p->down;
  return 0;
}

// output samples of a clip of L input samples: ceil(L up / down); OPEN for a stream that has not ended
OVC_HD int64_t n_out(const Plan& p, int64_t L) {
  if (L <= 0) return 0;
  if (L >= OPEN / (4 * MAX_M)) return OPEN;
  return (L * p.up + p.down - 1) / p.down;
}

OVC_HD int64_t t_of(const Plan& p, int64_t m) { return (m + p.pre_remove) * p.down - p.pre_pad; }

// input samples [*lo, *hi) that outputs [m0, m1) (m1 > m0) read; lo may be negative, hi may pass the clip's end:
// samples outside [0, L) are zero
OVC_HD void span(const Plan& p, int64_t m0, int64_t m1, int64_t* lo, int64_t* hi) {
  *lo = cdiv(t_of(p, m0) - p.taps + 1, p.up);
  *hi = t_of(p, m1 - 1) / p.up + 1;
}

// outputs whose support lies inside the first n_in samples: what a stream can emit before it ends
OVC_HD int64_t n_ready(const Plan& p, int64_t n_in) {
  if (n_in <= 0) return 0;
  if (n_in >= OPEN / (4 * MAX_M)) return OPEN;
  const int64_t r = fdiv(n_in * p.up - 1 + p.pre_pad, p.down) - p.pre_remove + 1;
  return r > 0 ? r : 0;
}

// y[m] in fp64.  x points at input sample x0 and must reach every sample of span(p, m, m + 1), with zeros standing
// for samples outside the clip; bank is the [up][K] layout of design_bank.  The per-output index arithmetic is 64-bit,
// the tap loop a 32-bit walk over two pointers (at most K taps, K <= 20 MAX_M + 1).
template <class T>
OVC_HD double output_at(const Plan& p, const double* bank, const T* x, int64_t x0, int64_t m) {
  const int64_t t = t_of(p, m);
  const int64_t jhi = t / p.up;
  const int64_t jlo = cdiv(t - p.taps + 1, p.up);
  const double* h = bank + (t - jhi * p.up) * p.K + (jlo - jhi + p.K - 1);   // the tap of input sample jlo
  const T* xs = x + (jlo - x0);
  const int n = (int)(jhi - jlo + 1);
  double acc = 0.0;
#if defined(__CUDACC__)
#pragma unroll 4
#endif
  for (int i = 0; i < n; ++i) acc = fma((double)xs[i], h[i], acc);
  return acc;
}

// ---- ovc_resample_rings: many streams, each with its own plan, read from ring rows and written to ring rows or packed
// buffers.  Every descriptor is clamped here, on the device, so that no index leaves `in` or `out` whatever the arrays
// hold; the same functions run in tests/hostcheck.

// first output a ring item may start at: keeps t_of(m) and the span arithmetic far from int64 overflow
constexpr int64_t MAX_POS = OPEN / (8 * MAX_M);

OVC_HD int64_t clamp64(int64_t v, int64_t lo, int64_t hi) { return v < lo ? lo : (v > hi ? hi : v); }

// v mod cap in [0, cap), cap > 0
OVC_HD int64_t wrap(int64_t v, int64_t cap) {
  const int64_t r = v % cap;
  return r < 0 ? r + cap : r;
}

// flat index of absolute sample s of a ring row: row * cap + s mod cap
OVC_HD int64_t ring_at(int64_t row, int64_t s, int64_t cap) { return row * cap + wrap(s, cap); }

struct RingItem {
  int plan;                     // plan id in [0, n_plans)
  int64_t in_row, in_len;       // input ring row and stream length (OPEN while the stream is open)
  int64_t m0, count;            // outputs [m0, m0 + count)
  int64_t out_row, out_off;     // output m goes to out[out_row * out_cap + (out_off + m - m0) mod out_cap]
};

// the clamped descriptor of one item: plan and rows into range, in_len >= 0, m0 into [0, MAX_POS], count into
// [0, max_count], out_off reduced mod out_cap (n_plans, in_rows, out_rows, out_cap >= 1; max_count >= 0)
OVC_HD RingItem ring_item(int64_t plan, int64_t in_row, int64_t in_len, int64_t m0, int64_t count, int64_t out_row,
                          int64_t out_off, int n_plans, int64_t in_rows, int64_t out_rows, int64_t out_cap,
                          int64_t max_count) {
  RingItem it;
  it.plan = (int)clamp64(plan, 0, n_plans - 1);
  it.in_row = clamp64(in_row, 0, in_rows - 1);
  it.in_len = in_len > 0 ? in_len : 0;
  it.m0 = clamp64(m0, 0, MAX_POS);
  it.count = clamp64(count, 0, max_count);
  it.out_row = clamp64(out_row, 0, out_rows - 1);
  it.out_off = wrap(out_off, out_cap);
  return it;
}

// flat index into `in` of input sample j of the item, or -1 when it reads as 0 (outside [0, in_len))
OVC_HD int64_t ring_in_at(const RingItem& it, int64_t j, int64_t in_cap) {
  return (j >= 0 && j < it.in_len) ? ring_at(it.in_row, j, in_cap) : -1;
}

// flat index into `out` of the item's i-th output (m = m0 + i), 0 <= i < count
OVC_HD int64_t ring_out_at(const RingItem& it, int64_t i, int64_t out_cap) {
  return ring_at(it.out_row, it.out_off + i, out_cap);
}

// modified Bessel function I0 by its power series sum (x^2 / 4)^k / (k!)^2
inline double bessel_i0(double x) {
  const double q = 0.25 * x * x;
  double term = 1.0, sum = 1.0;
  for (int k = 1; k < 500 && term > 1e-17 * sum; ++k) {
    term *= q / ((double)k * k);
    sum += term;
  }
  return sum;
}

// h[n], n in [0, N): firwin(N, 1 / M, window=('kaiser', 5.0)) * up
inline std::vector<double> design_filter(const Plan& p) {
  std::vector<double> h(p.taps);
  if (p.half == 0) {
    h[0] = 1.0;
    return h;
  }
  const double M = (double)(p.up > p.down ? p.up : p.down), fc = 1.0 / M, alpha = (double)p.half;
  const double i0b = bessel_i0(KAISER_BETA);
  double s = 0.0, comp = 0.0;   // Neumaier-compensated: a plain running sum of 25 k taps drifts ~1e-14 from firwin's
  for (int64_t n = 0; n < p.taps; ++n) {
    const double u = fc * (double)(n - p.half);
    const double sinc = u == 0.0 ? 1.0 : sin(PI * u) / (PI * u);
    const double r = ((double)n - alpha) / alpha;
    h[n] = fc * sinc * (bessel_i0(KAISER_BETA * sqrt(1.0 - r * r)) / i0b);
    const double t = s + h[n];
    comp += fabs(s) >= fabs(h[n]) ? (s - t) + h[n] : (h[n] - t) + s;
    s = t;
  }
  s += comp;
  for (auto& v : h) v = v / s * (double)p.up;
  return h;
}

// polyphase bank [up][K]: bank[ph][i] = h[ph + (K - 1 - i) up] (0 past N), so that output_at walks the input upward
inline std::vector<double> design_bank(const Plan& p) {
  const std::vector<double> h = design_filter(p);
  std::vector<double> bank((size_t)(p.up * p.K), 0.0);
  for (int64_t ph = 0; ph < p.up; ++ph)
    for (int64_t i = 0; i < p.K; ++i) {
      const int64_t n = ph + (p.K - 1 - i) * p.up;
      if (n < p.taps) bank[(size_t)(ph * p.K + i)] = h[(size_t)n];
    }
  return bank;
}

}  // namespace ovc_rs
