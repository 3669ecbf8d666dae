// g++ build of the ring-item rules of openvoice_b200/csrc/ovc_resample.h (ring_item, ring_in_at, ring_out_at) and a
// host loop with the semantics of resample_ring_kernel, so that tests/test_resample_ring_host.py can check them against
// NumPy and scipy without a GPU.  TEST CODE ONLY -- it is never linked into libovc_b200.so.
#include "../../openvoice_b200/csrc/ovc_resample.h"

using namespace ovc_rs;

extern "C" {

// desc7 = {plan, in_row, in_len, m0, count, out_row, out_off} -> the clamped descriptor in out7
void rr_item(const long long* desc7, int n_plans, long long in_rows, long long out_rows, long long out_cap,
             long long max_count, long long* out7) {
  const RingItem it = ring_item(desc7[0], desc7[1], desc7[2], desc7[3], desc7[4], desc7[5], desc7[6], n_plans, in_rows,
                                out_rows, out_cap, max_count);
  const long long v[7] = {it.plan, it.in_row, it.in_len, it.m0, it.count, it.out_row, it.out_off};
  for (int i = 0; i < 7; ++i) out7[i] = v[i];
}

long long rr_in_at(const long long* desc7, long long j, long long in_cap) {
  RingItem it{(int)desc7[0], desc7[1], desc7[2], desc7[3], desc7[4], desc7[5], desc7[6]};
  return ring_in_at(it, j, in_cap);
}

long long rr_out_at(const long long* desc7, long long i, long long out_cap) {
  RingItem it{(int)desc7[0], desc7[1], desc7[2], desc7[3], desc7[4], desc7[5], desc7[6]};
  return ring_out_at(it, i, out_cap);
}

// resample_ring_kernel on the host: plans from rates[2 n_plans] = {sr_in, sr_out, ...}, items desc[B][7]; each item
// is computed in tiles of `tile` outputs, each tile's span staged (as the kernel stages it) before output_at
int rr_run(int n_plans, const long long* rates, const float* in, long long in_rows, long long in_cap,
           const long long* desc, int B, float* out, long long out_rows, long long out_cap, long long max_count,
           int tile) {
  std::vector<Plan> plans(n_plans);
  std::vector<std::vector<double>> banks(n_plans);
  for (int k = 0; k < n_plans; ++k) {
    if (make_plan(rates[2 * k], rates[2 * k + 1], &plans[k]) != 0) return -1;
    banks[k] = design_bank(plans[k]);
  }
  for (int b = 0; b < B; ++b) {
    const long long* d = desc + 7 * b;
    const RingItem it = ring_item(d[0], d[1], d[2], d[3], d[4], d[5], d[6], n_plans, in_rows, out_rows, out_cap,
                                  max_count);
    const Plan& p = plans[it.plan];
    const int64_t nout = n_out(p, it.in_len);
    for (int64_t r0 = 0; r0 < it.count; r0 += tile) {
      const int64_t n = it.count - r0 < tile ? it.count - r0 : tile;
      const int64_t m0 = it.m0 + r0, mv = m0 + n < nout ? m0 + n : nout;
      int64_t s0 = 0, s1 = 0;
      if (mv > m0) span(p, m0, mv, &s0, &s1);
      std::vector<double> xs((size_t)(s1 - s0));
      for (int64_t j = s0; j < s1; ++j) {
        const int64_t k = ring_in_at(it, j, in_cap);
        xs[(size_t)(j - s0)] = k >= 0 ? in[k] : 0.f;
      }
      for (int64_t i = 0; i < n; ++i) {
        const int64_t m = m0 + i;
        out[ring_out_at(it, r0 + i, out_cap)] = m < nout ? (float)output_at(p, banks[it.plan].data(), xs.data(), s0, m) : 0.f;
      }
    }
  }
  return 0;
}

// the whole-signal one-shot loop: y[0, n_out(L)) of x[0, L), rounded to fp32 once
void rr_whole(long long sr_in, long long sr_out, const float* x, long long L, float* y) {
  Plan p;
  make_plan(sr_in, sr_out, &p);
  const std::vector<double> bank = design_bank(p);
  const int64_t n = n_out(p, L);
  if (n == 0) return;
  int64_t lo, hi;
  span(p, 0, n, &lo, &hi);
  std::vector<float> xs((size_t)(hi - lo), 0.f);
  for (int64_t j = lo < 0 ? 0 : lo; j < L && j < hi; ++j) xs[(size_t)(j - lo)] = x[j];
  for (int64_t m = 0; m < n; ++m) y[m] = (float)output_at(p, bank.data(), xs.data(), lo, m);
}

}  // extern "C"
