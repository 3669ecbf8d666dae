// g++ build of openvoice_b200/csrc/ovc_resample.h: the plan, filter bank, span and per-output functions the resample
// kernel calls, exposed so that tests/test_resample_host.py can check them against scipy without a GPU.  TEST CODE
// ONLY -- it is never linked into libovc_b200.so.
#include "../../openvoice_b200/csrc/ovc_resample.h"

using namespace ovc_rs;

extern "C" {

// out7 = {up, down, taps, K, half, pre_pad, pre_remove}; returns make_plan's status
int rs_plan(long long sr_in, long long sr_out, long long* out7) {
  Plan p;
  const int rc = make_plan(sr_in, sr_out, &p);
  if (rc == 0) {
    const long long v[7] = {p.up, p.down, p.taps, p.K, p.half, p.pre_pad, p.pre_remove};
    for (int i = 0; i < 7; ++i) out7[i] = v[i];
  }
  return rc;
}

void rs_filter(long long sr_in, long long sr_out, double* h) {
  Plan p;
  make_plan(sr_in, sr_out, &p);
  const std::vector<double> v = design_filter(p);
  for (size_t i = 0; i < v.size(); ++i) h[i] = v[i];
}

void rs_bank(long long sr_in, long long sr_out, double* bank) {
  Plan p;
  make_plan(sr_in, sr_out, &p);
  const std::vector<double> v = design_bank(p);
  for (size_t i = 0; i < v.size(); ++i) bank[i] = v[i];
}

long long rs_n_out(long long sr_in, long long sr_out, long long L) {
  Plan p;
  make_plan(sr_in, sr_out, &p);
  return n_out(p, L);
}

long long rs_n_ready(long long sr_in, long long sr_out, long long n_in) {
  Plan p;
  make_plan(sr_in, sr_out, &p);
  return n_ready(p, n_in);
}

void rs_span(long long sr_in, long long sr_out, long long m0, long long m1, long long* lohi) {
  Plan p;
  make_plan(sr_in, sr_out, &p);
  int64_t lo, hi;
  span(p, m0, m1, &lo, &hi);
  lohi[0] = lo;
  lohi[1] = hi;
}

// y[0, n_out(L)) of x[0, L) in fp64, one output_at call per sample
void rs_run(long long sr_in, long long sr_out, const float* x, long long L, double* y) {
  Plan p;
  make_plan(sr_in, sr_out, &p);
  const std::vector<double> bank = design_bank(p);
  const int64_t n = n_out(p, L);
  if (n == 0) return;
  int64_t lo, hi;                               // zero-padded copy of x covering the support of every output
  span(p, 0, n, &lo, &hi);
  std::vector<float> xs((size_t)(hi - lo), 0.f);
  for (int64_t j = lo < 0 ? 0 : lo; j < L && j < hi; ++j) xs[(size_t)(j - lo)] = x[j];
  for (int64_t m = 0; m < n; ++m) y[m] = output_at(p, bank.data(), xs.data(), lo, m);
}

}  // extern "C"
