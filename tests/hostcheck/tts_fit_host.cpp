// g++ build of the duration-fit rule of openvoice_b200/csrc/ovc_tts_ops.h (the functions tts_fit_kernel and
// durations_row share), for tests/test_tts_fit_host.py.  TEST CODE ONLY -- never linked into libovc_b200.so.
#include "../../openvoice_b200/csrc/ovc_tts_ops.h"

using namespace ovc_tts;

extern "C" {

// e = expf(logw) [rows][T]
long long hc_group_frames(const float* e, const long long* lens, int T, long long r0, long long r1, float s) {
  return fit_group_frames(e, lens, T, r0, r1, s);
}

float hc_fit_scale(const float* e, const long long* lens, int T, long long r0, long long r1, long long target, float lo,
                   float hi) {
  return fit_scale(e, lens, T, r0, r1, target, lo, hi);
}

}  // extern "C"
