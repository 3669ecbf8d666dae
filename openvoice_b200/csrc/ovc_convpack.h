// ovc_convpack.h -- host side of the fp32 CUDA-core conv family (ovc_conv.cuh): the packed weight layout, the row
// interleave of the paired epilogues and the polyphase tap map of the transposed convs.  The library (ovc_lib.cu) and
// the kernel harness (tests/kernelcheck/kc_f32.cu) both pack through these functions, so a test of the kernel runs on
// exactly the bytes the library uploads.  No device code.
#pragma once
#include <stddef.h>

namespace ovc {

// input channels after padding to whole ci-chunks of CI_CH (the padding rows are zero)
inline int conv_cin_pad(int cin, int CI_CH) { return (cin + CI_CH - 1) / CI_CH * CI_CH; }

// floats of one packed conv with `rows` packed output rows (a multiple of CO_T)
inline size_t conv_packed_floats(int rows, int cin, int K, int CO_T, int CI_CH) {
  return (size_t)(rows / CO_T) * conv_cin_pad(cin, CI_CH) * K * CO_T;
}

// packs W[row][ci][k] = wfun(row, ci, k) into dst as [row_tile][ci_pad][K][CO_T]: one ci-chunk of one row tile is ONE
// contiguous CI_CH * K * CO_T blob (one TMA bulk copy); channels past cin are zero
template <class WF>
inline void conv_pack_weights(float* dst, int rows, int cin, int K, int CO_T, int CI_CH, WF wfun) {
  const int row_tiles = rows / CO_T, cin_pad = conv_cin_pad(cin, CI_CH);
  for (int rt = 0; rt < row_tiles; ++rt)
    for (int ci = 0; ci < cin_pad; ++ci)
      for (int k = 0; k < K; ++k)
        for (int r = 0; r < CO_T; ++r)
          dst[(((size_t)rt * cin_pad + ci) * K + k) * CO_T + r] = ci < cin ? wfun(rt * CO_T + r, ci, k) : 0.f;
}

// packed row -> original row for the paired (tanh|sigmoid, m|logs) layouts: a thread's 8 rows
// are 4 channels of the first half followed by the same 4 channels of the second half
inline int paired_row(int p, int half) {
  const int q = p / 8, r = p % 8;
  return r < 4 ? 4 * q + r : half + 4 * q + (r - 4);
}

// ConvTranspose1d(cin -> cout, stride s, kernel kk, padding (kk - s) / 2) as a 3-tap conv cin -> s * cout:
//   out[co, s*n + ph] = sum_ci sum_m x[ci, n - m] * W[ci, co, s*m + ph + pad]
// packed row = co * s + ph; tap 0 / 1 / 2 reads x[n-1] / x[n] / x[n+1] (m = 1, 0, -1) and holds raw weight index
// kidx = s * (1 - tap) + ph + pad, or nothing (-1) outside [0, kk).  The (row, tap) pairs without a weight are the
// ones tap_is_zero<EPI_UPS8 / EPI_UPS2> (ovc_conv.cuh) skips.
inline int conv_ups_kidx(int s, int kk, int row, int tap) {
  const int pad = (kk - s) / 2, ph = row % s;
  const int kidx = s * (1 - tap) + ph + pad;
  return (kidx >= 0 && kidx < kk) ? kidx : -1;
}
// raw(ci, co, k) reads the [cin][cout][kk] weight
template <class RAW>
inline float conv_ups_weight(RAW raw, int s, int kk, int row, int ci, int tap) {
  const int kidx = conv_ups_kidx(s, kk, row, tap);
  return kidx >= 0 ? raw(ci, row / s, kidx) : 0.f;
}

}  // namespace ovc
