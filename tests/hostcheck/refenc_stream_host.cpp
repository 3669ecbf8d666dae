// Host build of the row rules of ovc_reference_encoder_stream (openvoice_b200/csrc/ovc_refenc_stream.h) for
// tests/test_refenc_stream_host.py: the same header the kernels include, compiled with g++.
#include "../../openvoice_b200/csrc/ovc_refenc_stream.h"

extern "C" {

long long re_ready(long long n, int hop, int nfft) { return ovc_re::ready(n, hop, nfft); }

long long re_limit(long long T, int l) { return ovc_re::limit(T, l); }

long long re_carry_lo(long long c) { return ovc_re::carry_lo(c); }

long long re_ws_floats(int M, int F) { return ovc_re::ws_floats(M, F); }

long long re_ws_rows(int M, int l) { return ovc_re::ws_rows(M, l); }

// W[7], carry offsets [6], h offset, floats per row
void re_geom(int F, long long* out) {
  const ovc_re::Geom g = ovc_re::geom(F);
  for (int l = 0; l <= ovc_re::LAYERS; ++l) out[l] = g.W[l];
  for (int l = 0; l < ovc_re::LAYERS; ++l) out[7 + l] = g.carry[l];
  out[13] = g.h;
  out[14] = g.floats;
}

// state_row, ring_row, c0, a1, a2, n_snap, T, tail, snap, snap_ok
void re_item(const long long* d, long long c0, long long state_rows, long long ring_rows, int max_new, int hop, int nfft,
             long long* out) {
  const int64_t dd[4] = {d[0], d[1], d[2], d[3]};
  const ovc_re::Item it = ovc_re::item(dd, c0, state_rows, ring_rows, max_new, hop, nfft);
  const long long v[10] = {it.state_row, it.ring_row, it.c0, it.a1, it.a2, it.n_snap, it.T, it.tail, it.snap, it.snap_ok};
  for (int i = 0; i < 10; ++i) out[i] = v[i];
}
}
