// g++ build of openvoice_b200/csrc/ovc_splice.h: the segment clamping, index and PCM16 rules the splice kernel applies
// to every element, run here as a plain loop so that tests/test_clone_host.py can check them against a NumPy model
// without a GPU.  TEST CODE ONLY -- it is never linked into libovc_b200.so.
#include "../../openvoice_b200/csrc/ovc_splice.h"

using namespace ovc_sp;

extern "C" {

// what splice_kernel writes, element by element
void sp_run(const float* src, long long src_rows, long long src_pitch, float* dst, long long dst_rows, long long dst_cap,
            const long long* seg, int S, int flags) {
  for (int s = 0; s < S; ++s) {
    const Seg g = load_seg((const int64_t*)seg, s, src_rows, src_pitch, dst_rows, dst_cap);
    for (int64_t i = 0; i < g.count; ++i) dst[dst_index(g, i, dst_cap)] = value(g, src, src_pitch, i, flags);
  }
}

// out5 = the clamped (src_row, src_off, count, dst_row, dst_off) of segment s
void sp_seg(const long long* seg, int s, long long src_rows, long long src_pitch, long long dst_rows, long long dst_cap,
            long long* out5) {
  const Seg g = load_seg((const int64_t*)seg, s, src_rows, src_pitch, dst_rows, dst_cap);
  const long long v[5] = {g.src_row, g.src_off, g.count, g.dst_row, g.dst_off};
  for (int i = 0; i < 5; ++i) out5[i] = v[i];
}

void sp_pcm16(const float* x, long long n, float* y) {
  for (long long i = 0; i < n; ++i) y[i] = pcm16(x[i]);
}

}  // extern "C"
