// Element rules of ovc_splice (include/ovc.h): copies of sample runs between device buffers, one segment per run.
// Segment s is the row seg[5 s .. 5 s + 5) = (src_row, src_off, count, dst_row, dst_off); its element i < count is
//
//   dst[dst_row * dst_cap + (dst_off + i) mod dst_cap] = f(src[src_row * src_pitch + src_off + i])   (0 if src_row < 0)
//
// with f the identity, or with PCM16 the int16 round trip of pcm16() below.  With SRC_WRAP the source is a ring too: the
// element read is src[src_row * src_pitch + (src_off + i) mod src_pitch].  load_seg clamps every descriptor value, so
// no element is read or written outside src [src_rows][src_pitch] or dst [dst_rows][dst_cap] whatever the table holds.
// The functions are OVC_HD so that the kernel and tests/hostcheck/splice_host.cpp evaluate the same expressions.
#pragma once
#include <math.h>
#include <stdint.h>

#ifndef OVC_HD
#if defined(__CUDACC__)
#define OVC_HD __host__ __device__ __forceinline__
#else
#define OVC_HD inline
#endif
#endif

namespace ovc_sp {

constexpr int PCM16 = 1;      // OVC_SPLICE_PCM16
constexpr int SRC_WRAP = 2;   // OVC_SPLICE_SRC_WRAP

struct Seg {
  int64_t src_row, src_off, count, dst_row, dst_off;
};

OVC_HD int64_t clamp64(int64_t v, int64_t lo, int64_t hi) { return v < lo ? lo : (v > hi ? hi : v); }

// Segment s, clamped: dst_row into [0, dst_rows), dst_off reduced mod dst_cap into [0, dst_cap), count into
// [0, dst_cap] (a segment never writes a ring slot twice).  A source row < 0 (or a call without source rows) is a gap
// of zeros; any other source row is clamped into [0, src_rows), src_off into [0, src_pitch], and count to the samples
// left in the source row after src_off -- or, with SRC_WRAP, src_off is reduced mod src_pitch into [0, src_pitch) and the
// count is not limited by the source (its reads wrap).
OVC_HD Seg load_seg(const int64_t* seg, int64_t s, int64_t src_rows, int64_t src_pitch, int64_t dst_rows, int64_t dst_cap,
                    int flags = 0) {
  const int64_t* v = seg + 5 * s;
  Seg g;
  g.dst_row = clamp64(v[3], 0, dst_rows - 1);
  g.dst_off = v[4] % dst_cap;
  if (g.dst_off < 0) g.dst_off += dst_cap;
  g.count = clamp64(v[2], 0, dst_cap);
  if (v[0] < 0 || src_rows < 1) {
    g.src_row = -1;
    g.src_off = 0;
  } else {
    g.src_row = v[0] < src_rows ? v[0] : src_rows - 1;
    if (flags & SRC_WRAP) {
      g.src_off = v[1] % src_pitch;
      if (g.src_off < 0) g.src_off += src_pitch;
    } else {
      g.src_off = clamp64(v[1], 0, src_pitch);
      if (g.count > src_pitch - g.src_off) g.count = src_pitch - g.src_off;
    }
  }
  return g;
}

// flat dst index of element i < g.count (dst_off < dst_cap and i < dst_cap, so one wrap at most)
OVC_HD int64_t dst_index(const Seg& g, int64_t i, int64_t dst_cap) {
  int64_t p = g.dst_off + i;
  if (p >= dst_cap) p -= dst_cap;
  return g.dst_row * dst_cap + p;
}

// The project's float -> PCM_16 -> float round trip (a float wav written as 16-bit PCM and read back, as librosa.load
// returns it): q = rint_even(fl32(x * 32767)), saturated to [-32768, 32767], then q / 32768.  NaN becomes 0.
OVC_HD float pcm16(float x) {
#if defined(__CUDA_ARCH__)
  float y = __fmul_rn(x, 32767.0f);
#else
  float y = x * 32767.0f;
#endif
  if (!(y == y)) return 0.0f;
  y = rintf(y);
  y = y < -32768.0f ? -32768.0f : (y > 32767.0f ? 32767.0f : y);
  return (float)(int)y / 32768.0f;
}

OVC_HD float value(const Seg& g, const float* src, int64_t src_pitch, int64_t i, int flags) {
  if (g.src_row < 0) return 0.0f;
  const int64_t j = (flags & SRC_WRAP) ? (g.src_off + i) % src_pitch : g.src_off + i;
  const float x = src[g.src_row * src_pitch + j];
  return (flags & PCM16) ? pcm16(x) : x;
}

#if defined(__CUDACC__)
// grid (x: element blocks, y: segments); both strided, so every element of every segment is written for any grid
__global__ void __launch_bounds__(256) splice_kernel(const float* __restrict__ src, int64_t src_rows, int64_t src_pitch,
                                                     const int64_t* __restrict__ seg, int S, float* __restrict__ dst,
                                                     int64_t dst_rows, int64_t dst_cap, int flags) {
  for (int s = blockIdx.y; s < S; s += gridDim.y) {
    const Seg g = load_seg(seg, s, src_rows, src_pitch, dst_rows, dst_cap, flags);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < g.count; i += (int64_t)gridDim.x * blockDim.x)
      dst[dst_index(g, i, dst_cap)] = value(g, src, src_pitch, i, flags);
  }
}
#endif

}  // namespace ovc_sp
