// Row rules of ovc_reference_encoder_stream (include/ovc.h): the ReferenceEncoder advanced with a live stream.
//
// A stream's state row holds c0, the spectrogram frames consumed so far, the GRU hidden state h, and for each of the
// six conv inputs (the LayerNorm output and conv1..conv5 outputs) its carry: the rows the next output rows still read.
// Frame t is final at n samples once its STFT support has arrived (ready()).  Layer l (input of conv l) has
// c_l = c0 >> l final rows: output row ho of a stride-2 conv reads input rows 2ho-1 .. 2ho+1, so c final inputs give
// c >> 1 final outputs, and the GRU has run c0 >> 6 steps.  The next output row reads input rows from 2 c_{l+1} - 1 on,
// which is c_l - 1 or c_l - 2: the carry keeps rows [max(0, c_l - 2), c_l) in slot row & 1.
//
// The snapshot of a prefix of n samples is ovc_reference_encoder_ragged on those n samples alone: T = n / hop frames,
// limits limit_0 = T, limit_{l+1} = (limit_l - 1) / 2 + 1.  Its rows below c_l are the stream's final rows; rows
// [c_l, limit_l) (at most two per layer) are the tail, computed from the carry and the tail rows of the layer below
// with the taps at or past limit_l skipped, exactly as refenc_conv_kernel skips them.
//
// The functions are OVC_HD so that the kernels and tests/hostcheck/refenc_stream_host.cpp evaluate the same expressions.
#pragma once
#include <stdint.h>

#ifndef OVC_HD
#if defined(__CUDACC__)
#define OVC_HD __host__ __device__ __forceinline__
#else
#define OVC_HD inline
#endif
#endif

namespace ovc_re {

constexpr int LAYERS = 6;
constexpr int HID = 128;           // GRU hidden size
constexpr int HEADER = 4;          // state row header: c0 as an int64 in floats [0, 2); the rest 0
constexpr int TAIL = 2;            // most tail rows of a snapshot at any layer (and GRU tail steps)
constexpr int64_t MAX_SAMPLES = int64_t(1) << 50;   // sample positions a descriptor is clamped to
constexpr int64_t MAX_FRAMES = int64_t(1) << 29;    // frames a state row's c0 is clamped to (72 days at 22.05 kHz)
constexpr int MAX_NEW = 1 << 16;                     // largest max_new_frames of a call

// channels of layer l (l = 6: conv6's output, the GRU input): 1, 32, 32, 64, 64, 128, 128
OVC_HD int filt(int l) { return l == 0 ? 1 : (l < 3 ? 32 : (l < 5 ? 64 : 128)); }

OVC_HD int64_t clamp64(int64_t v, int64_t lo, int64_t hi) { return v < lo ? lo : (v > hi ? hi : v); }

// streaming.ready_frames(n, hop, nfft, False): frames whose support [t*hop - pad, t*hop - pad + nfft) lies below n
OVC_HD int64_t ready(int64_t n, int hop, int nfft) {
  const int64_t pad = (nfft - hop) / 2;
  if (n + pad < nfft) return 0;
  const int64_t r = (n + pad - nfft) / hop + 1;
  return r < n / hop ? r : n / hop;
}

// rows of layer l of a prefix of T frames (the host's H[] formula)
OVC_HD int64_t limit(int64_t T, int l) {
  for (int i = 0; i < l; ++i) T = (T - 1) / 2 + 1;
  return T;
}

// first row of layer l the carry keeps once the layer has c rows
OVC_HD int64_t carry_lo(int64_t c) { return c > 2 ? c - 2 : 0; }

// state row geometry for spec_channels F: width and carry offset of each conv input, offset of h, floats per row
struct Geom {
  int W[LAYERS + 1];
  int64_t carry[LAYERS];
  int64_t h;
  int64_t floats;
};

OVC_HD Geom geom(int F) {
  Geom g;
  g.W[0] = F;
  for (int l = 0; l < LAYERS; ++l) g.W[l + 1] = (g.W[l] - 1) / 2 + 1;
  int64_t at = HEADER;
  for (int l = 0; l < LAYERS; ++l) {
    g.carry[l] = at;
    at += 2 * (int64_t)filt(l) * g.W[l];
  }
  g.h = at;
  g.floats = (at + HID + 3) / 4 * 4;
  return g;
}

// workspace rows of layer l (l = 6: the GRU input) for calls of at most M new frames: an advance adds at most
// (M >> l) + 1 rows, a snapshot tail at most TAIL
OVC_HD int64_t ws_rows(int M, int l) {
  const int64_t r = (int64_t)(M >> l) + 1;
  return r > TAIL ? r : TAIL;
}

// workspace floats of one item: rows of every layer, then the GRU input projections of its steps
OVC_HD int64_t ws_floats(int M, int F) {
  const Geom g = geom(F);
  int64_t n = 0;
  for (int l = 0; l <= LAYERS; ++l) n += ws_rows(M, l) * filt(l) * g.W[l];
  return (n + ws_rows(M, LAYERS) * 3 * HID + 63) / 64 * 64;
}

// one descriptor (state_row, ring_row, n_adv, n_snap), clamped, against a row that has consumed c0 frames:
// the row advances to a1 (the snapshot's final frames, when the snapshot can be taken), takes it, then advances to a2.
struct Item {
  int64_t state_row, ring_row, c0, a1, a2;
  int64_t n_snap, T;   // snapshot prefix (samples) and its frames
  int tail;            // snapshot tail frames [a1, a1 + tail)
  bool snap, snap_ok;
};

OVC_HD Item item(const int64_t* d, int64_t c0, int64_t state_rows, int64_t ring_rows, int max_new, int hop, int nfft) {
  Item it;
  it.state_row = clamp64(d[0], 0, state_rows - 1);
  it.ring_row = clamp64(d[1], 0, ring_rows - 1);
  it.c0 = clamp64(c0, 0, MAX_FRAMES);
  const int64_t top = it.c0 + (max_new > 0 ? max_new : 0);
  const int64_t n_adv = clamp64(d[2], 0, MAX_SAMPLES);
  it.n_snap = clamp64(d[3], 0, MAX_SAMPLES);
  it.snap = it.n_snap > 0;
  const int64_t rs = ready(it.n_snap, hop, nfft);
  it.T = it.n_snap / hop;
  it.snap_ok = it.snap && it.T >= 1 && it.n_snap > (nfft - hop) / 2 && rs >= it.c0 && rs <= top && it.T - rs <= TAIL;
  it.a1 = it.snap_ok ? rs : it.c0;
  it.a2 = clamp64(ready(n_adv, hop, nfft), it.a1, top);
  it.tail = it.snap_ok ? (int)(it.T - it.a1) : 0;
  return it;
}

}  // namespace ovc_re
