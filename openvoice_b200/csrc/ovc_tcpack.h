// ovc_tcpack.h -- host side of the split-precision tensor-core conv (ovc_tcconv.cuh): the packed weight format, the
// rules that decide which convs fit the kernel, the polyphase form of the transposed convs and the persistent launch
// geometry.  The library (ovc_lib.cu) and the kernel harness (tests/kernelcheck/kc_tcconv.cu) both pack and launch
// through these functions, so a test of the kernel runs exactly what the library runs.  No device code.
#pragma once
#include <cuda_fp16.h>
#include <stddef.h>
#include <stdint.h>

#include <algorithm>

namespace ovc {

constexpr int TCN_HMAX = 25;   // largest conv-1 halo (k = 11, dilation 5): the staged A tile holds 128 + 2 * 25 rows
constexpr int TCN_ROWS2 = 146;  // conv pair: rows of the on-chip conv-2 operand, 128 + 2 * H2 with conv-2 halo H2 <= 9

// weight slots (16 channels x 1 tap, hi and lo parts) in the shared-memory ring: TN = 32 holds k = 11 resident,
// TN = 64 k = 3; pairs hold both convs resident up to TN = 32 k = 11 and TN = 64 k = 3, and stream the rest
constexpr int tc_ring_slots(int TN, bool pair) {
  return pair ? (TN == 32 ? 44 : TN == 64 ? 24 : 12) : (TN == 32 ? 22 : 12);
}

// the geometry of one packed conv (TN = 0: the conv does not fit the tensor-core kernels)
struct TcGeom {
  int Cin = 0, Ntot = 0, K = 0, DIL = 1, TN = 0;
};

// column tile: the widest of 128 / 64 / 32 that divides the output row.  0 when the conv does not fit: the kernels stage
// 32 input channels at a time, write 32-column groups, and hold a halo of at most TCN_HMAX rows on either side.
inline int tc_tile_n(int Ntot, int Cin, int K, int DIL) {
  if (Ntot <= 0 || Cin <= 0 || K <= 0 || DIL <= 0) return 0;
  if (Ntot % 32 || Cin % 32 || (K - 1) / 2 * DIL > TCN_HMAX) return 0;
  return Ntot % 128 == 0 ? 128 : (Ntot % 64 == 0 ? 64 : 32);
}

// one weight slot = [column block (2)][hi | lo][TN][8 halfs]: the B operand of one 16-channel k-step of one tap
inline size_t tc_slot_halfs(int TN) { return (size_t)2 * 2 * TN * 8; }
// whole packed conv: [n_tile = Ntot / TN][Cin / 16][K] slots
inline size_t tc_packed_halfs(int Ntot, int Cin, int K, int TN) {
  return TN ? (size_t)(Ntot / TN) * (Cin / 16) * K * tc_slot_halfs(TN) : 0;
}
// index of half e of weight (n, ci, tap) in the packed array, part 0 = hi, 1 = lo
inline size_t tc_packed_index(int Cin, int K, int TN, int n, int ci, int tap, int part) {
  const int nt = n / TN, k16 = ci / 16, kc = (ci % 16) / 8, e = ci % 8;
  const size_t slot = ((size_t)nt * (Cin / 16) + k16) * K + tap;
  return slot * tc_slot_halfs(TN) + ((size_t)(kc * 2 + part) * TN + n % TN) * 8 + e;
}

// the split of one weight: hi = fp16(w), lo = fp16((w - hi) * 2^11) (ovc_tc.cuh)
inline void tc_split(float w, uint16_t& hi, uint16_t& lo) {
  const __half h = __float2half_rn(w);
  const __half l = __float2half_rn((w - __half2float(h)) * 2048.f);
  hi = __half_as_ushort(h);
  lo = __half_as_ushort(l);
}

// packs W[n][ci][tap] = wfun(n, ci, tap) into dst (tc_packed_halfs(...) halfs), laid out exactly as the kernel's
// shared-memory operand slots (one TMA bulk copy per slot)
template <class WF>
inline void tc_pack_weights(uint16_t* dst, int Ntot, int Cin, int K, int TN, WF wfun) {
  for (int nt = 0; nt < Ntot / TN; ++nt)
    for (int k16 = 0; k16 < Cin / 16; ++k16)
      for (int tap = 0; tap < K; ++tap) {
        uint16_t* sl = dst + (((size_t)nt * (Cin / 16) + k16) * K + tap) * tc_slot_halfs(TN);
        for (int kc = 0; kc < 2; ++kc)
          for (int n = 0; n < TN; ++n)
            for (int e = 0; e < 8; ++e) {
              uint16_t hi, lo;
              tc_split(wfun(nt * TN + n, k16 * 16 + kc * 8 + e, tap), hi, lo);
              sl[((kc * 2 + 0) * TN + n) * 8 + e] = hi;   // rows [0, TN) of the 2*TN-row operand
              sl[((kc * 2 + 1) * TN + n) * 8 + e] = lo;   // rows [TN, 2*TN)
            }
      }
}

// ConvTranspose1d(Cin -> cout, stride s, kernel kk, padding (kk - s) / 2) as a 3-tap conv Cin -> s * cout on channels-
// last rows: packed row = ph * cout + co, so input step n yields the output steps s*n + ph, ph < s; tap 0 / 1 / 2 reads
// x[n-1] / x[n] / x[n+1] and holds raw weight index kidx = s * (1 - tap) + ph + pad (zero outside [0, kk)).
// raw(ci, co, k) reads the [cin][cout][kk] weight.
template <class RAW>
inline float tc_ups_weight(RAW raw, int s, int kk, int cout, int row, int ci, int tap) {
  const int pad = (kk - s) / 2;
  const int ph = row / cout, co = row % cout;
  const int kidx = s * (1 - tap) + ph + pad;
  return (kidx >= 0 && kidx < kk) ? raw(ci, co, kidx) : 0.f;
}

// the pairs whose two convs' weights stay resident in shared memory next to the operand tiles (C = 32 / 64, conv 2 of
// dilation 1, k <= 5).  The pair kernel also streams the weights of larger pairs through its ring (tc_pair_fuses).
inline bool tc_pair_fits(const TcGeom& T1, const TcGeom& T2) {
  if (!(T1.TN == 32 || T1.TN == 64)) return false;
  const int ring = tc_ring_slots(T1.TN, true);
  return T1.Ntot == T1.TN && T1.Cin == T1.TN && T2.Ntot == T1.TN && T2.Cin == T1.TN && T2.TN == T1.TN && T2.K == T1.K &&
         T2.DIL == 1 && (T1.K - 1) / 2 * T1.DIL <= TCN_HMAX && 2 * (T1.Cin / 16) * T1.K <= ring && T1.K <= 5;
}

// a ResBlock conv pair runs as ONE kernel (tcconv_kernel<C, true>) when it is a square C = 32 / 64 / 128 pair, conv 2
// of dilation 1 and the same k, whose conv-2 halo fits the on-chip operand.  That includes every pair tc_pair_fits
// accepts; the kernel streams the weights of the others through its ring.  Measured per (C, k) on an H100, every
// generator pair of the C <= 128 stages is faster fused than as two launches (DESIGN.md, fused ResBlock conv pair).
inline bool tc_pair_fuses(const TcGeom& T1, const TcGeom& T2) {
  if (!(T1.TN == 32 || T1.TN == 64 || T1.TN == 128)) return false;
  return T1.Ntot == T1.TN && T1.Cin == T1.TN && T2.Ntot == T1.TN && T2.Cin == T1.TN && T2.TN == T1.TN && T2.K == T1.K &&
         T2.DIL == 1 && (T1.K - 1) / 2 * T1.DIL <= TCN_HMAX && 128 + 2 * ((T2.K - 1) / 2) <= TCN_ROWS2;
}

// persistent launch: the CTAs of one column tile (grid.y) walk the (utterance, time tile) list, tile = b * n_tt + i
struct TcGrid {
  int n_tt = 0, total = 0, grid_x = 0, ncol = 0;
};
// single conv: 128 output steps per tile, 1 / grid_div of the SMs shared by the column tiles (grid_div = 3: the three
// concurrent ResBlock branches of a small call)
inline TcGrid tc_grid(int t_len, int B, int Ntot, int TN, int sm_count, int grid_div) {
  TcGrid g;
  g.n_tt = (t_len + 127) / 128;
  g.total = g.n_tt * B;
  g.ncol = Ntot / TN;
  const int per_col = std::max(1, sm_count / g.ncol / std::max(1, grid_div));
  g.grid_x = std::min(g.total, per_col);
  return g;
}
// conv pair: a tile is 128 conv-1 steps and yields R = 128 - (k - 1) output steps; occ CTAs per SM
inline TcGrid tc_pair_grid(int t_len, int B, int K, int sm_count, int occ = 1) {
  TcGrid g;
  const int R = 128 - (K - 1);
  g.n_tt = (t_len + R - 1) / R;
  g.total = g.n_tt * B;
  g.ncol = 1;
  g.grid_x = std::min(g.total, occ * sm_count);
  return g;
}

// shared memory of one pair-kernel CTA (TcnCfg<TN, true, ...>): barriers, nabuf conv-1 operand buffers of 194 rows x 32
// channels, the conv-2 operand, ring weight slots
constexpr size_t tc_pair_smem(int TN, int nabuf, int ring) {
  return 1024 + (size_t)nabuf * 2 * 4 * 194 * 16 + (size_t)2 * (TN / 8) * TCN_ROWS2 * 16 + (size_t)ring * 2 * 2 * TN * 16;
}
// two CTAs per SM: 228 KB of shared memory per SM, less 1 KB the hardware reserves per CTA
constexpr size_t TCN_SMEM_OCC2 = (233472 - 2 * 1024) / 2;
// weight slots of a pair config: today's ring at one CTA per SM (two operand buffers); at two, as many as fit
constexpr int tc_pair_ring(int TN, int occ, int nabuf) {
  return occ == 1 ? tc_ring_slots(TN, true) : (int)((TCN_SMEM_OCC2 - tc_pair_smem(TN, nabuf, 0)) / (2 * 2 * TN * 16));
}

// CTAs per SM and conv-1 operand buffers of a fused pair (tc_pair_fuses).  Two CTAs per SM let one tile's MMAs run while
// the other CTA sits in an epilogue or at a named barrier; they halve the shared memory, so the ring and the operand
// buffers shrink.  A pair whose weights are resident at one CTA per SM only runs two per SM where they stay resident
// (a streamed slot costs L2 bandwidth on every tile).  Measured per (C, k) on an H100 (DESIGN.md, two pair CTAs per SM):
//   C = 32, k = 3: two buffers, ring 22 (12 slots resident);  k = 7: one buffer, ring 34 (28 slots resident)
//   C = 64, k = 7 / 11 (streamed either way): one buffer, ring 12
//   C = 32, k = 11 and C = 64, k = 3 (resident only at one CTA per SM) and C = 128: one CTA per SM
struct TcPairOcc {
  int occ = 1, nabuf = 2;
};
inline TcPairOcc tc_pair_occ(const TcGeom& T1, const TcGeom& T2) {
  TcPairOcc o;
  if (!tc_pair_fuses(T1, T2)) return o;
  const int n_w = 2 * (T1.Cin / 16) * T1.K;   // both convs' weight slots
  if (T1.TN == 32 && n_w <= tc_pair_ring(32, 2, 2)) o = {2, 2};
  else if (T1.TN == 32 && n_w <= tc_pair_ring(32, 2, 1)) o = {2, 1};
  else if (T1.TN == 64 && n_w > tc_pair_ring(64, 1, 2)) o = {2, 1};
  return o;
}

}  // namespace ovc
