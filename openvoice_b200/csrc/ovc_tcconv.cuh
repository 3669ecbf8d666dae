// ovc_tcconv.cuh -- split-precision (3xFP16) tensor-core Conv1d for the generator / WaveNet convs.
//
//   Y[t, n] = (bias[n] + sum_{tap, c} W[n, c, tap] * lrelu(X[t + (tap - (K-1)/2) * DIL, c]) [+ R[t, n]] [+ Y_old[t, n]]) * scale
//
// Channels-last fp32 activations X[b][t][C] (time-major rows).  Every operand is split x = hi + lo / 2^11 with
// hi = fp16(x), lo = fp16((x - hi) * 2^11) (22 mantissa bits, ovc_tc.cuh) and every product is evaluated as
// a_hi*b_hi + (a_lo*b_hi + a_hi*b_lo) / 2^11 by wgmma (fp16 operands, fp32 accumulation in registers): the hi*hi
// products in one accumulator, the two cross terms in a second one ("low-order accumulator"), joined in the
// epilogue.  A weight slot holds b_hi in rows [0, TN) and b_lo in rows [TN, 2 TN); the main and the low-order
// accumulator are disjoint halves of one register array, and every k-step issues three MMAs of width TN: a_hi * b_hi^T
// into the main one, a_hi * b_lo^T and a_lo * b_hi^T into the low-order one.  (A single 2*TN-wide MMA over both halves
// followed by a TN-wide one into the upper half would save an A-operand read, but MMAs of different shapes on
// overlapping accumulator registers make ptxas serialise the whole wgmma chain.)  Besides carrying the 2^-11 scale,
// the second accumulator keeps the long hi*hi sum apart from the small cross terms.  Measured per conv on an H100
// (tests/test_gpu_kernels.py, DESIGN.md section 4.1): |y - y_fp64| <= 2^-18 * (sum |w||a| + |bias| + |res| + |y_old|)
// elementwise, max |y - y_fp64| <= 3e-5 * rms(y); the single pass (passes = 1): 2^-10 and 4e-3.
//
// K-major, no-swizzle operand tiles (see ovc_tc.cuh): a convolution tap is a 16-byte-per-row shift of the A
// descriptor's start address, so all taps (any dilation) read ONE staged halo tile.
//
// tcconv_kernel<TN, PAIR, OCC, NAB>: persistent, OCC CTAs (three warpgroups each) per SM walk the (utterance, 128-step
// tile) list; OCC = 2 only for conv pairs of the C = 32 / 64 stages (tc_pair_occ), where a second CTA's MMAs run while
// the first sits in an epilogue or at a named barrier.
//   warp 0       weights by TMA bulk copies: resident in shared memory for the whole launch when they fit, else a ring
//                streams them per tile
//   warps 1-3    converters: global fp32 rows -> lrelu -> fp16 hi/lo split -> A operand layout, running ahead across
//                tiles (two operand buffers); rows outside the utterance become zeros here (zero padding, x_mask and
//                the ragged batch in one rule)
//   warpgroups 1, 2  MMAs of 64 tile rows each (accumulators in registers), then the fused epilogue from registers
//   warpgroup 3  STAGED only (TN = 128, tc_stage_pays): the MMA warpgroups stage each tile's results in shared memory and
//                this warpgroup runs the epilogue from there while they compute the next tile
// PAIR = true runs one ResBlock conv PAIR of the narrow generator stages in the same kernel:
//   t = c1(lrelu(x)) (k taps, dilation d);  y = (c2(lrelu(t)) + x [+ y_old]) * scale (k taps, dilation 1)
// The epilogue of conv 1 writes lrelu(t), split into hi/lo, straight into a shared-memory A operand of conv 2, so t
// never leaves the SM.  A tile is 128 conv-1 steps; conv 2 needs (k-1)/2 steps of t on either side, so it yields
// 128 - (k-1) output steps.
#pragma once
#include "ovc_conv.cuh"
#include "ovc_tc.cuh"
#include "ovc_tcpack.h"

namespace ovc {

struct TcConvArgs {
  const float* x; long long x_bs;     // [B][Lpitch][Cin]
  const uint16_t* w;                   // packed fp16 [n_tile][Cin/16][K][2 (8-channel column block)][hi|lo][TN][8]
  const float* bias; long long bias_bs; // [Ntot] (+ b * bias_bs: per-utterance speaker-conditioning bias of the WN gate)
  float* y; long long y_bs; int y_ld;  // [B][Lpitch][y_ld]
  const float* r;                      // residual, same geometry as y (nullable)
  float* s; long long s_bs;            // EPI 2: skip accumulator [B][Lpitch][y_ld]
  int epi;                             // 0 linear (bias, residual, accumulate, scale) | 1 WN gate | 2 WN res/skip
  int split; int first;                // EPI 2: columns < split update y (x += rs), the rest go to s[col - split] (= / +=)
  const long long* lens; int tmax; int mul;   // valid steps = min(tmax, lens[b]) * mul   (lens NULL -> tmax)
  const long long* lens_x; int has_lens_x;    // when set: the INPUT's own validity limit (generator conv_pre on a padded batch:
                                              // z_hat * y_mask is cut at the frame lengths, the output runs to tmax)
  int Cin; int Ntot; int K; int DIL;   // Ntot = output row width (C for a ResBlock conv, stride*Cout for a polyphase transposed conv)
  float slope; float scale; int accumulate;
  int passes;   // 3: split precision (a_hi*b_hi + a_lo*b_hi + a_hi*b_lo); 1: single-pass fp16 (11-bit operands, like cuDNN's TF32 default)
  const uint16_t* w2; const float* bias2;   // PAIR: conv 2 (Cin = Ntot = TN, dilation 1); x is also the residual
  long long bias_ts;                   // per-frame conditioning: + min(t, tmax - 1) * bias_ts (0: one vector per item)
};

// Programmatic dependent launch (launch_tc sets the stream-serialization attribute): the NEXT kernel's CTAs may start
// their prologue (barriers, weight TMA) while this grid drains; a thread must pass pdl_wait() before it touches
// anything the PREVIOUS kernel wrote (or overwrites anything it read).
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(int id, int threads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// The conv result of accumulator-fragment element j (j < TN / 2) of a thread: v = lo / 2^11 + hi (ovc_tc.cuh: fragment
// columns [0, TN) main accumulator, [TN, 2 TN) low-order accumulator), or hi alone for the single pass.
template <int TN>
__device__ __forceinline__ float tc_result(const float (&d)[TN], bool two, int j) {
  return two ? fmaf(d[TN / 2 + j], tc::kLoInv, d[j]) : d[j];
}

// Epilogue of one thread's two rows (tile rows row_a and row_a + 8, output steps t0 + row) x TN columns of an
// accumulator fragment whose element j holds the conv result v_at(j) (tc_result).  The MMA warpgroups run it on their
// registers; the store warpgroup of the staged kernels (TcnCfg::STAGED) on the same values read back from shared memory,
// with the fragment layout of the MMA thread it stands in for, so both paths perform the same operations on the same
// fp32 values.  Four consecutive threads cover 32 contiguous bytes of an output row, so every global access of a warp is
// whole sectors.
// PF: a per-frame conditioning vector (bias_ts != 0); tc_epilogue_v picks the instantiation, so a per-item call runs
// the epilogue it always ran.
template <int TN, bool PF, class V>
__device__ __forceinline__ void tc_epilogue_body(const TcConvArgs& a, V v_at, int b, int t0, int n0, int lim, int row_a) {
  const int csub = (threadIdx.x & 3) * 2;
  float* yb = a.y + (size_t)b * a.y_bs;
  const float* rb = a.r ? a.r + (size_t)b * a.y_bs : nullptr;
  float* sb = a.s ? a.s + (size_t)b * a.s_bs : nullptr;
  const int ta = t0 + row_a, tb = ta + 8;
  const bool oka = ta < lim, okb = tb < lim;
  // rows ta and tb are different frames: with a per-frame conditioning vector each reads its own
  const float* bias_a = a.bias + (size_t)b * a.bias_bs + (PF ? (size_t)min(ta, a.tmax - 1) * a.bias_ts : 0);
  const float* bias_b = a.bias + (size_t)b * a.bias_bs + (PF ? (size_t)min(tb, a.tmax - 1) * a.bias_ts : 0);
#pragma unroll
  for (int c0 = 0; c0 < TN; c0 += 32) {
    float v[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] = v_at(c0 / 2 + i);
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const float2 bq = __ldg(reinterpret_cast<const float2*>(bias_a + n0 + c0 + 8 * g + csub));
      const float2 br = PF ? __ldg(reinterpret_cast<const float2*>(bias_b + n0 + c0 + 8 * g + csub)) : bq;
      v[4 * g] += bq.x; v[4 * g + 1] += bq.y; v[4 * g + 2] += br.x; v[4 * g + 3] += br.y;
    }
    if (a.epi == 0) {
      // ---- linear: bias, residual, MRF accumulate, scale
      float* ypa = yb + (size_t)ta * a.y_ld + n0 + c0 + csub;
      float* ypb = yb + (size_t)tb * a.y_ld + n0 + c0 + csub;
      const float* rpa = rb ? rb + (size_t)ta * a.y_ld + n0 + c0 + csub : nullptr;
      const float* rpb = rb ? rb + (size_t)tb * a.y_ld + n0 + c0 + csub : nullptr;
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        float2 oa = make_float2(v[4 * g], v[4 * g + 1]), ob = make_float2(v[4 * g + 2], v[4 * g + 3]);
        if (rb) {
          const float2 qa = oka ? *reinterpret_cast<const float2*>(rpa + 8 * g) : make_float2(0.f, 0.f);
          const float2 qb = okb ? *reinterpret_cast<const float2*>(rpb + 8 * g) : make_float2(0.f, 0.f);
          oa.x += qa.x; oa.y += qa.y; ob.x += qb.x; ob.y += qb.y;
        }
        if (a.accumulate) {
          const float2 ya = oka ? *reinterpret_cast<const float2*>(ypa + 8 * g) : make_float2(0.f, 0.f);
          const float2 yc = okb ? *reinterpret_cast<const float2*>(ypb + 8 * g) : make_float2(0.f, 0.f);
          oa.x = ya.x + oa.x; oa.y = ya.y + oa.y;
          ob.x = yc.x + ob.x; ob.y = yc.y + ob.y;
        }
        if (a.scale != 1.f) { oa.x *= a.scale; oa.y *= a.scale; ob.x *= a.scale; ob.y *= a.scale; }
        if (oka) *reinterpret_cast<float2*>(ypa + 8 * g) = oa;
        if (okb) *reinterpret_cast<float2*>(ypb + 8 * g) = ob;
      }
    } else if (a.epi == 1) {
      // ---- WaveNet gate (modules.py:185-210): columns [0,16) of the group are the tanh inputs of 16 channels,
      // [16,32) their sigmoid partners -> 16 output channels at column (n0 + c0) / 2
      float* ypa = yb + (size_t)ta * a.y_ld + ((n0 + c0) >> 1) + csub;
      float* ypb = yb + (size_t)tb * a.y_ld + ((n0 + c0) >> 1) + csub;
#pragma unroll
      for (int g = 0; g < 2; ++g) {
        const float2 oa = make_float2(tanhf(v[4 * g]) * sigmoidf_acc(v[4 * (g + 2)]),
                                      tanhf(v[4 * g + 1]) * sigmoidf_acc(v[4 * (g + 2) + 1]));
        const float2 ob = make_float2(tanhf(v[4 * g + 2]) * sigmoidf_acc(v[4 * (g + 2) + 2]),
                                      tanhf(v[4 * g + 3]) * sigmoidf_acc(v[4 * (g + 2) + 3]));
        if (oka) *reinterpret_cast<float2*>(ypa + 8 * g) = oa;
        if (okb) *reinterpret_cast<float2*>(ypb + 8 * g) = ob;
      }
    } else {
      // ---- WaveNet res/skip: columns < split update x in place (x += res), the rest go to the skip sum (= / +=)
      const int col = n0 + c0;
      const bool to_x = col < a.split;          // uniform per 32-column group (split is a multiple of 32)
      const bool add = to_x || !a.first;
      float* dst = (to_x ? yb + col : sb + (col - a.split)) + csub;
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        float2 oa = make_float2(v[4 * g], v[4 * g + 1]), ob = make_float2(v[4 * g + 2], v[4 * g + 3]);
        if (add) {
          const float2 qa = oka ? *reinterpret_cast<const float2*>(dst + (size_t)ta * a.y_ld + 8 * g) : make_float2(0.f, 0.f);
          const float2 qb = okb ? *reinterpret_cast<const float2*>(dst + (size_t)tb * a.y_ld + 8 * g) : make_float2(0.f, 0.f);
          oa = make_float2(qa.x + oa.x, qa.y + oa.y);
          ob = make_float2(qb.x + ob.x, qb.y + ob.y);
        }
        if (oka) *reinterpret_cast<float2*>(dst + (size_t)ta * a.y_ld + 8 * g) = oa;
        if (okb) *reinterpret_cast<float2*>(dst + (size_t)tb * a.y_ld + 8 * g) = ob;
      }
    }
  }
}

template <int TN, class V>
__device__ __forceinline__ void tc_epilogue_v(const TcConvArgs& a, V v_at, int b, int t0, int n0, int lim, int row_a) {
  if (a.bias_ts) tc_epilogue_body<TN, true>(a, v_at, b, t0, n0, lim, row_a);
  else tc_epilogue_body<TN, false>(a, v_at, b, t0, n0, lim, row_a);
}

template <int TN>
__device__ __forceinline__ void tc_epilogue(const TcConvArgs& a, const float (&d)[TN], int b, int t0, int n0, int lim, int row_a) {
  const bool two = a.passes == 3;
  tc_epilogue_v<TN>(a, [&](int j) { return tc_result<TN>(d, two, j); }, b, t0, n0, lim, row_a);
}
// the linear epilogue of a conv pair's conv 2: bias2, the pair's input as the residual, y_old, scale; rows past
// t0 + R are the discarded output steps of the tile
__device__ __forceinline__ TcConvArgs tc_pair_epilogue_args(const TcConvArgs& a, int TN) {
  TcConvArgs e = a;
  e.y_ld = TN; e.r = a.x; e.bias = a.bias2; e.bias_bs = 0; e.bias_ts = 0; e.epi = 0;
  return e;
}

// one k-step x tap of a warpgroup's 64 rows: main (+)= a_hi * b_hi^T, low (+)= a_hi * b_lo^T + a_lo * b_hi^T
template <int TN>
__device__ __forceinline__ void tc_mma_step(float (&d)[TN], uint64_t a_hi, uint64_t a_lo, uint64_t b, bool three, bool first) {
  float (&lo)[TN / 2] = *reinterpret_cast<float(*)[TN / 2]>(&d[TN / 2]);
  float (&hi)[TN / 2] = *reinterpret_cast<float(*)[TN / 2]>(&d[0]);
  tc::Wgmma<TN>::mma(hi, a_hi, b, first ? 0 : 1);
  if (three) {
    tc::Wgmma<TN>::mma(lo, a_hi, b + TN, first ? 0 : 1);   // b_lo: rows [TN, 2 TN) of the slot, TN * 16 bytes on
    tc::Wgmma<TN>::mma(lo, a_lo, b, 1);
  }
}

constexpr int TCN_THREADS = 384;   // warpgroup 0: producers; warpgroups 1, 2: MMAs + epilogue (TcnCfg::THREADS unless STAGED)
constexpr int TCN_NCT = 96;        // converter threads (warps 1-3)

// OCC: CTAs per SM (2: pairs of the C = 32 / 64 stages only, ovc_tcpack.h tc_pair_occ); NAB: conv-1 operand buffers;
// STAGED (TN = 128, one CTA per SM): a fourth warpgroup runs the global epilogue of each tile from a staging tile in
// shared memory while the MMA warpgroups go on with the next tile
template <int TN, bool PAIR, int OCC = 1, int NAB = 2, bool STAGED = false>
struct TcnCfg {
  static_assert(!PAIR || TN == 32 || TN == 64 || TN == 128, "conv pairs: C = 32, 64 or 128");
  static_assert(OCC == 1 || (PAIR && TN <= 64), "two CTAs per SM: C = 32 / 64 pairs");
  static_assert(!STAGED || (TN == 128 && OCC == 1), "staged epilogue: TN = 128, one CTA per SM");
  // warpgroup 0: producers; warpgroups 1, 2: MMAs (+ the epilogue unless STAGED); warpgroup 3 (STAGED): the epilogue
  static constexpr int THREADS = STAGED ? TCN_THREADS + 128 : TCN_THREADS;
  static constexpr int KCH = 32, NKC = KCH / 8;                   // channels per converted A chunk
  static constexpr int ROWS = 194;                                // A pitch in rows: >= 128 + 2 * TCN_HMAX, = 2 (mod 8)
  static constexpr int ROWS2 = TCN_ROWS2;                         // PAIR: conv-2 A pitch: 128 + 2 * H2 rows, H2 <= 9
  static constexpr int NABUF = NAB;
  static constexpr int RING = PAIR ? tc_pair_ring(TN, OCC, NAB) : tc_ring_slots(TN, PAIR);   // weight slots (ovc_tcpack.h)
  static constexpr int SLOT_BYTES = 2 * 2 * TN * 16;
  static constexpr int A_BUF_BYTES = 2 * NKC * ROWS * 16;         // [hi|lo][column block][row][8 halfs]
  static constexpr int A2_BYTES = PAIR ? 2 * (TN / 8) * ROWS2 * 16 : 0;
  // STAGED: the conv results of one tile, fp32, [fragment element j < TN / 2][MMA thread t < 256] (conflict-free: a warp
  // writes and reads 32 consecutive words).  A pair stages in its conv-2 operand, dead once conv 2's MMAs are done and
  // not rewritten before the next tile's conv-1 epilogue; a single conv adds a buffer of its own.
  static constexpr int STAGE_BYTES = STAGED ? (TN / 2) * 256 * 4 : 0;
  static_assert(!STAGED || !PAIR || STAGE_BYTES <= A2_BYTES, "a pair's staging tile lies in its conv-2 operand");
  static constexpr int SBUF_BYTES = STAGED && !PAIR ? STAGE_BYTES : 0;
  static constexpr size_t SMEM_BYTES = 1024 + NABUF * A_BUF_BYTES + A2_BYTES + RING * SLOT_BYTES + SBUF_BYTES;
  static_assert(!PAIR || SMEM_BYTES == tc_pair_smem(TN, NABUF, RING), "tc_pair_smem");
  static_assert(SMEM_BYTES <= (OCC == 1 ? 232448 : TCN_SMEM_OCC2), "shared memory budget");
  static_assert((2 * NABUF + 2 * RING + 2) * 8 <= 1024, "barrier area");
  // registers per thread after the producers hand theirs to the MMA warpgroups: 128 x 56 + 256 x 224 = 63 K at one CTA
  // per SM, 128 x 32 + 256 x 104 = 30 K (of the 32 K the launch bounds give a CTA) at two.  STAGED: 128 x 32 (producers)
  // + 256 x 184 (MMAs: the accumulators and, in a pair, the conv-1 epilogue; ptxas allocates 180 there) + 128 x 112 (the
  // store warpgroup: room for many loads in flight; at 32 it spills) = 64 K
  static constexpr int PROD_REGS = OCC == 1 && !STAGED ? 56 : 32, MMA_REGS = STAGED ? 184 : OCC == 1 ? 224 : 104;
  static constexpr int STORE_REGS = 112;
  static_assert(128 * PROD_REGS + 256 * MMA_REGS + (STAGED ? 128 * STORE_REGS : 0) <= 65536 / OCC, "register budget");
};

template <int TN, bool PAIR, int OCC = 1, int NAB = 2, bool STAGED = false>
__global__ void __launch_bounds__(TcnCfg<TN, PAIR, OCC, NAB, STAGED>::THREADS, OCC) tcconv_kernel(const TcConvArgs a, int n_tt, int total) {
  using Cfg = TcnCfg<TN, PAIR, OCC, NAB, STAGED>;
  constexpr int ROWS = Cfg::ROWS, ROWS2 = Cfg::ROWS2, NABUF = Cfg::NABUF, RING = Cfg::RING, NKC = Cfg::NKC;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw);
  uint64_t *a_full = bars, *a_empty = bars + NABUF, *b_full = a_empty + NABUF, *b_empty = b_full + RING;
  uint64_t *s_full = b_empty + RING, *s_empty = s_full + 1;   // STAGED: the staging tile holds a tile / is free
  unsigned char* abuf = smem_raw + 1024;
  unsigned char* a2buf = abuf + NABUF * Cfg::A_BUF_BYTES;
  unsigned char* bring = a2buf + Cfg::A2_BYTES;
  float* stage = reinterpret_cast<float*>(PAIR ? a2buf : bring + RING * Cfg::SLOT_BYTES);

  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);   // provably warp-uniform
  const int H1 = (a.K - 1) / 2 * a.DIL;
  const int H2 = PAIR ? (a.K - 1) / 2 : 0;
  const int R = 128 - 2 * H2;                  // output steps per tile
  const int rows8 = (128 + 2 * H1 + 7) & ~7;   // staged input rows per chunk
  const int nq = a.Cin / Cfg::KCH;
  const int n_slots = (a.Cin / 16) * a.K;      // weight slots per conv
  const int n_w = PAIR ? 2 * n_slots : n_slots;
  const bool resident = n_w <= RING;
  if (H1 > TCN_HMAX || (PAIR && 128 + 2 * H2 > ROWS2)) __trap();   // host: tc_tile_n / tc_pair_fuses (ovc_tcpack.h)
  constexpr uint32_t BYTES = Cfg::SLOT_BYTES;

  if (tid == 0) {
    for (int i = 0; i < NABUF; ++i) { mbar_init(&a_full[i], TCN_NCT); mbar_init(&a_empty[i], 2); }
    for (int i = 0; i < RING; ++i) { mbar_init(&b_full[i], 1); mbar_init(&b_empty[i], 2); }
    if (STAGED) { mbar_init(s_full, 256); mbar_init(s_empty, 128); }
    fence_mbar_init();
  }
  if (PAIR) {
    // rows of the conv-2 operand that conv 1 never produces (the taps of the discarded last output rows read them)
    for (int i = tid; i < Cfg::A2_BYTES / 16; i += Cfg::THREADS) reinterpret_cast<uint4*>(a2buf)[i] = make_uint4(0u, 0u, 0u, 0u);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  pdl_launch_dependents();
  if (warp != 0) pdl_wait();   // warp 0 only streams the (constant) weights: it may run ahead of the previous kernel's end

  // every role walks the same tile sequence
#define TCN_FOR_TILES                                                                                   \
  for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {                                        \
    const int b = tile / n_tt, t0 = (tile % n_tt) * R;                                                  \
    const int lim = (a.lens ? (int)min((long long)a.tmax, a.lens[b]) : a.tmax) * a.mul;                 \
    const int lim_x = a.has_lens_x ? (int)min((long long)a.tmax, a.lens_x[b]) * a.mul : lim;            \
    (void)lim_x;                                                                                        \
    if (t0 >= lim) continue;

  if (warp < 4) {
    tc::regs_dealloc<Cfg::PROD_REGS>();
    if (warp == 0) {
      // ------------------------------------------------------------ weights
      if (lane == 0) {
        const unsigned char* wt = reinterpret_cast<const unsigned char*>(a.w) + (size_t)blockIdx.y * n_slots * BYTES;
        if (resident) {
          for (int it = 0; it < n_w; ++it) {
            const unsigned char* src = it < n_slots ? wt + (size_t)it * BYTES
                                                    : reinterpret_cast<const unsigned char*>(a.w2) + (size_t)(it - n_slots) * BYTES;
            mbar_expect_tx(&b_full[it], BYTES);
            tma_bulk_g2s(bring + it * BYTES, src, BYTES, &b_full[it]);
          }
          // a CTA whose tiles all lie past their utterances never waits on these copies: they must have landed before
          // the CTA can exit (its shared memory may be handed to the next kernel's CTA)
          for (int it = 0; it < n_w; ++it) mbar_wait(&b_full[it], 0u);
        } else {
          // streamed: every tile takes conv 1's slots (and a pair's conv-2 slots after them) in the MMA order
          int slot = 0;
          uint32_t phase = 1;   // the first pass over the ring finds every slot free
          TCN_FOR_TILES
            (void)b;
            for (int it = 0; it < n_w; ++it) {
              const unsigned char* src = it < n_slots ? wt + (size_t)it * BYTES
                                                      : reinterpret_cast<const unsigned char*>(a.w2) + (size_t)(it - n_slots) * BYTES;
              mbar_wait(&b_empty[slot], phase);
              mbar_expect_tx(&b_full[slot], BYTES);
              tma_bulk_g2s(bring + slot * BYTES, src, BYTES, &b_full[slot]);
              if (++slot == RING) { slot = 0; phase ^= 1; }
            }
          }
        }
      }
    } else {
      // ------------------------------------------------------------ converters (run ahead across tiles)
      const int pt = tid - 32;
      const int items = rows8 * NKC;            // item i = (row i / 4, column block i % 4): 32 bytes of one row
      int buf = 0;
      uint32_t ephase = 1;
      TCN_FOR_TILES
        const float* xb = a.x + (size_t)b * a.x_bs;
        const int r0 = t0 - H2 - H1;            // input step of staged row 0
        for (int q = 0; q < nq; ++q) {
          mbar_wait(&a_empty[buf], ephase);
          unsigned char* ah = abuf + buf * Cfg::A_BUF_BYTES;
          unsigned char* al = ah + NKC * ROWS * 16;
          constexpr int PB = 2;   // items (32 bytes each) in flight per thread
          for (int i0 = pt; i0 < items; i0 += TCN_NCT * PB) {
            float4 v0[PB], v1[PB];
#pragma unroll
            for (int u = 0; u < PB; ++u) {
              const int i = i0 + TCN_NCT * u;
              const int row = i >> 2, kc = i & 3;
              const int t = r0 + row;
              v0[u] = make_float4(0.f, 0.f, 0.f, 0.f);
              v1[u] = v0[u];
              if (i < items && t >= 0 && t < lim_x) {
                const float4* src = reinterpret_cast<const float4*>(xb + (size_t)t * a.Cin + q * Cfg::KCH + kc * 8);
                v0[u] = src[0];
                v1[u] = src[1];
              }
            }
#pragma unroll
            for (int u = 0; u < PB; ++u) {
              const int i = i0 + TCN_NCT * u;
              if (i >= items) break;
              const int row = i >> 2, kc = i & 3;
              uint4 hi, lo;
              tc::split_f16x8(v0[u], v1[u], a.slope, hi, lo);
              *reinterpret_cast<uint4*>(ah + (kc * ROWS + row) * 16) = hi;
              *reinterpret_cast<uint4*>(al + (kc * ROWS + row) * 16) = lo;
            }
          }
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic writes -> tensor-core (async) proxy
          mbar_arrive(&a_full[buf]);
          if (++buf == NABUF) { buf = 0; ephase ^= 1; }
        }
      }
    }
  } else if (STAGED && warp >= 12) {
    // ------------------------------------------------------------ store warpgroup (STAGED): the global epilogue of each
    // tile, for both MMA warpgroups' rows, from the staging tile
    tc::regs_dealloc<Cfg::STORE_REGS>();
    const int st = tid & 127;
    uint32_t phase = 0;
    TCN_FOR_TILES
      // a pair's conv-1 epilogue rewrites the staging tile (its conv-2 operand): the previous tile has been read
      if (PAIR) named_bar_arrive(1, 384);
      mbar_wait(s_full, phase);
      phase ^= 1;
#pragma unroll 1
      for (int h = 0; h < 2; ++h) {
        const float* sv = stage + h * 128 + st;   // stands in for MMA thread 128 h + st
        const auto v_at = [&](int j) { return sv[j * 256]; };
        const int row_a = 64 * h + 16 * (warp & 3) + (lane >> 2);
        if constexpr (PAIR) tc_epilogue_v<TN>(tc_pair_epilogue_args(a, TN), v_at, b, t0, 0, min(lim, t0 + R), row_a);
        else tc_epilogue_v<TN>(a, v_at, b, t0, blockIdx.y * TN, lim, row_a);
      }
      if (!PAIR) mbar_arrive(s_empty);
    }
  } else {
    // ------------------------------------------------------------ MMA warpgroups: rows [64 wg, +64) of every tile
    tc::regs_alloc<Cfg::MMA_REGS>();
    const int wg = (warp >> 2) - 1;
    const bool leader = (tid & 127) == 0;
    const int row_a = 64 * wg + 16 * (warp & 3) + (lane >> 2);   // this thread's first accumulator row
    constexpr uint32_t LBO_A = ROWS * 16, LBO_A2 = ROWS2 * 16, LBO_B = 2 * TN * 16, SBO = 128;
    constexpr uint32_t A_LO16 = (NKC * ROWS * 16) >> 4, A2_LO16 = ((TN / 8) * ROWS2 * 16) >> 4, SLOT16 = BYTES >> 4;
    const uint64_t a_proto = tc::make_desc(0, LBO_A, SBO), b_proto = tc::make_desc(0, LBO_B, SBO);
    const uint64_t b_ring = b_proto + (tc::smem_addr(bring) >> 4);
    const bool three = a.passes == 3;
    float d[TN];
#pragma unroll
    for (int i = 0; i < TN; ++i) d[i] = 0.f;
    // STAGED: this thread's conv results -> the staging tile, then on to the next tile (the store warpgroup takes it)
    const auto stage_tile = [&]() {
#pragma unroll
      for (int j = 0; j < TN / 2; ++j) stage[j * 256 + tid - 128] = tc_result<TN>(d, three, j);
      mbar_arrive(s_full);
    };
    uint32_t sphase = 1;   // the first tile finds the staging tile free
    (void)sphase;
    if (resident)
      for (int it = 0; it < n_w; ++it) mbar_wait(&b_full[it], 0u);   // resident weights: waited on once
    int slot = 0, buf = 0;
    uint32_t bphase = 0, aphase = 0;
    TCN_FOR_TILES
      (void)lim_x;
      // ---- conv (conv 1 of a pair)
      bool first = true;
      if (resident) slot = 0;
      for (int q = 0; q < nq; ++q) {
        mbar_wait(&a_full[buf], aphase);
        tc::fence_regs(d);
        tc::wgmma_fence();
        int prev = -1;
        for (int j = 0; j < 2; ++j) {
          uint64_t a_cur = a_proto + ((tc::smem_addr(abuf + buf * Cfg::A_BUF_BYTES) + 64 * wg * 16 + 2 * j * LBO_A) >> 4);
          for (int tap = 0; tap < a.K; ++tap) {
            if (!resident) mbar_wait(&b_full[slot], bphase);
            // output row i reads staged row i + tap * DIL: the staged tile starts at the first output step - H
            tc_mma_step<TN>(d, a_cur, a_cur + A_LO16, b_ring + (uint32_t)slot * SLOT16, three, first);
            tc::wgmma_commit();
            if (!resident) {
              tc::wgmma_wait<1>();                              // the previous step's MMAs have read their slot
              if (leader && prev >= 0) mbar_arrive(&b_empty[prev]);
              prev = slot;
            }
            first = false;
            a_cur += a.DIL;
            if (++slot == RING) { slot = 0; bphase ^= 1; }
          }
        }
        tc::wgmma_wait<0>();
        tc::fence_regs(d);
        if (leader) {
          if (prev >= 0) mbar_arrive(&b_empty[prev]);
          mbar_arrive(&a_empty[buf]);
        }
        if (++buf == NABUF) { buf = 0; aphase ^= 1; }
      }
      if constexpr (!PAIR) {
        if constexpr (STAGED) {
          mbar_wait(s_empty, sphase);
          sphase ^= 1;
          stage_tile();
        } else {
          tc_epilogue<TN>(a, d, b, t0, blockIdx.y * TN, lim, row_a);
        }
      } else {
        // ---- conv-1 epilogue: bias, leaky-relu, hi/lo split -> conv-2 A operand (rows = steps t0 - H2 + row)
        // both warpgroups are done reading the conv-2 operand of the previous tile (and STAGED: the store warpgroup is
        // done reading the previous tile's results staged there)
        named_bar_sync(1, STAGED ? 384 : 256);
        unsigned char* a2h = a2buf;
        unsigned char* a2l = a2buf + (TN / 8) * ROWS2 * 16;
        const int ta = t0 - H2 + row_a, tb = ta + 8;
        // t lives on steps [0, lim): outside them conv 2 sees zero padding, not conv 1 evaluated on padding
        const bool oka = ta >= 0 && ta < lim, okb = tb >= 0 && tb < lim;
        const int csub = (lane & 3) * 2;
#pragma unroll
        for (int g = 0; g < TN / 8; ++g) {
          const float2 bq = __ldg(reinterpret_cast<const float2*>(a.bias + 8 * g + csub));
          float x[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) x[i] = (three ? fmaf(d[TN / 2 + 4 * g + i], tc::kLoInv, d[4 * g + i]) : d[4 * g + i]) + ((i & 1) ? bq.y : bq.x);
          x[0] = oka ? fmaxf(x[0], x[0] * a.slope) : 0.f;
          x[1] = oka ? fmaxf(x[1], x[1] * a.slope) : 0.f;
          x[2] = okb ? fmaxf(x[2], x[2] * a.slope) : 0.f;
          x[3] = okb ? fmaxf(x[3], x[3] * a.slope) : 0.f;
          const __half2 ha = __floats2half2_rn(x[0], x[1]), hb = __floats2half2_rn(x[2], x[3]);
          const float2 fa = __half22float2(ha), fb = __half22float2(hb);
          const __half2 la = __floats2half2_rn((x[0] - fa.x) * tc::kLoScale, (x[1] - fa.y) * tc::kLoScale);
          const __half2 lb = __floats2half2_rn((x[2] - fb.x) * tc::kLoScale, (x[3] - fb.y) * tc::kLoScale);
          const int oa = (g * ROWS2 + row_a) * 16 + (lane & 3) * 4, ob = oa + 8 * 16;
          *reinterpret_cast<__half2*>(a2h + oa) = ha;
          *reinterpret_cast<__half2*>(a2h + ob) = hb;
          *reinterpret_cast<__half2*>(a2l + oa) = la;
          *reinterpret_cast<__half2*>(a2l + ob) = lb;
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic writes -> tensor-core (async) proxy
        named_bar_sync(2, 256);   // every row of the conv-2 operand is written
        // ---- conv 2 (dilation 1, weights in the resident slots after conv 1's, or the next ones of the stream)
        const uint64_t a2_proto = tc::make_desc(0, LBO_A2, SBO);
        tc::fence_regs(d);
        tc::wgmma_fence();
        bool first2 = true;
        int prev = -1;
        for (int kk = 0; kk < TN / 16; ++kk) {
          uint64_t a_cur = a2_proto + ((tc::smem_addr(a2buf) + 64 * wg * 16 + 2 * kk * LBO_A2) >> 4);
          for (int tap = 0; tap < a.K; ++tap) {
            if (resident) {
              tc_mma_step<TN>(d, a_cur, a_cur + A2_LO16, b_ring + (uint32_t)(n_slots + kk * a.K + tap) * SLOT16, three, first2);
            } else {
              mbar_wait(&b_full[slot], bphase);
              tc_mma_step<TN>(d, a_cur, a_cur + A2_LO16, b_ring + (uint32_t)slot * SLOT16, three, first2);
              tc::wgmma_commit();
              tc::wgmma_wait<1>();                              // the previous step's MMAs have read their slot
              if (leader && prev >= 0) mbar_arrive(&b_empty[prev]);
              prev = slot;
              if (++slot == RING) { slot = 0; bphase ^= 1; }
            }
            first2 = false;
            a_cur += 1;
          }
        }
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::fence_regs(d);
        if (leader && prev >= 0) mbar_arrive(&b_empty[prev]);
        if constexpr (STAGED) {
          // the staging tile overlays the conv-2 operand, and each warpgroup's MMAs read halo rows of the other's
          named_bar_sync(3, 256);
          // rows >= 128 of the operand (zero) are overwritten too: only the accumulator rows >= R read them, and
          // those rows are the discarded output steps of every tile
          stage_tile();
        } else {
          tc_epilogue<TN>(tc_pair_epilogue_args(a, TN), d, b, t0, 0, min(lim, t0 + R), row_a);
        }
      }
    }
  }
#undef TCN_FOR_TILES
}

// a tcconv_kernel instantiation with its dynamic shared memory and block size; fn = nullptr when none is built
struct TcKernel {
  void (*fn)(TcConvArgs, int, int) = nullptr;
  size_t smem = 0;
  int threads = 0;
};
using TcPairKernel = TcKernel;   // the unstaged pair kernels: threads = TCN_THREADS
template <int TN, bool PAIR, int OCC = 1, int NAB = 2, bool STAGED = false>
inline TcKernel tc_kernel() {
  using Cfg = TcnCfg<TN, PAIR, OCC, NAB, STAGED>;
  return {tcconv_kernel<TN, PAIR, OCC, NAB, STAGED>, Cfg::SMEM_BYTES, Cfg::THREADS};
}
// whether a TN = 128 conv (or C = 128 pair) of k taps runs the staged epilogue when OVC_OPT_STAGED_EPI is on.  The store
// warpgroup takes longer over a tile's epilogue than the two MMA warpgroups did, so it only pays where a tile's MMAs
// outlast it: measured on an H100 (DESIGN.md, staged epilogue), split precision at k >= 5 gains, while k = 1 / 3 and
// every single-pass shape but k = 11 lose or break even.
inline bool tc_stage_pays(int K, int passes) { return passes * K >= 15; }
// the single-conv kernel of column tile TN; staged: TN = 128 runs the staged epilogue (OVC_OPT_STAGED_EPI)
inline TcKernel tc_conv_kernel(int TN, bool staged) {
  if (TN == 128) return staged ? tc_kernel<128, false, 1, 2, true>() : tc_kernel<128, false>();
  if (TN == 64) return tc_kernel<64, false>();
  if (TN == 32) return tc_kernel<32, false>();
  return {};
}
// the pair kernel of a (C, tc_pair_occ) config; staged: C = 128 runs the staged epilogue
inline TcKernel tc_pair_kernel(int C, TcPairOcc o, bool staged = false) {
  if (o.occ == 1 && o.nabuf == 2) {
    if (C == 128) return staged ? tc_kernel<128, true, 1, 2, true>() : tc_kernel<128, true>();
    if (C == 64) return tc_kernel<64, true>();
    if (C == 32) return tc_kernel<32, true>();
  } else if (o.occ == 2) {
    if (C == 32 && o.nabuf == 2) return tc_kernel<32, true, 2, 2>();
    if (C == 32 && o.nabuf == 1) return tc_kernel<32, true, 2, 1>();
    if (C == 64 && o.nabuf == 1) return tc_kernel<64, true, 2, 1>();
  }
  return {};
}
// the two-CTA-per-SM configs tc_pair_occ can pick
constexpr int TCN_N_OCC2 = 3;
constexpr struct { int C; TcPairOcc o; } kTcPairOcc2[TCN_N_OCC2] = {{32, {2, 2}}, {32, {2, 1}}, {64, {2, 1}}};

// conv_post on channels-last input: y[b, t] = tanh(sum_{k<7, ci<C} w[ci, k] * lrelu_0.01(x[b, t+k-3, ci]))
// (models.py:287-289).  HBM-bound (132 B per sample): a CTA stages 256+6 rows with coalesced 16-byte loads into a
// transposed, conflict-free shared tile (leaky_relu applied once), then one thread per output sample.
template <int C>
__global__ void __launch_bounds__(256) conv_post_cl_kernel(const float* __restrict__ x, long long x_bs,
                                                           const float* __restrict__ w, float* __restrict__ y,
                                                           long long y_bs, int y_len, const long long* lens, int tmax,
                                                           int mul) {
  constexpr int TB = 256, ROWS = TB + 6, LD = ROWS + 3;   // LD odd: conflict-free transposed stores
  __shared__ float ws[7][C];
  __shared__ float xs[C][LD];
  for (int i = threadIdx.x; i < C * 7; i += blockDim.x) ws[i % 7][i / 7] = w[i];
  const int b = blockIdx.y;
  const int lim = (lens ? (int)min((long long)tmax, lens[b]) : tmax) * mul;
  const int t0 = blockIdx.x * TB;
  const float* xb = x + (size_t)b * x_bs;
  for (int idx = threadIdx.x; idx < ROWS * (C / 4); idx += blockDim.x) {
    const int row = idx / (C / 4), q = idx % (C / 4);
    const int tt = t0 - 3 + row;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (tt >= 0 && tt < lim) v = *reinterpret_cast<const float4*>(xb + (size_t)tt * C + 4 * q);
    xs[4 * q + 0][row] = v.x > 0.f ? v.x : 0.01f * v.x;
    xs[4 * q + 1][row] = v.y > 0.f ? v.y : 0.01f * v.y;
    xs[4 * q + 2][row] = v.z > 0.f ? v.z : 0.01f * v.z;
    xs[4 * q + 3][row] = v.w > 0.f ? v.w : 0.01f * v.w;
  }
  __syncthreads();
  const int t = t0 + threadIdx.x;
  if (t >= y_len) return;
  float acc = 0.f;
  if (t < lim) {
#pragma unroll
    for (int k = 0; k < 7; ++k)
#pragma unroll 8
      for (int ci = 0; ci < C; ++ci) acc = fmaf(ws[k][ci], xs[ci][threadIdx.x + k], acc);
    acc = tanhf(acc);
  }
  y[(size_t)b * y_bs + t] = acc;
}

// [B][C][pitch] <-> [B][pitch][C] tiled transpose (32x32 through shared memory)
__global__ void __launch_bounds__(256) transpose_kernel(const float* __restrict__ src, float* __restrict__ dst, int rows,
                                                        int cols, long long bs) {
  __shared__ float tile[32][33];
  const float* s = src + (size_t)blockIdx.z * bs;
  float* d = dst + (size_t)blockIdx.z * bs;
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int i = ty; i < 32; i += 8) {
    const int r = r0 + i, c = c0 + tx;
    tile[i][tx] = (r < rows && c < cols) ? s[(size_t)r * cols + c] : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int c = c0 + i, r = r0 + tx;
    if (r < rows && c < cols) d[(size_t)c * rows + r] = tile[tx][i];
  }
}

}  // namespace ovc
