// kc_tcconv.cu -- test harness of the split-precision tensor-core conv (openvoice_b200/csrc/ovc_tcconv.cuh).
//
// Runs the library's own kernel (tcconv_kernel<TN, PAIR>) and packing code (ovc_tcpack.h) on buffers the caller owns,
// one launch at a time, so tests/test_gpu_kernels.py can compare single convs with an fp64 reference.  Every launch is
// checked on the host first: a configuration the fit rules refuse returns an error and never reaches the kernel.
// Built by `make -C openvoice_b200/csrc kernelcheck` into tests/kernelcheck/libovc_kc.so; the ctypes front end is
// tests/kernelcheck/kc.py.
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <utility>

#include "ovc_tcconv.cuh"
#include "ovc_tcpack.h"

using namespace ovc;

namespace {

thread_local std::string g_err;
cudaStream_t g_stream = nullptr;
int g_sms = 0;
bool g_attr_done = false;

int fail(const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_err = buf;
  return -1;
}

#define KC_CK(expr)                                                                      \
  do {                                                                                   \
    cudaError_t e_ = (expr);                                                             \
    if (e_ != cudaSuccess) return fail("%s: %s", #expr, cudaGetErrorString(e_));         \
  } while (0)

int setup() {
  if (g_stream) return 0;
  int dev = 0;
  KC_CK(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  KC_CK(cudaGetDeviceProperties(&prop, dev));
  if (prop.major != 9) return fail("the kernel is built for sm_90a, device is sm_%d%d", prop.major, prop.minor);
  if (!g_attr_done) {
    KC_CK(cudaFuncSetAttribute(tcconv_kernel<128, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TcnCfg<128, false>::SMEM_BYTES));
    KC_CK(cudaFuncSetAttribute(tcconv_kernel<64, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TcnCfg<64, false>::SMEM_BYTES));
    KC_CK(cudaFuncSetAttribute(tcconv_kernel<32, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TcnCfg<32, false>::SMEM_BYTES));
    KC_CK(cudaFuncSetAttribute(tcconv_kernel<64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TcnCfg<64, true>::SMEM_BYTES));
    KC_CK(cudaFuncSetAttribute(tcconv_kernel<32, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TcnCfg<32, true>::SMEM_BYTES));
    g_attr_done = true;
  }
  g_sms = prop.multiProcessorCount;
  KC_CK(cudaStreamCreateWithFlags(&g_stream, cudaStreamNonBlocking));
  return 0;
}

template <class... KArgs, class... Args>
cudaError_t launch_ex(void (*kernel)(KArgs...), dim3 grid, size_t smem, bool pdl, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = dim3((unsigned)TCN_THREADS, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = g_stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

}  // namespace

// one launch, every TcConvArgs field plus the launch options (pointers are device addresses, 0 = null)
struct KcConv {
  const float* x; const uint16_t* w; const float* bias; float* y; const float* r; float* s;
  const long long* lens; const long long* lens_x; const uint16_t* w2; const float* bias2;
  long long x_bs, bias_bs, y_bs, s_bs;
  int y_ld, epi, split, first, tmax, mul, has_lens_x, Cin, Ntot, K, DIL, accumulate, passes, grid_div, pdl, B;
  float slope, scale;
};

namespace {

int check_common(const KcConv* k, int TN) {
  if (!TN) return fail("conv %d -> %d (k %d, dilation %d) does not fit the tensor-core kernel", k->Cin, k->Ntot, k->K, k->DIL);
  if (!(k->slope >= 0.f && k->slope <= 1.f)) return fail("leaky_relu slope %g outside [0, 1]", (double)k->slope);
  if (k->passes != 1 && k->passes != 3) return fail("passes must be 1 or 3, not %d", k->passes);
  if (k->B < 1 || k->tmax < 1 || k->mul < 1) return fail("empty launch (B %d, tmax %d, mul %d)", k->B, k->tmax, k->mul);
  if (!k->x || !k->w || !k->bias || !k->y) return fail("x, w, bias and y are required");
  if (k->has_lens_x && !k->lens_x) return fail("has_lens_x without lens_x");
  return 0;
}

TcConvArgs to_args(const KcConv* k) {
  TcConvArgs a{};
  a.x = k->x; a.x_bs = k->x_bs; a.w = k->w; a.bias = k->bias; a.bias_bs = k->bias_bs;
  a.y = k->y; a.y_bs = k->y_bs; a.y_ld = k->y_ld; a.r = k->r; a.s = k->s; a.s_bs = k->s_bs;
  a.epi = k->epi; a.split = k->split; a.first = k->first;
  a.lens = k->lens; a.tmax = k->tmax; a.mul = k->mul; a.lens_x = k->lens_x; a.has_lens_x = k->has_lens_x;
  a.Cin = k->Cin; a.Ntot = k->Ntot; a.K = k->K; a.DIL = k->DIL;
  a.slope = k->slope; a.scale = k->scale; a.accumulate = k->accumulate; a.passes = k->passes;
  a.w2 = k->w2; a.bias2 = k->bias2;
  return a;
}

}  // namespace

extern "C" {

__attribute__((visibility("default"))) const char* kc_error() { return g_err.c_str(); }

// ---- host only: fit rules, packing, geometry
__attribute__((visibility("default"))) int kc_tile_n(int Ntot, int Cin, int K, int DIL) { return tc_tile_n(Ntot, Cin, K, DIL); }
__attribute__((visibility("default"))) int kc_ring_slots(int TN, int pair) { return tc_ring_slots(TN, pair != 0); }
__attribute__((visibility("default"))) long long kc_packed_halfs(int Ntot, int Cin, int K, int TN) {
  return (long long)tc_packed_halfs(Ntot, Cin, K, TN);
}
__attribute__((visibility("default"))) int kc_pair_fits(int C1, int N1, int K1, int D1, int C2, int N2, int K2, int D2) {
  TcGeom a, b;
  a.Cin = C1; a.Ntot = N1; a.K = K1; a.DIL = D1; a.TN = tc_tile_n(N1, C1, K1, D1);
  b.Cin = C2; b.Ntot = N2; b.K = K2; b.DIL = D2; b.TN = tc_tile_n(N2, C2, K2, D2);
  return tc_pair_fits(a, b) ? 1 : 0;
}
// w: fp32 [Ntot][Cin][K]; out: kc_packed_halfs(...) halfs.  Returns TN, or 0 (nothing written) when the conv does not fit.
__attribute__((visibility("default"))) int kc_pack(const float* w, int Ntot, int Cin, int K, int DIL, uint16_t* out) {
  const int TN = tc_tile_n(Ntot, Cin, K, DIL);
  if (!TN) return 0;
  tc_pack_weights(out, Ntot, Cin, K, TN, [&](int n, int ci, int tap) { return w[((size_t)n * Cin + ci) * K + tap]; });
  return TN;
}
// ConvTranspose1d weight [cin][cout][kk] (stride s) -> the unpacked polyphase 3-tap weight [s * cout][cin][3]
__attribute__((visibility("default"))) void kc_ups_weights(const float* raw, int cin, int cout, int kk, int s, float* out) {
  auto rw = [&](int ci, int co, int k) { return raw[((size_t)ci * cout + co) * kk + k]; };
  for (int row = 0; row < s * cout; ++row)
    for (int ci = 0; ci < cin; ++ci)
      for (int tap = 0; tap < 3; ++tap) out[((size_t)row * cin + ci) * 3 + tap] = tc_ups_weight(rw, s, kk, cout, row, ci, tap);
}
// out: {n_tt, total, grid_x, ncol}
__attribute__((visibility("default"))) void kc_grid(int t_len, int B, int Ntot, int TN, int sm_count, int grid_div, int pair, int K,
                                                    int* out) {
  const TcGrid g = pair ? tc_pair_grid(t_len, B, K, sm_count) : tc_grid(t_len, B, Ntot, TN, sm_count, grid_div);
  out[0] = g.n_tt; out[1] = g.total; out[2] = g.grid_x; out[3] = g.ncol;
}
// mutation controls on a packed array (host memory): kind 0 zeroes every lo row; kind 1 swaps the slots of taps i and j
// (every column tile and channel slot); kind 2 zeroes the hi and lo parts of 16-channel slot i of column tile j, all taps
__attribute__((visibility("default"))) int kc_corrupt(uint16_t* p, int Ntot, int Cin, int K, int TN, int kind, int i, int j) {
  if (!TN || Ntot % TN || Cin % 16) return fail("bad geometry");
  const size_t sh = tc_slot_halfs(TN);
  const int nt_n = Ntot / TN, k16_n = Cin / 16;
  for (int nt = 0; nt < nt_n; ++nt)
    for (int k16 = 0; k16 < k16_n; ++k16) {
      uint16_t* base = p + ((size_t)nt * k16_n + k16) * K * sh;
      if (kind == 0) {
        for (int tap = 0; tap < K; ++tap)
          for (int kc = 0; kc < 2; ++kc) memset(base + tap * sh + (size_t)(kc * 2 + 1) * TN * 8, 0, (size_t)TN * 8 * 2);
      } else if (kind == 1) {
        if (i < 0 || j < 0 || i >= K || j >= K) return fail("tap out of range");
        for (size_t e = 0; e < sh; ++e) std::swap(base[i * sh + e], base[j * sh + e]);
      } else if (kind == 2) {
        if (i < 0 || i >= k16_n || j < 0 || j >= nt_n) return fail("slot out of range");
        if (k16 == i && nt == j) memset(base, 0, K * sh * 2);
      } else {
        return fail("unknown corruption %d", kind);
      }
    }
  return 0;
}

// ---- device
__attribute__((visibility("default"))) int kc_sm_count() { return setup() ? -1 : g_sms; }

// one conv (PAIR = false).  w / bias are packed by kc_pack; TN follows from the geometry.
__attribute__((visibility("default"))) int kc_conv(const KcConv* k) {
  if (setup()) return -1;
  const int TN = tc_tile_n(k->Ntot, k->Cin, k->K, k->DIL);
  if (check_common(k, TN)) return -1;
  if (k->epi < 0 || k->epi > 2) return fail("epilogue %d", k->epi);
  if (k->epi == 0 && k->y_ld < k->Ntot) return fail("y_ld %d < Ntot %d", k->y_ld, k->Ntot);
  if (k->epi == 1 && k->y_ld < k->Ntot / 2) return fail("gate: y_ld %d < Ntot / 2", k->y_ld);
  if (k->epi == 2 && (k->split % 32 || k->split < 0 || k->split > k->Ntot || k->y_ld < k->split ||
                      k->y_ld < k->Ntot - k->split || (k->split < k->Ntot && !k->s)))
    return fail("res/skip: split %d, Ntot %d, y_ld %d", k->split, k->Ntot, k->y_ld);
  const TcGrid g = tc_grid(k->tmax * k->mul, k->B, k->Ntot, TN, g_sms, k->grid_div);
  const TcConvArgs a = to_args(k);
  const dim3 pg((unsigned)g.grid_x, g.ncol, 1);
  const bool pdl = k->pdl != 0;
  if (TN == 128) KC_CK(launch_ex(tcconv_kernel<128, false>, pg, TcnCfg<128, false>::SMEM_BYTES, pdl, a, g.n_tt, g.total));
  else if (TN == 64) KC_CK(launch_ex(tcconv_kernel<64, false>, pg, TcnCfg<64, false>::SMEM_BYTES, pdl, a, g.n_tt, g.total));
  else KC_CK(launch_ex(tcconv_kernel<32, false>, pg, TcnCfg<32, false>::SMEM_BYTES, pdl, a, g.n_tt, g.total));
  KC_CK(cudaGetLastError());
  return 0;
}

// one ResBlock conv pair: w / bias conv 1 (dilation DIL), w2 / bias2 conv 2 (dilation 1), residual = x, y_ld = C
__attribute__((visibility("default"))) int kc_pair(const KcConv* k) {
  if (setup()) return -1;
  const int TN = tc_tile_n(k->Ntot, k->Cin, k->K, k->DIL);
  if (check_common(k, TN)) return -1;
  TcGeom a1, a2;
  a1.Cin = k->Cin; a1.Ntot = k->Ntot; a1.K = k->K; a1.DIL = k->DIL; a1.TN = TN;
  a2 = a1; a2.DIL = 1; a2.TN = tc_tile_n(k->Ntot, k->Cin, k->K, 1);
  if (!tc_pair_fits(a1, a2)) return fail("the pair C %d, k %d, dilation %d does not fit the pair kernel", k->Cin, k->K, k->DIL);
  if (!k->w2 || !k->bias2) return fail("pair: w2 and bias2 are required");
  if (k->epi != 0 || k->r || k->has_lens_x || k->y_ld != TN) return fail("pair: linear epilogue, residual = x, y_ld = C only");
  const TcGrid g = tc_pair_grid(k->tmax * k->mul, k->B, k->K, g_sms);
  const TcConvArgs a = to_args(k);
  const dim3 pg((unsigned)g.grid_x, 1, 1);
  const bool pdl = k->pdl != 0;
  if (TN == 64) KC_CK(launch_ex(tcconv_kernel<64, true>, pg, TcnCfg<64, true>::SMEM_BYTES, pdl, a, g.n_tt, g.total));
  else KC_CK(launch_ex(tcconv_kernel<32, true>, pg, TcnCfg<32, true>::SMEM_BYTES, pdl, a, g.n_tt, g.total));
  KC_CK(cudaGetLastError());
  return 0;
}

__attribute__((visibility("default"))) int kc_sync() {
  if (setup()) return -1;
  KC_CK(cudaStreamSynchronize(g_stream));
  KC_CK(cudaGetLastError());
  return 0;
}

}  // extern "C"
