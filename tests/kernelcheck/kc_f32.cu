// kc_f32.cu -- test harness of the fp32 CUDA-core conv family (openvoice_b200/csrc/ovc_conv.cuh) and of the two
// conv_post kernels.
//
// The conv launches go through the library's own compiled instantiations (launch_<name> / prepare_<name> of
// ovc_variants.h, linked from the library's ovc_group*.o), and the weights are packed by the library's own code
// (ovc_convpack.h), so tests/test_gpu_conv_f32.py runs exactly the machine code and bytes the library ships.  The
// conv_post kernels are instantiated from their headers as the library does.  Every launch is checked on the host
// first: unknown variants, misaligned or too small buffers and inconsistent arguments return an error string and never
// reach the device.  Built by `make -C openvoice_b200/csrc kernelcheck` into tests/kernelcheck/libovc_kc_f32.so; the
// ctypes front end is tests/kernelcheck/kc_f32.py.
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <utility>

#include "ovc_convpack.h"
#include "ovc_small.cuh"
#include "ovc_tcconv.cuh"
#include "ovc_variants.h"

using namespace ovc;

namespace {

thread_local std::string g_err;
cudaStream_t g_stream = nullptr;
CallParams* g_callp = nullptr;

struct VariantEntry {
  const char* name;
  int K, DIL, CO_T, T_T, CI_CH, EPI, NG, XALIGN;
  LaunchFn launch;
  PrepareFn prepare;
};
const VariantEntry kV[V_COUNT] = {
#define X(name, K, D, WM, WN, CI, EPI, NG, XA) {#name, K, D, 32 * WM, 64 * WN, CI, EPI, NG, XA, launch_##name, prepare_##name},
    OVC_VARIANTS_ALL(X)
#undef X
};

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
  if (prop.major != 9) return fail("the kernels are built for sm_90a, device is sm_%d%d", prop.major, prop.minor);
  for (int v = 0; v < V_COUNT; ++v) KC_CK(kV[v].prepare());
  KC_CK(cudaMalloc(&g_callp, sizeof(CallParams)));
  KC_CK(cudaStreamCreateWithFlags(&g_stream, cudaStreamNonBlocking));
  return 0;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// a [B][nrows][pitch] region of which rows [0, nrows) and steps [0, width) are touched: pitch >= width and n elements
// cover the last one
int check_region(const char* what, long long n, long long bs, long long pitch, int B, long long nrows, long long width) {
  if (nrows <= 0 || width <= 0) return 0;
  if (pitch < width) return fail("%s: pitch %lld < %lld steps touched", what, pitch, width);
  if (bs < 0) return fail("%s: negative batch stride", what);
  const long long need = (long long)(B - 1) * bs + (nrows - 1) * pitch + width;
  if (n < need) return fail("%s: %lld elements, the launch touches %lld", what, n, need);
  return 0;
}

// float4 access: 16-byte base, pitch and batch stride in whole vectors
int check_vec(const char* what, const void* p, long long bs, long long pitch) {
  if (!aligned16(p) || bs % 4 || pitch % 4)
    return fail("%s: float4 access needs a 16-byte base, pitch and batch stride (got %p, %lld, %lld)", what, p, pitch, bs);
  return 0;
}

}  // namespace

// one conv1d_f32 launch: every ConvArgs field, the launch geometry, the element counts of the buffers and an optional
// device CallParams (pointers are device addresses, 0 = null)
struct KcF32 {
  const float* x; const float* w; const float* bias; float* y; const float* r; float* s;
  const long long* lens_in; const long long* lens_out;
  const unsigned long long* it_seed; const long long* it_stream; const long long* it_frame0; const float* it_tau;
  long long x_bs, bias_bs, y_bs, r_bs, s_bs;
  long long x_n, w_n, bias_n, y_n, r_n, s_n;
  unsigned long long seed, cp_seed;
  int variant, x_pitch, cin, rows, y_pitch, r_pitch, s_pitch, tmax, mul_in, mul_out, flags, split, t_len, B;
  int lens_in_n, lens_out_n, items_n, use_callp;
  float slope, scale, tau, sign, cp_tau;
};

// conv_post: y[b, t] = tanh(conv(lrelu_0.01(x), w, pad 3)), [C][pitch] (channels_last = 0) or [t][C] input
struct KcPost {
  const float* x; const float* w; float* y; const long long* lens;
  long long x_bs, x_n, w_n, y_bs, y_n;
  int x_pitch, y_len, tmax, mul, B, lens_n, channels_last;
};

namespace {

int check_conv(const KcF32* k) {
  if (k->variant < 0 || k->variant >= V_COUNT) return fail("unknown variant %d", k->variant);
  const VariantEntry& v = kV[k->variant];
  if (k->B < 1 || k->B > 65535 || k->tmax < 1 || k->mul_in < 1 || k->mul_out < 1 || k->t_len < 1 || k->cin < 1)
    return fail("%s: empty or oversized launch (B %d, tmax %d, mul %d / %d, t_len %d, cin %d)", v.name, k->B, k->tmax,
                k->mul_in, k->mul_out, k->t_len, k->cin);
  if ((long long)k->tmax * k->mul_in > INT_MAX / 16 || (long long)k->tmax * k->mul_out > INT_MAX / 16 || k->t_len > INT_MAX / 16)
    return fail("%s: time axis too long", v.name);
  if (k->rows < v.CO_T || k->rows % v.CO_T || k->rows / v.CO_T > 65535)
    return fail("%s: %d rows is not a positive multiple of the %d-row tile", v.name, k->rows, v.CO_T);
  if (k->split % v.CO_T || k->split < 0 || k->split > k->rows)
    return fail("%s: split %d is not a multiple of CO_T %d in [0, %d]", v.name, k->split, v.CO_T, k->rows);
  if (!k->x || !k->w || !k->bias || !k->y) return fail("%s: x, w, bias and y are required", v.name);
  if ((k->lens_in && k->lens_in_n < k->B) || (k->lens_out && k->lens_out_n < k->B))
    return fail("%s: lens arrays shorter than B", v.name);
  if (k->use_callp && (k->it_seed || k->it_stream || k->it_frame0 || k->it_tau) && k->items_n < k->B)
    return fail("%s: per-item arrays shorter than B", v.name);
  // x: rows [0, cin), steps below the input limit <= tmax * mul_in
  const long long in_w = (long long)k->tmax * k->mul_in;
  if (v.XALIGN == 16) {
    if (check_vec("x (16-byte cp.async)", k->x, k->x_bs, k->x_pitch)) return -1;
  } else if (reinterpret_cast<uintptr_t>(k->x) & 3) {
    return fail("x: 4-byte cp.async needs a 4-byte aligned base");
  }
  if (check_region("x", k->x_n, k->x_bs, k->x_pitch, k->B, k->cin, in_w)) return -1;
  if (!aligned16(k->w)) return fail("w: the TMA bulk copy needs a 16-byte aligned base");
  const long long wn = (long long)conv_packed_floats(k->rows, k->cin, v.K, v.CO_T, v.CI_CH);
  if (k->w_n < wn) return fail("w: %lld floats, the packed conv has %lld", k->w_n, wn);
  // outputs: steps below min(out limit, the grid's time tiles)
  const long long n_tt = (k->t_len + v.T_T - 1) / v.T_T;
  const long long tw = std::min((long long)k->tmax * k->mul_out, n_tt * v.T_T);
  const bool per_item_bias = v.EPI == EPI_LINEAR || v.EPI == EPI_GATE;
  const long long bias_rows = v.EPI == EPI_UPS8 ? k->rows / 8 : v.EPI == EPI_UPS2 ? k->rows / 2 : k->rows;
  const long long bias_need = (per_item_bias ? (long long)(k->B - 1) * k->bias_bs : 0) + bias_rows;
  if (k->bias_bs < 0 || k->bias_n < bias_need) return fail("bias: %lld floats, the launch reads %lld", k->bias_n, bias_need);
  long long y_rows = k->rows, y_width = tw;
  switch (v.EPI) {
    case EPI_GATE: case EPI_PROJ: y_rows = k->rows / 2; break;
    case EPI_RESSKIP: y_rows = k->split; break;
    case EPI_UPS8: y_rows = k->rows / 8; y_width = 8 * tw; break;
    case EPI_UPS2: y_rows = k->rows / 2; y_width = 2 * tw; break;
    default: break;
  }
  const bool y_vec = v.EPI != EPI_PROJ && v.EPI != EPI_COUPLE;
  if (y_vec && check_vec("y", k->y, k->y_bs, k->y_pitch)) return -1;
  if (check_region("y", k->y_n, k->y_bs, k->y_pitch, k->B, y_rows, y_width)) return -1;
  if (v.EPI == EPI_RESSKIP && k->split < k->rows) {
    if (!k->s) return fail("%s: rows past split %d go to s, which is null", v.name, k->split);
    if (check_vec("s", k->s, k->s_bs, k->s_pitch)) return -1;
    if (check_region("s", k->s_n, k->s_bs, k->s_pitch, k->B, k->rows - k->split, tw)) return -1;
  }
  if (k->r && v.EPI == EPI_LINEAR) {
    if (check_vec("r", k->r, k->r_bs, k->r_pitch)) return -1;
    if (check_region("r", k->r_n, k->r_bs, k->r_pitch, k->B, k->rows, tw)) return -1;
  }
  if (k->r && v.EPI == EPI_PROJ && check_region("noise", k->r_n, k->r_bs, k->r_pitch, k->B, k->rows / 2, tw)) return -1;
  if (k->r && v.EPI != EPI_LINEAR && v.EPI != EPI_PROJ) return fail("%s: r is read by LINEAR and PROJ only", v.name);
  return 0;
}

ConvArgs to_args(const KcF32* k) {
  const VariantEntry& v = kV[k->variant];
  ConvArgs a{};
  a.x = k->x; a.x_bs = k->x_bs; a.x_pitch = k->x_pitch; a.cin = k->cin;
  a.w = k->w; a.bias = k->bias; a.bias_bs = k->bias_bs;
  a.n_chunks = (k->cin + v.CI_CH - 1) / v.CI_CH;
  a.y = k->y; a.y_bs = k->y_bs; a.y_pitch = k->y_pitch;
  a.r = k->r; a.r_bs = k->r_bs; a.r_pitch = k->r_pitch;
  a.s = k->s; a.s_bs = k->s_bs; a.s_pitch = k->s_pitch;
  a.lens_in = k->lens_in; a.lens_out = k->lens_out; a.tmax = k->tmax; a.mul_in = k->mul_in; a.mul_out = k->mul_out;
  a.slope = k->slope; a.scale = k->scale; a.tau = k->tau; a.sign = k->sign;
  a.flags = k->flags; a.split = k->split; a.seed = k->seed;
  a.callp = k->use_callp ? g_callp : nullptr;
  return a;
}

int check_post(const KcPost* k) {
  if (k->B < 1 || k->B > 65535 || k->tmax < 1 || k->mul < 1 || k->y_len < 1)
    return fail("conv_post: empty or oversized launch (B %d, tmax %d, mul %d, y_len %d)", k->B, k->tmax, k->mul, k->y_len);
  if ((long long)k->tmax * k->mul > INT_MAX / 16 || k->y_len > INT_MAX / 16) return fail("conv_post: time axis too long");
  if (!k->x || !k->w || !k->y) return fail("conv_post: x, w and y are required");
  if (k->lens && k->lens_n < k->B) return fail("conv_post: lens shorter than B");
  if (k->w_n < 32 * 7) return fail("conv_post: w has %lld floats, not 224", k->w_n);
  const long long lim = (long long)k->tmax * k->mul;
  if (k->channels_last) {
    if (check_vec("x", k->x, k->x_bs, 32)) return -1;
    if (check_region("x", k->x_n, k->x_bs, 32 * lim, k->B, 1, 32 * lim)) return -1;
  } else {
    // whole float4 stores of 4 samples: y_len must be a multiple of 4 or the last store runs past it
    if (k->y_len % 4) return fail("conv_post [C][pitch]: y_len %d is not a multiple of 4", k->y_len);
    if (check_vec("x", k->x, k->x_bs, k->x_pitch) || check_vec("y", k->y, k->y_bs, 4)) return -1;
    if (check_region("x", k->x_n, k->x_bs, k->x_pitch, k->B, 32, (lim + 3) / 4 * 4)) return -1;
  }
  return check_region("y", k->y_n, k->y_bs, k->y_len, k->B, 1, k->y_len);
}

}  // namespace

extern "C" {

__attribute__((visibility("default"))) const char* kc_error() { return g_err.c_str(); }

// ---- host only: the variant table, packing, interleave and polyphase map
__attribute__((visibility("default"))) int kc_variant_count() { return V_COUNT; }
// out: {K, DIL, CO_T, T_T, CI_CH, EPI, NG, XALIGN}; returns the name, NULL for an unknown variant
__attribute__((visibility("default"))) const char* kc_variant(int v, int* out) {
  if (v < 0 || v >= V_COUNT) return nullptr;
  const VariantEntry& q = kV[v];
  const int f[8] = {q.K, q.DIL, q.CO_T, q.T_T, q.CI_CH, q.EPI, q.NG, q.XALIGN};
  memcpy(out, f, sizeof f);
  return q.name;
}
__attribute__((visibility("default"))) long long kc_packed_floats(int v, int rows, int cin) {
  if (v < 0 || v >= V_COUNT) return -1;
  return (long long)conv_packed_floats(rows, cin, kV[v].K, kV[v].CO_T, kV[v].CI_CH);
}
__attribute__((visibility("default"))) int kc_paired_row(int p, int half) { return paired_row(p, half); }
__attribute__((visibility("default"))) int kc_ups_kidx(int s, int kk, int row, int tap) { return conv_ups_kidx(s, kk, row, tap); }
// the (tap, packed row mod 8) pairs the transposed-conv kernels skip
__attribute__((visibility("default"))) int kc_tap_is_zero(int s, int k, int r) {
  return s == 8 ? tap_is_zero<EPI_UPS8>(k, r) : tap_is_zero<EPI_UPS2>(k, r);
}
// w: [rows][cin][K] in natural row order; paired = 1 reads row paired_row(p, rows / 2) for packed row p (the gate and
// projection layouts).  out: kc_packed_floats(v, rows, cin) floats.
__attribute__((visibility("default"))) int kc_pack(int v, const float* w, int rows, int cin, int paired, float* out) {
  if (v < 0 || v >= V_COUNT) return fail("unknown variant %d", v);
  const VariantEntry& q = kV[v];
  if (rows < q.CO_T || rows % q.CO_T || cin < 1) return fail("%s: %d rows, cin %d", q.name, rows, cin);
  const int K = q.K;
  conv_pack_weights(out, rows, cin, K, q.CO_T, q.CI_CH, [&](int p, int ci, int k) {
    const int row = paired ? paired_row(p, rows / 2) : p;
    return w[((size_t)row * cin + ci) * K + k];
  });
  return 0;
}
// raw ConvTranspose1d weight [cin][cout][kk] of stride s -> the packed polyphase conv of an UPS8 / UPS2 variant
__attribute__((visibility("default"))) int kc_pack_ups(int v, const float* raw, int cin, int cout, int kk, int s, float* out) {
  if (v < 0 || v >= V_COUNT) return fail("unknown variant %d", v);
  const VariantEntry& q = kV[v];
  if (q.EPI != (s == 8 ? EPI_UPS8 : EPI_UPS2) || (s != 8 && s != 2) || kk != 2 * s || (cout * s) % q.CO_T)
    return fail("%s: transposed conv %d -> %d, stride %d, kernel %d", q.name, cin, cout, s, kk);
  auto rw = [&](int ci, int co, int k) { return raw[((size_t)ci * cout + co) * kk + k]; };
  conv_pack_weights(out, cout * s, cin, 3, q.CO_T, q.CI_CH,
                    [&](int row, int ci, int tap) { return conv_ups_weight(rw, s, kk, row, ci, tap); });
  return 0;
}
// mutation controls on a packed array (host memory): kind 0 swaps taps i and j of every row tile and channel; kind 1
// zeroes ci-chunk i of row tile j (every channel of the chunk, every tap and row)
__attribute__((visibility("default"))) int kc_corrupt(int v, float* p, int rows, int cin, int kind, int i, int j) {
  if (v < 0 || v >= V_COUNT) return fail("unknown variant %d", v);
  const VariantEntry& q = kV[v];
  const int K = q.K, cin_pad = conv_cin_pad(cin, q.CI_CH), row_tiles = rows / q.CO_T;
  if (kind == 0) {
    if (i < 0 || j < 0 || i >= K || j >= K || i == j) return fail("taps %d, %d of %d", i, j, K);
    for (int rt = 0; rt < row_tiles; ++rt)
      for (int ci = 0; ci < cin_pad; ++ci) {
        float* b = p + ((size_t)rt * cin_pad + ci) * K * q.CO_T;
        for (int r = 0; r < q.CO_T; ++r) std::swap(b[i * q.CO_T + r], b[j * q.CO_T + r]);
      }
  } else if (kind == 1) {
    if (i < 0 || i >= cin_pad / q.CI_CH || j < 0 || j >= row_tiles) return fail("chunk %d of row tile %d", i, j);
    memset(p + ((size_t)j * cin_pad + (size_t)i * q.CI_CH) * K * q.CO_T, 0, sizeof(float) * q.CI_CH * K * q.CO_T);
  } else {
    return fail("unknown corruption %d", kind);
  }
  return 0;
}

// ---- device
__attribute__((visibility("default"))) int kc_setup() { return setup(); }

__attribute__((visibility("default"))) int kc_conv(const KcF32* k) {
  if (setup() || check_conv(k)) return -1;
  const VariantEntry& v = kV[k->variant];
  if (k->use_callp) {
    CallParams cp{};
    cp.seed = k->cp_seed; cp.tau = k->cp_tau;
    cp.items.seed = k->it_seed; cp.items.stream = k->it_stream; cp.items.frame0 = k->it_frame0; cp.items.tau = k->it_tau;
    KC_CK(cudaMemcpyAsync(g_callp, &cp, sizeof cp, cudaMemcpyHostToDevice, g_stream));
    KC_CK(cudaStreamSynchronize(g_stream));
  }
  KC_CK(v.launch(to_args(k), k->t_len, k->rows / v.CO_T, k->B, g_stream));
  return 0;
}

__attribute__((visibility("default"))) int kc_conv_post(const KcPost* k) {
  if (setup() || check_post(k)) return -1;
  if (k->channels_last) {
    const dim3 grid((k->y_len + 255) / 256, k->B);
    conv_post_cl_kernel<32><<<grid, 256, 0, g_stream>>>(k->x, k->x_bs, k->w, k->y, k->y_bs, k->y_len, k->lens, k->tmax, k->mul);
  } else {
    const dim3 grid((k->y_len / 4 + 255) / 256, k->B);
    conv_post_kernel<32><<<grid, 256, 0, g_stream>>>(k->x, k->x_bs, k->x_pitch, k->w, k->y, k->y_bs, k->y_len, k->lens,
                                                     k->tmax, k->mul);
  }
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
