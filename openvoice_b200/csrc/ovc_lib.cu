// ovc_lib.cu -- host side of libovc_b200.so: context, checkpoint ingestion (weight-norm folding,
// Flip absorption, kernel-layout packing), workspace arena, the launch sequence of
// SynthesizerTrn.voice_conversion (openvoice/models.py:492-499) and the C ABI of include/ovc.h.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/ovc.h"
#include "ovc_convpack.h"
#include "ovc_small.cuh"
#include "ovc_tcconv.cuh"
#include "ovc_tts.cuh"
#include "ovc_refenc.cuh"
#include "ovc_resample.cuh"
#include "ovc_splice.h"
#include "ovc_variants.h"

namespace ovc {

static thread_local std::string g_err;

static int fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}

// every ABI entry point runs on its context's device and puts the caller's current device back on exit (PyTorch
// reads the current device through cudaGetDevice: a converter on cuda:N must not move the caller's default)
struct DeviceGuard {
  int prev = -1;
  bool ok = true;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != dev) ok = cudaSetDevice(dev) == cudaSuccess;
  }
  ~DeviceGuard() {
    int cur = -1;
    if (prev >= 0 && cudaGetDevice(&cur) == cudaSuccess && cur != prev) cudaSetDevice(prev);
  }
};
#define ON_DEVICE(c)                                                                              \
  DeviceGuard dev_guard_((c)->device);                                                            \
  if (!dev_guard_.ok) return fail(OVC_ERR_CUDA, "cudaSetDevice(%d) failed", (c)->device)

#define CK(expr)                                                                                  \
  do {                                                                                            \
    cudaError_t e_ = (expr);                                                                      \
    if (e_ != cudaSuccess)                                                                        \
      return fail(OVC_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, \
                  __LINE__);                                                                      \
  } while (0)

#define TRY(expr)                   \
  do {                              \
    int rc_ = (expr);               \
    if (rc_ != OVC_OK) return rc_;  \
  } while (0)

static const VariantInfo kInfo[V_COUNT] = {
#define X(name, K, D, WM, WN, CI, EPI, NG, XA)                                                    \
  {#name, K, D, 32 * WM, 64 * WN, CI, EPI, 32 * WM * WN, ConvCfg<K, D, WM, WN, CI, EPI, NG, XA>::SMEM_BYTES},
    OVC_VARIANTS_ALL(X)
#undef X
};
static const LaunchFn kLaunch[V_COUNT] = {
#define X(name, K, D, WM, WN, CI, EPI, NG, XA) launch_##name,
    OVC_VARIANTS_ALL(X)
#undef X
};
static const PrepareFn kPrepare[V_COUNT] = {
#define X(name, K, D, WM, WN, CI, EPI, NG, XA) prepare_##name,
    OVC_VARIANTS_ALL(X)
#undef X
};

struct HostTensor {
  std::vector<int64_t> shape;
  std::vector<float> data;
  int64_t numel() const {
    int64_t n = 1;
    for (auto s : shape) n *= s;
    return n;
  }
};

// one convolution as the kernels see it
struct ConvLayer {
  int variant = -1;
  int rows = 0;        // packed output rows (multiple of CO_T)
  int row_tiles = 0;
  int cin = 0;         // real input channels
  int n_chunks = 0;
  size_t w_off = 0;    // float offsets into the device weight arena
  size_t b_off = 0;
  int K = 1;           // true taps / channels, for FLOP accounting
  int cout = 0;
  int out_mul = 1;     // outputs per input step (transposed convs: stride)
};

// one ResBlock conv as the tensor-core kernel sees it (pre-split hi/lo weights in operand layout)
struct TcLayer : TcGeom {
  size_t w_off = 0;   // float offsets into the tc weight arena
  size_t b_off = 0;
};

struct WNLayers {
  std::vector<ConvLayer> in, rs;
  std::vector<TcLayer> tc_in, tc_rs;   // tensor-core twins (channels-last)
};

// V1 TTS front half (TextEncoder / DurationPredictor / StochasticDurationPredictor, models.py:16-180): dense convs
// as tensor-core layers, small fp32 parameters as offsets into the fp32 arena.  Hyper-parameters are read off the
// checkpoint shapes (the reference takes them from config.json: api.py:26-31, models.py:451-465).
// k = 3 convs and the whole duration chain stay on the CUDA cores in plain fp32: the FFMA conv kernel on a [C][T]
// copy when the shape fits a variant (k 3, N % 64 == 0: every released checkpoint), else the one-thread-per-output
// kernel (sequential fmaf chain over w [K][Cin][N])
struct Fp32Dense { size_t w = 0, b = 0; int Cin = 0, K = 0, N = 0; bool fast = false; ConvLayer cl; };
struct DdsLayers {            // DDSConv, modules.py:84-113
  size_t sep_w[3] = {0}, sep_b[3] = {0}, n1g[3] = {0}, n1b[3] = {0}, n2g[3] = {0}, n2b[3] = {0};
  Fp32Dense c1x1[3];          // fp32: the spline inverses downstream amplify conditioning errors up to 1e3 x
};
struct TtsLayers {
  bool ready = false;
  int n_vocab = 0, n_speakers = 0, H = 0, C = 0, Fc = 0, heads = 0, n_layers = 0, window = 0, D = 0;
  size_t emb = 0, emb_g = 0;
  std::vector<TcLayer> qkv, o;
  std::vector<Fp32Dense> ffn1, ffn2;
  std::vector<size_t> relk, relv, ln1g, ln1b, ln2g, ln2b;
  TcLayer proj;
  Fp32Dense dp_c1, dp_c2, sdp_pre, sdp_proj;
  size_t dp_n1g = 0, dp_n1b = 0, dp_n2g = 0, dp_n2b = 0, dp_pw = 0, dp_pb = 0, dp_cw = 0, dp_cb = 0, sdp_cw = 0, sdp_cb = 0,
         ea = 0;               // ea: {m[0], logs[0]} of sdp.flows.0
  DdsLayers dds[4];            // 0: sdp.convs, j = 1..3: sdp.flows.{2j+1}.convs (flows.1 is never run in reverse, models.py:172)
  size_t cf_pre_w[4] = {0}, cf_pre_b[4] = {0}, cf_pw[4] = {0}, cf_pb[4] = {0};
};

struct DebugBuf {
  float* d = nullptr;
  int64_t shape[4] = {0, 0, 0, 0};
  size_t floats = 0;
};

}  // namespace ovc

using namespace ovc;

struct ovc_ctx {
  ovc_hparams hp{};
  int device = 0;
  int sm_count = 0;
  std::map<std::string, HostTensor> sd;
  bool finalized = false;

  // device weights
  float* d_w = nullptr;
  size_t w_floats = 0;
  std::vector<float> h_w;   // staging while packing

  // layers
  ConvLayer enc_pre, enc_pre16, enc_proj;
  WNLayers enc_wn;
  ConvLayer flow_pre[4], flow_post[4];
  WNLayers flow_wn[4];
  ConvLayer dec_pre, dec_ups[4];
  ConvLayer rb_c1[12][3], rb_c2[12][3];
  TcLayer tc_c1[12][3], tc_c2[12][3], tc_ups[4], tc_pre;
  float* d_tcw = nullptr;      // tensor-core weight arena (hi/lo split)
  std::vector<float> h_tcw;
  int precision = 0;           // 0: fp32 FFMA everywhere; 1: 3xFP16 split-precision wgmma convs; 2: single-pass fp16
  bool tts_simple = false;     // OVC_OPT_TTS_SIMPLE
  bool use_graph = true;       // OVC_OPT_GRAPH
  int use_pdl = 2;             // OVC_OPT_PDL: 0 off, 1 every tensor-core conv, 2 (default) the WaveNet stacks only -- short kernels
                               // whose fill / drain dominates
  // small calls: the three ResBlock branches of an MRF stage run concurrently on three streams, each kernel on a third
  // of the SMs (OVC_OPT_BRANCHES; taken when B * Tmax <= par_frames = 512 frames)
  bool use_branches = true;
  int par_frames = 512;
  bool use_pair = true;        // OVC_OPT_PAIR: the ResBlock conv pairs of the C <= 128 stages as ONE kernel (tcconv_kernel<C, true>, tc_pair_fuses)
  bool use_pair_occ = true;    // OVC_OPT_PAIR_OCC: pairs run two CTAs per SM where tc_pair_occ picks it
  bool use_staged_epi = true;  // OVC_OPT_STAGED_EPI: the TN = 128 convs and C = 128 pairs hand their epilogue to a store warpgroup
  bool pair_occ2_ok[TCN_N_OCC2] = {};   // the device fits two CTAs per SM of kTcPairOcc2[i] (occupancy query at load)
  cudaStream_t br_stream[2] = {nullptr, nullptr};
  cudaEvent_t br_ev[4] = {nullptr, nullptr, nullptr, nullptr};
  size_t post_w_off = 0;
  // cond mat-vec
  size_t cond_w_off = 0, cond_b_off = 0;
  int* d_cond_wrow = nullptr;
  int* d_cond_sel = nullptr;
  int cond_rows_out = 0;
  int cond_off_enc = 0, cond_off_fsrc = 0, cond_off_ftgt = 0, cond_off_dec = 0;
  int cond_off_enc_tc = 0, cond_off_fsrc_tc = 0, cond_off_ftgt_tc = 0;   // same vectors in the tc kernel's column order
  // per-frame conditioning (a side whose embedding varies over time): the output columns of the sections that read a
  // varying side, for column order o (0 fp32 kernels, 1 tensor cores) and varying sides m (1 src, 2 tgt, 3 both; index
  // m - 1); cond_pf_off: column of section enc / flow src / flow tgt / dec in that vector, -1 = the per-item vector
  int* d_cond_cols[2][3] = {};
  int cond_pf_cols[2][3] = {};
  int cond_pf_off[2][3][4] = {};

  // STFT tables (twiddles exp(-2 pi i m / 1024), periodic hann window)
  float2* d_tw = nullptr;
  float* d_win = nullptr;

  // ReferenceEncoder (extract_se): offsets into d_w, own scratch
  bool has_refenc = false;
  size_t re_conv_w[6] = {0}, re_conv_b[6] = {0}, re_wih = 0, re_whh = 0, re_bih = 0, re_bhh = 0, re_pw = 0, re_pb = 0,
         re_lng = 0, re_lnb = 0;
  int re_gru_in = 0;           // columns of ref_enc.gru.weight_ih_l0
  float* d_re = nullptr;
  size_t re_floats = 0;
  float* d_res = nullptr;      // ovc_reference_encoder_stream: spectrogram columns and layer rows of its items
  size_t res_floats = 0;

  // ovc_resample: one fp64 polyphase bank per reduced (up, down) pair, built on first use and kept
  std::map<std::pair<int64_t, int64_t>, double*> rs_banks;
  bool rs_smem_opt_in = false;   // resample_kernel's dynamic shared-memory limit raised (once per context)
  // ovc_resample_plan: the plan table of ovc_resample_rings (banks shared with rs_banks), and the tile and shared memory
  // that fit its worst plan
  std::vector<RsRingPlan> rs_plans;
  RsRingPlan* d_rs_plans = nullptr;
  int rs_ring_tile = 256;
  size_t rs_ring_smem = 0;

  // workspace
  float* d_ws = nullptr;
  size_t ws_floats = 0;

  // TTS front half: layers, text-side workspace, and what ovc_tts_encode leaves for ovc_tts_decode
  TtsLayers tts;
  float* d_tts = nullptr;
  size_t tts_floats = 0;
  int tts_B = 0, tts_T = 0;
  bool tts_gtok = false;   // the pending encode took per-token speaker vectors

  // profiling
  bool prof = false;
  std::vector<cudaEvent_t> ev;
  size_t ev_used = 0;
  double prof_ms = 0, prof_flops = 0, prof_bytes = 0;
  int64_t prof_launches = 0;
  std::vector<double> ev_flops, ev_bytes;
  std::vector<int> ev_variant, ev_family, ev_tag;   // tag: (Cin << 16 | K << 8 | dilation) of a tensor-core launch, else 0

  // debug taps
  bool debug = false;
  std::map<std::string, DebugBuf> taps;

  int launches = 0;

  // CUDA-graph replay of a repeated call (OVC_OPT_GRAPH): the launch sequence of a (entry point, shapes, buffers,
  // options) signature is captured on an internal stream the second time it is seen and replayed from then on; the
  // per-call scalars (noise seed, tau) reach the kernels through d_callp
  struct GraphEntry {
    std::vector<uintptr_t> key;
    cudaGraphExec_t exec = nullptr;
    int launches = 0;
    int seen = 0;
    uint64_t stamp = 0;
  };
  std::vector<GraphEntry> graphs;
  uint64_t graph_clock = 0;
  cudaStream_t cap_stream = nullptr;
  ovc::CallParams* d_callp = nullptr;
  int graph_replays = 0;       // diagnostics: calls served by a replay since creation
};

namespace ovc {

static size_t round_up(size_t v, size_t m) { return (v + m - 1) / m * m; }
static void drop_graphs(ovc_ctx* c);

static const HostTensor* find(const ovc_ctx* c, const std::string& k) {
  auto it = c->sd.find(k);
  return it == c->sd.end() ? nullptr : &it->second;
}

static std::string shape_str(const std::vector<int64_t>& shape) {
  std::string s = "[";
  for (size_t i = 0; i < shape.size(); ++i) s += (i ? ", " : "") + (shape[i] < 0 ? std::string("*") : std::to_string(shape[i]));
  return s + "]";
}

// checkpoint tensor `key` of the given shape (-1: any size, a dim the caller reads a hyper-parameter from).  Every
// tensor the packing code indexes comes through here or conv_weight, so no index can run past a tensor's end.
static int tensor(const ovc_ctx* c, const std::string& key, const std::vector<int64_t>& shape, const HostTensor** out) {
  const HostTensor* t = find(c, key);
  if (!t) return fail(OVC_ERR_MISSING, "checkpoint tensor '%s' is missing", key.c_str());
  bool ok = t->shape.size() == shape.size();
  for (size_t i = 0; ok && i < shape.size(); ++i) ok = shape[i] < 0 || t->shape[i] == shape[i];
  if (!ok)
    return fail(OVC_ERR_INVALID, "checkpoint tensor '%s' has shape %s, expected %s", key.c_str(), shape_str(t->shape).c_str(),
                shape_str(shape).c_str());
  *out = t;
  return OVC_OK;
}

// effective weight of a (possibly weight-normed) conv: `.weight`, or g * v / ||v|| over dims != 0 with one g per
// slice of v's dim 0 (torch.nn.utils.weight_norm dim=0; modules.py:160,172,182, models.py:247)
static int conv_weight(const ovc_ctx* c, const std::string& prefix, const std::vector<int64_t>& shape, HostTensor* out) {
  const HostTensor *v, *g;
  if (find(c, prefix + ".weight")) {
    TRY(tensor(c, prefix + ".weight", shape, &v));
    *out = *v;
    return OVC_OK;
  }
  TRY(tensor(c, prefix + ".weight_v", shape, &v));
  const int64_t d0 = v->shape[0];
  const int64_t inner = v->numel() / d0;
  if (!(g = find(c, prefix + ".weight_g"))) return fail(OVC_ERR_MISSING, "checkpoint tensor '%s.weight_g' is missing", prefix.c_str());
  if (g->numel() != d0)
    return fail(OVC_ERR_INVALID, "checkpoint tensor '%s.weight_g' has shape %s, expected %lld elements", prefix.c_str(),
                shape_str(g->shape).c_str(), (long long)d0);
  *out = *v;
  for (int64_t i = 0; i < d0; ++i) {
    double ss = 0;
    for (int64_t j = 0; j < inner; ++j) { const double q = v->data[i * inner + j]; ss += q * q; }
    const float scale = g->data[i] / (float)std::sqrt(ss);
    for (int64_t j = 0; j < inner; ++j) out->data[i * inner + j] = v->data[i * inner + j] * scale;
  }
  return OVC_OK;
}

// append a plain fp32 blob to a weight arena; returns its (256-byte aligned) float offset
static size_t append(std::vector<float>& arena, const std::vector<float>& v) {
  const size_t o = round_up(arena.size(), 64);
  arena.resize(o + v.size());
  std::copy(v.begin(), v.end(), arena.begin() + o);
  return o;
}

// append a packed conv to the staging arena.  wfun(row_packed, ci, k) -> weight; bfun(row) -> bias
template <class WF, class BF>
static ConvLayer pack_conv(ovc_ctx* c, int variant, int rows, int cin, WF wfun, BF bfun, int bias_rows,
                           int trueK, int cout) {
  const VariantInfo& vi = kInfo[variant];
  ConvLayer L;
  L.variant = variant;
  L.rows = rows;
  L.row_tiles = rows / vi.CO_T;
  L.cin = cin;
  L.n_chunks = (cin + vi.CI_CH - 1) / vi.CI_CH;
  L.K = trueK;
  L.cout = cout;
  L.w_off = round_up(c->h_w.size(), 64);   // 256-byte aligned blobs (TMA bulk needs 16)
  c->h_w.resize(L.w_off + conv_packed_floats(rows, cin, vi.K, vi.CO_T, vi.CI_CH), 0.f);
  conv_pack_weights(c->h_w.data() + L.w_off, rows, cin, vi.K, vi.CO_T, vi.CI_CH, wfun);
  L.b_off = round_up(c->h_w.size(), 64);
  c->h_w.resize(L.b_off + bias_rows, 0.f);
  for (int r = 0; r < bias_rows; ++r) c->h_w[L.b_off + r] = bfun(r);
  return L;
}

// column order of the tensor-core WN gate: every 32-column group = 16 tanh rows then their 16 sigmoid partners
static inline int paired_row32(int p, int half) {
  const int g = p / 32, r = p % 32;
  return r < 16 ? 16 * g + r : half + 16 * g + (r - 16);
}

static int dec_variant(int C, int K, int D) {
  const int cls = C >= 128 ? 0 : (C == 64 ? 1 : 2);
  static const int tab[3][3][3] = {
      {{V_A_K3D1, V_A_K3D3, V_A_K3D5}, {V_A_K7D1, V_A_K7D3, V_A_K7D5}, {V_A_K11D1, V_A_K11D3, V_A_K11D5}},
      {{V_B_K3D1, V_B_K3D3, V_B_K3D5}, {V_B_K7D1, V_B_K7D3, V_B_K7D5}, {V_B_K11D1, V_B_K11D3, V_B_K11D5}},
      {{V_C_K3D1, V_C_K3D3, V_C_K3D5}, {V_C_K7D1, V_C_K7D3, V_C_K7D5}, {V_C_K11D1, V_C_K11D3, V_C_K11D5}}};
  const int ki = K == 3 ? 0 : (K == 7 ? 1 : 2);
  const int di = D == 1 ? 0 : (D == 3 ? 1 : 2);
  return tab[cls][ki][di];
}

static int validate_hparams(const ovc_hparams* hp) {
  if (hp->inter_channels != 192 || hp->hidden_channels != 192)
    return fail(OVC_ERR_INVALID, "kernels are specialised for inter_channels = hidden_channels = 192 (got %d, %d)",
                hp->inter_channels, hp->hidden_channels);
  if (hp->spec_channels < 1 || hp->spec_channels > 4096) return fail(OVC_ERR_INVALID, "bad spec_channels %d", hp->spec_channels);
  if (hp->gin_channels < 1 || hp->gin_channels > 4096) return fail(OVC_ERR_INVALID, "bad gin_channels %d", hp->gin_channels);
  if (hp->resblock != 1) return fail(OVC_ERR_INVALID, "only resblock \"1\" (ResBlock1) is supported, got %d", hp->resblock);
  if (hp->n_resblock_kernels != 3 || hp->resblock_kernel_sizes[0] != 3 || hp->resblock_kernel_sizes[1] != 7 ||
      hp->resblock_kernel_sizes[2] != 11)
    return fail(OVC_ERR_INVALID, "resblock_kernel_sizes must be [3,7,11]");
  for (int j = 0; j < 3; ++j)
    if (hp->resblock_dilations[j][0] != 1 || hp->resblock_dilations[j][1] != 3 || hp->resblock_dilations[j][2] != 5)
      return fail(OVC_ERR_INVALID, "resblock_dilation_sizes must be [[1,3,5]]*3");
  static const int ur[4] = {8, 8, 2, 2}, uk[4] = {16, 16, 4, 4};
  if (hp->n_upsamples != 4) return fail(OVC_ERR_INVALID, "need 4 upsample stages");
  for (int i = 0; i < 4; ++i)
    if (hp->upsample_rates[i] != ur[i] || hp->upsample_kernel_sizes[i] != uk[i])
      return fail(OVC_ERR_INVALID, "upsample_rates/kernel_sizes must be [8,8,2,2]/[16,16,4,4]");
  if (hp->upsample_initial_channel != 512) return fail(OVC_ERR_INVALID, "upsample_initial_channel must be 512");
  if (hp->hop_length != 256) return fail(OVC_ERR_INVALID, "hop_length must be 256");
  return OVC_OK;
}

static bool key_is_hot(const std::string& k) {
  if (k.rfind("sdp.post_", 0) == 0) return false;   // training-only half of the SDP (models.py:118-125)
  return k.rfind("enc_q.", 0) == 0 || k.rfind("flow.", 0) == 0 || k.rfind("dec.", 0) == 0 || k.rfind("ref_enc.", 0) == 0 ||
         k.rfind("enc_p.", 0) == 0 || k.rfind("dp.", 0) == 0 || k.rfind("sdp.", 0) == 0 || k.rfind("emb_g.", 0) == 0;
}

// tensor-core copy of a conv: fp16 [n_tile][Cin/16][K][column block][hi|lo][TN][8]: hi = fp16(w), lo = fp16((w - hi) * 2^11)
// (ovc_tcpack.h), laid out exactly as the kernel's shared-memory operand slots (one TMA bulk copy per slot)
template <class WF, class BF>
static TcLayer pack_tc(ovc_ctx* c, int Ntot, int Cin, int K, int DIL, WF wfun, BF bfun) {
  TcLayer T;
  T.Cin = Cin; T.Ntot = Ntot; T.K = K; T.DIL = DIL;
  T.TN = tc_tile_n(Ntot, Cin, K, DIL);
  if (!T.TN) return T;
  T.w_off = round_up(c->h_tcw.size(), 64);
  c->h_tcw.resize(T.w_off + tc_packed_halfs(Ntot, Cin, K, T.TN) / 2, 0.f);
  tc_pack_weights(reinterpret_cast<uint16_t*>(c->h_tcw.data() + T.w_off), Ntot, Cin, K, T.TN, wfun);
  T.b_off = round_up(c->h_tcw.size(), 64);
  c->h_tcw.resize(T.b_off + Ntot, 0.f);
  for (int n = 0; n < Ntot; ++n) c->h_tcw[T.b_off + n] = bfun(n);
  return T;
}

// WN stack (modules.py:133-183): every layer folded once, packed for the FFMA kernels into h_w and for the
// tensor-core kernels into h_tcw.  The in_layer biases reach the kernels through the conditioning vector.
static int pack_wn(ovc_ctx* c, const std::string& prefix, int n_layers, WNLayers* out) {
  const int H = 192;
  *out = WNLayers();
  for (int i = 0; i < n_layers; ++i) {
    HostTensor w, r;
    const HostTensor* rb;
    const std::string prs = prefix + ".res_skip_layers." + std::to_string(i);
    const int rows = (i < n_layers - 1) ? 2 * H : H;
    TRY(conv_weight(c, prefix + ".in_layers." + std::to_string(i), {2 * H, H, 5}, &w));
    TRY(conv_weight(c, prs, {rows, H, 1}, &r));
    TRY(tensor(c, prs + ".bias", {rows}, &rb));
    out->in.push_back(pack_conv(
        c, V_WN_IN, 2 * H, H,
        [&](int p, int ci, int k) { return w.data[((size_t)paired_row(p, H) * H + ci) * 5 + k]; },
        [&](int) { return 0.f; }, 0, 5, 2 * H));
    out->rs.push_back(pack_conv(
        c, V_WN_RS, rows, H, [&](int p, int ci, int) { return r.data[(size_t)p * H + ci]; },
        [&](int p) { return rb->data[p]; }, rows, 1, rows));
    out->tc_in.push_back(pack_tc(
        c, 2 * H, H, 5, 1, [&](int p, int ci, int k) { return w.data[((size_t)paired_row32(p, H) * H + ci) * 5 + k]; },
        [&](int) { return 0.f; }));
    out->tc_rs.push_back(pack_tc(
        c, rows, H, 1, 1, [&](int p, int ci, int) { return r.data[(size_t)p * H + ci]; },
        [&](int p) { return rb->data[p]; }));
  }
  return OVC_OK;
}

#include "ovc_tts_pack.inc"   // pack_tts(): V1 TTS front-half weights (text encoder, duration predictors, emb_g)

static int finalize(ovc_ctx* c) {
  const ovc_hparams& hp = c->hp;
  const int H = 192, S = hp.spec_channels, G = hp.gin_channels;
  drop_graphs(c);               // captured launches point at the old weight arenas
  c->h_w.clear();
  c->h_tcw.clear();

  // ---- posterior encoder (models.py:182-221)
  {
    const HostTensor *w, *b, *pw, *pb;
    TRY(tensor(c, "enc_q.pre.weight", {H, S, 1}, &w));
    TRY(tensor(c, "enc_q.pre.bias", {H}, &b));
    c->enc_pre = pack_conv(c, V_ENC_PRE, H, S, [&](int p, int ci, int) { return w->data[(size_t)p * S + ci]; },
                           [&](int p) { return b->data[p]; }, H, 1, H);
    c->enc_pre16 = c->enc_pre;            // same packing, 16-byte cp.async when the spectrogram pitch allows it
    c->enc_pre16.variant = V_FLOW_PRE;
    TRY(pack_wn(c, "enc_q.enc", 16, &c->enc_wn));
    TRY(tensor(c, "enc_q.proj.weight", {2 * H, H, 1}, &pw));
    TRY(tensor(c, "enc_q.proj.bias", {2 * H}, &pb));
    c->enc_proj = pack_conv(c, V_ENC_PROJ, 2 * H, H,
                            [&](int p, int ci, int) { return pw->data[(size_t)paired_row(p, H) * H + ci]; },
                            [&](int p) { return pb->data[paired_row(p, H)]; }, 2 * H, 1, 2 * H);
  }
  // ---- flow: 4 x (coupling, Flip) (models.py:385-388).  The Flips are absorbed: coupling f sees
  // the channel-reversed tensor iff f is odd, in both directions, so its `pre` reads the physical
  // upper half with reversed columns and its `post` writes the physical lower half with reversed rows.
  for (int f = 0; f < 4; ++f) {
    const std::string p = "flow.flows." + std::to_string(2 * f);
    const bool flipped = f & 1;
    const HostTensor *w, *b, *pw, *pb;
    TRY(tensor(c, p + ".pre.weight", {H, 96, 1}, &w));
    TRY(tensor(c, p + ".pre.bias", {H}, &b));
    c->flow_pre[f] = pack_conv(
        c, V_FLOW_PRE, H, 96,
        [&](int r, int ci, int) { return w->data[(size_t)r * 96 + (flipped ? 95 - ci : ci)]; },
        [&](int r) { return b->data[r]; }, H, 1, H);
    TRY(pack_wn(c, p + ".enc", 4, &c->flow_wn[f]));
    TRY(tensor(c, p + ".post.weight", {96, H, 1}, &pw));   // mean_only couplings only
    TRY(tensor(c, p + ".post.bias", {96}, &pb));
    c->flow_post[f] = pack_conv(
        c, V_FLOW_POST, 96, H,
        [&](int r, int ci, int) { return pw->data[(size_t)(flipped ? 95 - r : r) * H + ci]; },
        [&](int r) { return pb->data[flipped ? 95 - r : r]; }, 96, 1, 96);
  }
  // ---- generator (models.py:224-291)
  {
    const HostTensor* w;
    TRY(tensor(c, "dec.conv_pre.weight", {512, H, 7}, &w));
    // bias comes per batch item from the cond kernel (conv_pre.bias + cond(g))
    c->dec_pre = pack_conv(c, V_A_K7D1, 512, H, [&](int r, int ci, int k) { return w->data[((size_t)r * H + ci) * 7 + k]; },
                           [&](int) { return 0.f; }, 0, 7, 512);
    c->tc_pre = pack_tc(c, 512, H, 7, 1, [&](int r, int ci, int k) { return w->data[((size_t)r * H + ci) * 7 + k]; },
                        [&](int) { return 0.f; });
  }
  int ch = 512;
  for (int i = 0; i < 4; ++i) {
    const int s = hp.upsample_rates[i], kk = hp.upsample_kernel_sizes[i];
    const int cin = ch, cout = ch / 2;
    const std::string p = "dec.ups." + std::to_string(i);
    HostTensor w;   // [cin][cout][kk], weight-norm over dim 0 = cin (SURVEY appendix C.12)
    const HostTensor* b;
    TRY(conv_weight(c, p, {cin, cout, kk}, &w));
    TRY(tensor(c, p + ".bias", {cout}, &b));
    const int variant = s == 8 ? V_UPS8_A : (cout * s >= 128 ? V_UPS2_A : V_UPS2_B);
    auto raw = [&](int ci, int co, int k) { return w.data[((size_t)ci * cout + co) * kk + k]; };
    // polyphase (ovc_convpack.h): packed row = co*s + ph, tap 0/1/2 <-> x[n-1], x[n], x[n+1]
    c->dec_ups[i] = pack_conv(
        c, variant, cout * s, cin, [&](int row, int ci, int tap) { return conv_ups_weight(raw, s, kk, row, ci, tap); },
        [&](int co) { return b->data[co]; }, cout, 2, cout);
    c->dec_ups[i].out_mul = s;
    // tensor-core form: channels-last, row = ph * cout + co, so input step n yields the s output rows s*n .. s*n+s-1
    c->tc_ups[i] = pack_tc(
        c, s * cout, cin, 3, 1, [&](int row, int ci, int tap) { return tc_ups_weight(raw, s, kk, cout, row, ci, tap); },
        [&](int row) { return b->data[row % cout]; });
    ch = cout;
    for (int j = 0; j < 3; ++j) {
      const int K = hp.resblock_kernel_sizes[j];
      const int rbi = i * 3 + j;
      for (int d = 0; d < 3; ++d) {
        for (int which = 0; which < 2; ++which) {
          const std::string q = "dec.resblocks." + std::to_string(rbi) + (which ? ".convs2." : ".convs1.") + std::to_string(d);
          HostTensor rw;
          const HostTensor* rbias;
          TRY(conv_weight(c, q, {ch, ch, K}, &rw));
          TRY(tensor(c, q + ".bias", {ch}, &rbias));
          const int dil = which ? 1 : hp.resblock_dilations[j][d];
          ConvLayer L = pack_conv(c, dec_variant(ch, K, dil), ch, ch,
                                  [&](int r, int ci, int k) { return rw.data[((size_t)r * ch + ci) * K + k]; },
                                  [&](int r) { return rbias->data[r]; }, ch, K, ch);
          (which ? c->rb_c2 : c->rb_c1)[rbi][d] = L;
          (which ? c->tc_c2 : c->tc_c1)[rbi][d] =
              pack_tc(c, ch, ch, K, dil, [&](int r, int ci, int k) { return rw.data[((size_t)r * ch + ci) * K + k]; },
                      [&](int r) { return rbias->data[r]; });
        }
      }
    }
  }
  {
    const HostTensor* w;
    TRY(tensor(c, "dec.conv_post.weight", {1, 32, 7}, &w));
    c->post_w_off = append(c->h_w, w->data);
  }
  // ---- speaker conditioning mat-vec: stack cond_layer of enc_q, of the 4 couplings and dec.cond
  std::vector<int> wrow, sel;
  std::vector<float> cbias;
  {
    std::vector<float> cw;
    struct WnCond { int first_row; const HostTensor* b; std::vector<const HostTensor*> in_b; };
    WnCond wc[5];   // 0: enc_q, 1..4: the couplings
    for (int s = 0; s < 5; ++s) {
      const std::string p = s ? "flow.flows." + std::to_string(2 * s - 2) + ".enc" : std::string("enc_q.enc");
      const int n_layers = s ? 4 : 16;
      HostTensor w;
      TRY(conv_weight(c, p + ".cond_layer", {2 * H * n_layers, G, 1}, &w));
      TRY(tensor(c, p + ".cond_layer.bias", {2 * H * n_layers}, &wc[s].b));
      wc[s].in_b.resize(n_layers);
      for (int l = 0; l < n_layers; ++l) TRY(tensor(c, p + ".in_layers." + std::to_string(l) + ".bias", {2 * H}, &wc[s].in_b[l]));
      wc[s].first_row = (int)(cw.size() / G);
      cw.insert(cw.end(), w.data.begin(), w.data.end());
    }
    // sections enc_q, couplings on the source speaker, couplings on the target speaker; then the same three in the
    // tensor-core kernel's column order
    int (*const order[2])(int, int) = {paired_row, paired_row32};
    int* const off[2][3] = {{&c->cond_off_enc, &c->cond_off_fsrc, &c->cond_off_ftgt},
                            {&c->cond_off_enc_tc, &c->cond_off_fsrc_tc, &c->cond_off_ftgt_tc}};
    const int selv[3] = {hp.zero_g ? 0 : 1, 1, 2};
    for (int o = 0; o < 2; ++o)
      for (int sec = 0; sec < 3; ++sec) {
        *off[o][sec] = (int)wrow.size();
        for (int s = sec ? 1 : 0; s < (sec ? 5 : 1); ++s)
          for (int l = 0; l < (int)wc[s].in_b.size(); ++l)
            for (int p = 0; p < 2 * H; ++p) {
              const int r = order[o](p, H);
              wrow.push_back(wc[s].first_row + l * 2 * H + r);
              sel.push_back(selv[sec]);
              cbias.push_back(wc[s].b->data[l * 2 * H + r] + wc[s].in_b[l]->data[r]);
            }
      }
    const HostTensor *dw, *db, *cpb;
    TRY(tensor(c, "dec.cond.weight", {512, G, 1}, &dw));
    TRY(tensor(c, "dec.cond.bias", {512}, &db));
    TRY(tensor(c, "dec.conv_pre.bias", {512}, &cpb));
    c->cond_off_dec = (int)wrow.size();
    const int dec_first = (int)(cw.size() / G);
    cw.insert(cw.end(), dw->data.begin(), dw->data.end());
    for (int r = 0; r < 512; ++r) {
      wrow.push_back(dec_first + r);
      sel.push_back(hp.zero_g ? 0 : 2);
      cbias.push_back(db->data[r] + cpb->data[r]);
    }
    c->cond_rows_out = (int)wrow.size();
    c->cond_w_off = append(c->h_w, cw);
    c->cond_b_off = append(c->h_w, cbias);
  }
  if (G > COND_GIN_MAX) return fail(OVC_ERR_INVALID, "gin_channels %d exceeds the conditioning kernel's %d", G, COND_GIN_MAX);
  std::vector<int> pf_cols[2][3];
  {
    const int sec_off[2][4] = {{c->cond_off_enc, c->cond_off_fsrc, c->cond_off_ftgt, c->cond_off_dec},
                               {c->cond_off_enc_tc, c->cond_off_fsrc_tc, c->cond_off_ftgt_tc, c->cond_off_dec}};
    const int sec_len[4] = {c->cond_off_fsrc - c->cond_off_enc, c->cond_off_ftgt - c->cond_off_fsrc,
                            c->cond_off_enc_tc - c->cond_off_ftgt, 512};
    for (int o = 0; o < 2; ++o)
      for (int m = 1; m <= 3; ++m) {
        std::vector<int>& cols = pf_cols[o][m - 1];
        for (int sec = 0; sec < 4; ++sec) {
          const int sl = sel[sec_off[o][sec]];
          c->cond_pf_off[o][m - 1][sec] = -1;
          if (sl == 0 || !(m & sl)) continue;
          c->cond_pf_off[o][m - 1][sec] = (int)cols.size();
          for (int i = 0; i < sec_len[sec]; ++i) cols.push_back(sec_off[o][sec] + i);
        }
        c->cond_pf_cols[o][m - 1] = (int)cols.size();
      }
    // cond_kernel reads one side per CTA: every aligned block of COND_ROWS output columns must read the same side
    auto uniform = [&](const std::vector<int>& cols, int n) {
      auto col = [&](int i) { return cols.empty() ? i : cols[i]; };
      for (int i = 0; i < n; ++i)
        if (sel[col(i)] != sel[col(i / COND_ROWS * COND_ROWS)]) return false;
      return true;
    };
    bool ok = uniform({}, (int)sel.size());
    for (auto& oc : pf_cols)
      for (auto& cols : oc) ok = ok && uniform(cols, (int)cols.size());
    if (!ok) return fail(OVC_ERR_INVALID, "conditioning sections are not aligned to %d rows", COND_ROWS);
  }
  // ---- ReferenceEncoder (optional: only extract_se needs it; models.py:301-338)
  c->has_refenc = false;
  if (find(c, "ref_enc.proj.weight")) {
    static const int filt[7] = {1, 32, 32, 64, 64, 128, 128};
    for (int i = 0; i < 6; ++i) {
      const std::string q = "ref_enc.convs." + std::to_string(i);
      HostTensor w;
      const HostTensor* b;
      TRY(conv_weight(c, q, {filt[i + 1], filt[i], 3, 3}, &w));
      TRY(tensor(c, q + ".bias", {filt[i + 1]}, &b));
      c->re_conv_w[i] = append(c->h_w, w.data);
      c->re_conv_b[i] = append(c->h_w, b->data);
    }
    int w6 = S;   // width after the six stride-2 convs (models.py:330-337)
    for (int i = 0; i < 6; ++i) w6 = (w6 - 1) / 2 + 1;
    c->re_gru_in = 128 * w6;
    const struct { const char* key; std::vector<int64_t> shape; size_t* off; } re[8] = {
        {"ref_enc.gru.weight_ih_l0", {384, c->re_gru_in}, &c->re_wih}, {"ref_enc.gru.weight_hh_l0", {384, 128}, &c->re_whh},
        {"ref_enc.gru.bias_ih_l0", {384}, &c->re_bih},                 {"ref_enc.gru.bias_hh_l0", {384}, &c->re_bhh},
        {"ref_enc.proj.weight", {G, 128}, &c->re_pw},                  {"ref_enc.proj.bias", {G}, &c->re_pb},
        {"ref_enc.layernorm.weight", {S}, &c->re_lng},                 {"ref_enc.layernorm.bias", {S}, &c->re_lnb}};
    for (const auto& e : re) {
      const HostTensor* t;
      TRY(tensor(c, e.key, e.shape, &t));
      *e.off = append(c->h_w, t->data);
    }
    c->has_refenc = true;
  }
  // ---- V1 TTS front half (optional: base-speaker checkpoints only, models.py:451-465)
  c->tts = TtsLayers();
  if (find(c, "enc_p.emb.weight")) TRY(pack_tts(c));
  // ---- upload
  ON_DEVICE(c);
  if (c->d_w) { cudaFree(c->d_w); c->d_w = nullptr; }
  c->w_floats = c->h_w.size();
  CK(cudaMalloc(&c->d_w, c->w_floats * sizeof(float)));
  CK(cudaMemcpy(c->d_w, c->h_w.data(), c->w_floats * sizeof(float), cudaMemcpyHostToDevice));
  if (c->d_tcw) { cudaFree(c->d_tcw); c->d_tcw = nullptr; }
  CK(cudaMalloc(&c->d_tcw, c->h_tcw.size() * sizeof(float)));
  CK(cudaMemcpy(c->d_tcw, c->h_tcw.data(), c->h_tcw.size() * sizeof(float), cudaMemcpyHostToDevice));
  c->h_tcw.clear();
  c->h_tcw.shrink_to_fit();
  for (int TN : {128, 64, 32})
    for (bool staged : {false, true}) {
      const TcKernel k = tc_conv_kernel(TN, staged), p = tc_pair_kernel(TN, TcPairOcc(), staged);
      CK(cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k.smem));
      CK(cudaFuncSetAttribute(p.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem));
    }
  for (int i = 0; i < TCN_N_OCC2; ++i) {
    // a config runs two CTAs per SM only where the device confirms they fit: otherwise its pairs keep one CTA per SM
    // (and a grid of one CTA per SM), never a doubled grid on one
    const TcKernel k = tc_pair_kernel(kTcPairOcc2[i].C, kTcPairOcc2[i].o);
    CK(cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k.smem));
    int blocks = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, k.fn, k.threads, k.smem));
    c->pair_occ2_ok[i] = blocks >= 2;
    if (blocks < 2)
      fprintf(stderr, "ovc: the C = %d conv-pair kernel with %d operand buffer(s) fits %d CTA(s) per SM, not 2; its pairs run "
              "one CTA per SM\n", kTcPairOcc2[i].C, kTcPairOcc2[i].o.nabuf, blocks);
  }
  if (c->d_cond_wrow) cudaFree(c->d_cond_wrow);
  if (c->d_cond_sel) cudaFree(c->d_cond_sel);
  CK(cudaMalloc(&c->d_cond_wrow, wrow.size() * sizeof(int)));
  CK(cudaMalloc(&c->d_cond_sel, sel.size() * sizeof(int)));
  CK(cudaMemcpy(c->d_cond_wrow, wrow.data(), wrow.size() * sizeof(int), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(c->d_cond_sel, sel.data(), sel.size() * sizeof(int), cudaMemcpyHostToDevice));
  for (int o = 0; o < 2; ++o)
    for (int m = 0; m < 3; ++m) {
      if (c->d_cond_cols[o][m]) cudaFree(c->d_cond_cols[o][m]);
      c->d_cond_cols[o][m] = nullptr;
      if (pf_cols[o][m].empty()) continue;
      CK(cudaMalloc(&c->d_cond_cols[o][m], pf_cols[o][m].size() * sizeof(int)));
      CK(cudaMemcpy(c->d_cond_cols[o][m], pf_cols[o][m].data(), pf_cols[o][m].size() * sizeof(int), cudaMemcpyHostToDevice));
    }
  if (!c->d_tw) {
    std::vector<float2> tw(STFT_N);
    std::vector<float> win(STFT_N);
    const double PI = 3.14159265358979323846;
    for (int m = 0; m < STFT_N; ++m) {
      tw[m] = make_float2((float)std::cos(2.0 * PI * m / STFT_N), (float)(-std::sin(2.0 * PI * m / STFT_N)));
      win[m] = (float)(0.5 - 0.5 * std::cos(2.0 * PI * m / STFT_N));   // torch.hann_window(periodic=True)
    }
    CK(cudaMalloc(&c->d_tw, STFT_N * sizeof(float2)));
    CK(cudaMalloc(&c->d_win, STFT_N * sizeof(float)));
    CK(cudaMemcpy(c->d_tw, tw.data(), STFT_N * sizeof(float2), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(c->d_win, win.data(), STFT_N * sizeof(float), cudaMemcpyHostToDevice));
  }
  c->h_w.clear();
  c->h_w.shrink_to_fit();
  c->sd.clear();
  for (int v = 0; v < V_COUNT; ++v) CK(kPrepare[v]());
  c->finalized = true;
  return OVC_OK;
}

// ---------------------------------------------------------------------------------------------
// workspace layout
// ---------------------------------------------------------------------------------------------
struct WsLayout {
  int P;   // frame pitch (multiple of 4)
  size_t cond, cond_pf, g_pf, x, skip, acts, z, dpre, bufA, bufB, bufC, bufD, bufE, bufF, spec, frames, win_g, win_len, total;
  size_t brB[2], brC[2];   // per-branch ResBlock buffers of the concurrent-branch mode (small calls only)
  bool branches;
};
// pf_cols: columns of the per-frame conditioning vector (0: every embedding is per item, no per-frame buffer);
// g_frames: also a [B][gin][Tmax] per-frame speaker embedding (the TTS decode after a per-token encode)
static WsLayout ws_layout(const ovc_ctx* c, int B, int Tmax, int pf_cols = 0, bool g_frames = false) {
  WsLayout L;
  L.P = (int)round_up((size_t)Tmax, 4);
  size_t o = 0;
  auto take = [&](size_t n) { size_t r = o; o = round_up(o + n, 64); return r; };
  L.cond = take((size_t)B * c->cond_rows_out);
  L.cond_pf = pf_cols ? take((size_t)B * Tmax * pf_cols) : 0;
  L.g_pf = g_frames ? take((size_t)B * c->hp.gin_channels * Tmax) : 0;
  L.x = take((size_t)B * 192 * L.P);
  L.skip = take((size_t)B * 192 * L.P);
  L.acts = take((size_t)B * 192 * L.P);
  L.z = take((size_t)B * 192 * L.P);
  L.dpre = take((size_t)B * 512 * L.P);
  const size_t big = (size_t)B * 8192 * L.P;
  L.bufA = take(big);
  L.bufB = take(big);
  L.bufC = take(big);
  L.bufD = take(big);
  L.bufE = c->precision ? take((size_t)B * 512 * L.P) : 0;     // conv_pre output, channels-last
  L.bufF = (c->precision && c->debug) ? take(big) : 0;        // [C][T] scratch of the debug taps only
  L.branches = c->precision && c->use_branches && (long long)B * Tmax <= c->par_frames;
  for (int j = 0; j < 2; ++j) {
    L.brB[j] = L.branches ? take(big) : 0;
    L.brC[j] = L.branches ? take(big) : 0;
  }
  L.spec = take((size_t)B * c->hp.spec_channels * L.P);
  L.frames = take((size_t)2 * B + 4);   // B int64
  L.win_g = take((size_t)B * c->hp.gin_channels);   // ovc_tts_decode_windows: g of each window's row
  L.win_len = take((size_t)2 * B + 4);              // and its decode length, B int64
  L.total = o;
  return L;
}

struct Run {
  ovc_ctx* c;
  cudaStream_t st;
  int B, Tmax, P;
  const long long* lens;
  const long long* glens;   // generator lengths: lens when ragged, NULL (= Tmax) otherwise
  double sum_len;           // sum over batch of generator frames (for FLOP/byte accounting): B*Tmax upper bound
};

static int launch(Run& r, const ConvLayer& L, ConvArgs a, int t_len, bool mrf = false, double flops = 0,
                  double bytes = 0) {
  a.w = r.c->d_w + L.w_off;
  a.n_chunks = L.n_chunks;
  a.cin = L.cin;
  a.tmax = r.Tmax;
  if (a.scale == 0.f) a.scale = 1.f;
  ovc_ctx* c = r.c;
  const bool prof = c->prof;
  if (prof) {
    if (c->ev_used + 2 > c->ev.size()) {
      const size_t old = c->ev.size();
      c->ev.resize(old + 512);
      for (size_t i = old; i < c->ev.size(); ++i) CK(cudaEventCreate(&c->ev[i]));
    }
    CK(cudaEventRecord(c->ev[c->ev_used], r.st));
  }
  CK(kLaunch[L.variant](a, t_len, L.row_tiles, r.B, r.st));
  c->launches++;
  if (prof) {
    CK(cudaEventRecord(c->ev[c->ev_used + 1], r.st));
    c->ev_used += 2;
    // algorithmic work of this launch over all B * t_len positions (upper bound for ragged batches)
    const double units = (double)r.B * t_len;
    c->ev_flops.push_back(2.0 * L.cout * L.cin * L.K * units * L.out_mul);
    c->ev_bytes.push_back(4.0 * units * ((double)L.cin + (double)L.cout * L.out_mul));
    c->ev_variant.push_back(L.variant);
    c->ev_family.push_back(mrf ? 1 : 0);
    c->ev_tag.push_back(0);
  }
  (void)flops; (void)bytes;
  return OVC_OK;
}

static int tap(Run& r, const char* name, const float* src, int C, int T, int pitch) {
  ovc_ctx* c = r.c;
  if (!c->debug) return OVC_OK;
  DebugBuf& d = c->taps[name];
  const size_t n = (size_t)r.B * C * pitch;
  if (d.floats < n) {
    if (d.d) cudaFree(d.d);
    CK(cudaMalloc(&d.d, n * sizeof(float)));
    d.floats = n;
  }
  d.shape[0] = r.B; d.shape[1] = C; d.shape[2] = T; d.shape[3] = pitch;
  CK(cudaMemcpyAsync(d.d, src, n * sizeof(float), cudaMemcpyDeviceToDevice, r.st));
  return OVC_OK;
}


// profiling bracket shared by the non-conv1d_f32 launches
static int prof_begin(Run& r) {
  ovc_ctx* c = r.c;
  if (!c->prof) return OVC_OK;
  if (c->ev_used + 2 > c->ev.size()) {
    const size_t old = c->ev.size();
    c->ev.resize(old + 512);
    for (size_t i = old; i < c->ev.size(); ++i) CK(cudaEventCreate(&c->ev[i]));
  }
  CK(cudaEventRecord(c->ev[c->ev_used], r.st));
  return OVC_OK;
}
static int prof_end(Run& r, int variant, int family, double flops, double bytes, int tag = 0) {
  ovc_ctx* c = r.c;
  if (!c->prof) return OVC_OK;
  CK(cudaEventRecord(c->ev[c->ev_used + 1], r.st));
  c->ev_used += 2;
  c->ev_flops.push_back(flops);
  c->ev_bytes.push_back(bytes);
  c->ev_variant.push_back(variant);
  c->ev_family.push_back(family);
  c->ev_tag.push_back(tag);
  return OVC_OK;
}
enum { V_TCPAIR128 = -14, V_TCPAIR64 = -12, V_TCPAIR32 = -13, V_TC128 = -1, V_TC64 = -2, V_TC32 = -3, V_TRANSPOSE = -4, V_TTS_DENSE = -5, V_TTS_LN = -6, V_TTS_SCORES = -7,
       V_TTS_ATTN = -8, V_TTS_DW = -9, V_TTS_SPLINE = -10, V_TTS_MISC = -11 };
static const char* variant_name(int v) {
  if (v >= 0) return kInfo[v].name;
  switch (v) {
    case V_TCPAIR128: return "PAIR_N128";
    case V_TCPAIR64: return "PAIR_N64";
    case V_TCPAIR32: return "PAIR_N32";
    case V_TC128: return "TC3_N128";
    case V_TC64: return "TC3_N64";
    case V_TC32: return "TC3_N32";
    case V_TTS_DENSE: return "TTS_DENSE32";
    case V_TTS_LN: return "TTS_LAYERNORM";
    case V_TTS_SCORES: return "TTS_SCORES";
    case V_TTS_ATTN: return "TTS_ATTN_OUT";
    case V_TTS_DW: return "TTS_DWCONV";
    case V_TTS_SPLINE: return "TTS_SPLINE";
    case V_TTS_MISC: return "TTS_MISC";
    default: return "TRANSPOSE";
  }
}

// one conv on the tensor cores (3xFP16 split precision / single-pass fp16), channels-last in/out.  t_len / mul are in INPUT steps.
struct TcExtra {
  int epi = 0;                    // 0 linear, 1 WN gate, 2 WN res/skip
  const float* bias = nullptr;    // override (per-utterance conditioning vector), with stride
  long long bias_bs = 0, bias_ts = 0;
  float* s = nullptr;             // skip accumulator (EPI 2)
  int split = 0, first = 0;
  int y_ld = 0;                   // output row width when it differs from Ntot
  bool use_lens_frames = false;   // limits are the frame lengths (enc/flow) instead of the generator lengths
  const long long* lens_x = nullptr; bool has_lens_x = false;   // the input's own limit (TcConvArgs.lens_x)
  int grid_div = 1;               // persistent kernel: use 1 / grid_div of the SMs (concurrent ResBlock branches)
};
// kernel launch with (optionally) the programmatic-stream-serialization attribute: the kernel may begin while its
// predecessor in the stream drains; it calls griddepcontrol.wait before it touches dependent data (ovc_tcconv.cuh)
template <class... KArgs, class... Args>
static cudaError_t launch_ex(void (*kernel)(KArgs...), dim3 grid, int block, size_t smem, cudaStream_t st, bool pdl, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = dim3((unsigned)block, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

static int launch_tc(Run& r, const TcLayer& T, const float* x, float* y, const float* res, int t_len, int mul, float slope,
                     float scale, int accumulate, int family, const TcExtra& ex = TcExtra()) {
  TcConvArgs a{};
  const int y_ld = ex.y_ld ? ex.y_ld : T.Ntot;
  a.x = x; a.x_bs = (long long)T.Cin * r.P * mul;
  a.w = reinterpret_cast<const uint16_t*>(r.c->d_tcw + T.w_off);
  a.bias = ex.bias ? ex.bias : r.c->d_tcw + T.b_off; a.bias_bs = ex.bias_bs; a.bias_ts = ex.bias_ts;
  a.y = y; a.y_bs = (long long)y_ld * r.P * mul; a.y_ld = y_ld;
  a.r = res;
  a.s = ex.s; a.s_bs = a.y_bs;
  a.epi = ex.epi; a.split = ex.split; a.first = ex.first;
  a.lens = ex.use_lens_frames ? r.lens : r.glens; a.tmax = r.Tmax; a.mul = mul;
  a.lens_x = ex.lens_x; a.has_lens_x = ex.has_lens_x ? 1 : 0;
  a.Cin = T.Cin; a.Ntot = T.Ntot; a.K = T.K; a.DIL = T.DIL;
  a.slope = slope; a.scale = scale; a.accumulate = accumulate;
  a.passes = r.c->precision == 2 ? 1 : 3;
  if (T.TN == 0) return fail(OVC_ERR_INVALID, "conv %d -> %d (k %d, dilation %d) does not fit the tensor-core kernels", T.Cin, T.Ntot, T.K, T.DIL);
  if (!(slope >= 0.f && slope <= 1.f)) return fail(OVC_ERR_INVALID, "leaky_relu slope %g outside [0, 1]", (double)slope);
  TRY(prof_begin(r));
  // persistent: one CTA per SM walks the (utterance, 128-step tile) list; column tiles (if any) on grid.y
  const TcGrid g = tc_grid(t_len, r.B, T.Ntot, T.TN, r.c->sm_count, ex.grid_div);
  const int n_tt = g.n_tt, total = g.total;
  dim3 pg((unsigned)g.grid_x, g.ncol, 1);
  const bool pdl = r.c->use_pdl == 1 || (r.c->use_pdl == 2 && ex.epi != 0);
  const TcKernel k = tc_conv_kernel(T.TN, r.c->use_staged_epi && tc_stage_pays(T.K, a.passes));
  CK(launch_ex(k.fn, pg, k.threads, k.smem, r.st, pdl, a, n_tt, total));
  CK(cudaGetLastError());
  r.c->launches++;
  const double units = (double)r.B * t_len;
  const int eff_k = family == 2 ? 2 : T.K;   // polyphase transposed conv: 2 of the 3 packed taps are non-zero per row
  TRY(prof_end(r, T.TN == 128 ? V_TC128 : T.TN == 64 ? V_TC64 : V_TC32, family == 1 ? 1 : 0, 2.0 * T.Cin * T.Ntot * eff_k * units,
               4.0 * (T.Cin + T.Ntot * (1 + (res ? 1 : 0) + (accumulate ? 1 : 0))) * units, (T.Cin << 16) | (T.K << 8) | T.DIL));
  return OVC_OK;
}

// one ResBlock conv pair (c1 dilated, c2 dilation 1, residual = the pair's input) as ONE kernel: C = 128 / 64 / 32
// stages, where tc_pair_fuses (ovc_tcpack.h) accepts the pair
static int launch_pair(Run& r, const TcLayer& T1, const TcLayer& T2, const float* x, float* y, int t_len, int mul, float slope,
                       float scale, int accumulate) {
  TcConvArgs a{};
  const int C = T1.TN;
  a.x = x; a.x_bs = (long long)C * r.P * mul;
  a.w = reinterpret_cast<const uint16_t*>(r.c->d_tcw + T1.w_off);
  a.w2 = reinterpret_cast<const uint16_t*>(r.c->d_tcw + T2.w_off);
  a.bias = r.c->d_tcw + T1.b_off; a.bias2 = r.c->d_tcw + T2.b_off;
  a.y = y; a.y_bs = a.x_bs; a.y_ld = C;
  a.lens = r.glens; a.tmax = r.Tmax; a.mul = mul;
  a.Cin = C; a.Ntot = C; a.K = T1.K; a.DIL = T1.DIL;
  a.slope = slope; a.scale = scale; a.accumulate = accumulate;
  a.passes = r.c->precision == 2 ? 1 : 3;
  TcPairOcc o = r.c->use_pair_occ ? tc_pair_occ(T1, T2) : TcPairOcc();
  for (int i = 0; i < TCN_N_OCC2; ++i)
    if (o.occ == 2 && kTcPairOcc2[i].C == C && kTcPairOcc2[i].o.nabuf == o.nabuf && !r.c->pair_occ2_ok[i]) o = TcPairOcc();
  const TcKernel k = tc_pair_kernel(C, o, r.c->use_staged_epi && tc_stage_pays(T1.K, a.passes));
  if (!k.fn) return fail(OVC_ERR_INVALID, "no conv-pair kernel for C = %d at %d CTA(s) per SM, %d operand buffer(s)", C, o.occ, o.nabuf);
  const TcGrid g = tc_pair_grid(t_len, r.B, T1.K, r.c->sm_count, o.occ);
  const int n_tt = g.n_tt, total = g.total;
  TRY(prof_begin(r));
  dim3 pg((unsigned)g.grid_x, 1, 1);
  CK(launch_ex(k.fn, pg, k.threads, k.smem, r.st, false, a, n_tt, total));
  CK(cudaGetLastError());
  r.c->launches++;
  const double units = (double)r.B * t_len;
  TRY(prof_end(r, C == 128 ? V_TCPAIR128 : C == 64 ? V_TCPAIR64 : V_TCPAIR32, 1, 2.0 * 2.0 * C * C * T1.K * units, 4.0 * C * (2 + (accumulate ? 1 : 0)) * units,
               (C << 16) | (T1.K << 8) | T1.DIL));
  return OVC_OK;
}

static int launch_transpose(Run& r, const float* src, float* dst, int rows, int cols) {
  dim3 grid((cols + 31) / 32, (rows + 31) / 32, r.B);
  TRY(prof_begin(r));
  transpose_kernel<<<grid, 256, 0, r.st>>>(src, dst, rows, cols, (long long)rows * cols);
  CK(cudaGetLastError());
  r.c->launches++;
  TRY(prof_end(r, V_TRANSPOSE, 0, 0.0, 8.0 * rows * cols * r.B));
  return OVC_OK;
}

// where a conditioned layer reads its vector: item b, frame t, column n at p + b * bs + min(t, Tmax - 1) * ts + n
struct CondRef {
  const float* p; long long bs, ts;
  CondRef at(int col) const { return {p + col, bs, ts}; }
};

// one WN stack (modules.py:185-210): x <- in place, skip <- output
static int run_wn(Run& r, const WNLayers& wn, float* x, float* skip, float* acts, const CondRef& cond) {
  const int P = r.P, T = r.Tmax;
  const long long bs = 192LL * P;
  const int n = (int)wn.in.size();
  for (int i = 0; i < n; ++i) {
    ConvArgs a{};
    a.x = x; a.x_bs = bs; a.x_pitch = P;
    a.bias = cond.p + (size_t)i * 384; a.bias_bs = cond.bs; a.bias_ts = cond.ts;
    a.y = acts; a.y_bs = bs; a.y_pitch = P;
    a.lens_in = r.lens; a.lens_out = r.lens; a.mul_in = 1; a.mul_out = 1;
    a.slope = 1.f;
    TRY(launch(r, wn.in[i], a, T));
    ConvArgs b{};
    b.x = acts; b.x_bs = bs; b.x_pitch = P;
    b.bias = r.c->d_w + wn.rs[i].b_off; b.bias_bs = 0;
    b.y = x; b.y_bs = bs; b.y_pitch = P;
    b.s = skip; b.s_bs = bs; b.s_pitch = P;
    b.lens_in = r.lens; b.lens_out = r.lens; b.mul_in = 1; b.mul_out = 1;
    b.slope = 1.f;
    b.split = (i < n - 1) ? 192 : 0;
    b.flags = (i == 0) ? F_FIRST : 0;
    TRY(launch(r, wn.rs[i], b, T));
  }
  return OVC_OK;
}

// the same stack on the tensor cores: x, acts, skip live channels-last inside the stack; h comes in and the
// output leaves in the [C][T] layout of the small FFMA kernels around it (pre / proj / post)
static int run_wn_tc(Run& r, const WNLayers& wn, float* x, float* skip, float* acts, float* x_cl, float* skip_cl,
                     const CondRef& cond_tc) {
  const int P = r.P, T = r.Tmax;
  const int n = (int)wn.tc_in.size();
  TRY(launch_transpose(r, x, x_cl, 192, P));
  for (int i = 0; i < n; ++i) {
    TcExtra g;
    g.epi = 1; g.bias = cond_tc.p + (size_t)i * 384; g.bias_bs = cond_tc.bs; g.bias_ts = cond_tc.ts; g.y_ld = 192;
    g.use_lens_frames = true;
    TRY(launch_tc(r, wn.tc_in[i], x_cl, acts, nullptr, T, 1, 1.f, 1.f, 0, 0, g));
    TcExtra q;
    q.epi = 2; q.s = skip_cl; q.split = (i < n - 1) ? 192 : 0; q.first = (i == 0); q.y_ld = 192; q.use_lens_frames = true;
    TRY(launch_tc(r, wn.tc_rs[i], acts, x_cl, nullptr, T, 1, 1.f, 1.f, 0, 0, q));
  }
  TRY(launch_transpose(r, skip_cl, skip, P, 192));
  return OVC_OK;
}

// cond: the conditioning of this direction's couplings (flow src forward, flow tgt in reverse), in the column order of
// the precision mode
static int run_flow(Run& r, const WsLayout& W, float* ws, bool reverse, const CondRef& cond) {
  ovc_ctx* c = r.c;
  const int P = r.P, T = r.Tmax;
  const long long bs = 192LL * P;
  float* z = ws + W.z;
  float* x = ws + W.x;
  float* skip = ws + W.skip;
  float* acts = ws + W.acts;
  for (int step = 0; step < 4; ++step) {
    const int f = reverse ? 3 - step : step;
    const bool flipped = f & 1;
    // pre: x0 (physical lower half, or upper half when flipped) -> h     (modules.py:438-439)
    ConvArgs a{};
    a.x = z + (flipped ? 96 * (size_t)P : 0); a.x_bs = bs; a.x_pitch = P;
    a.bias = c->d_w + c->flow_pre[f].b_off; a.bias_bs = 0;
    a.y = x; a.y_bs = bs; a.y_pitch = P;
    a.lens_in = r.lens; a.lens_out = r.lens; a.mul_in = 1; a.mul_out = 1;
    a.slope = 1.f; a.scale = 1.f;
    TRY(launch(r, c->flow_pre[f], a, T));
    if (c->precision >= 1) {
      TRY(run_wn_tc(r, c->flow_wn[f], x, skip, acts, ws + W.bufA, ws + W.bufB, cond.at(f * 4 * 384)));
    } else {
      TRY(run_wn(r, c->flow_wn[f], x, skip, acts, cond.at(f * 4 * 384)));
    }
    // post + coupling update of x1 in place                                (modules.py:441-454)
    ConvArgs b{};
    b.x = skip; b.x_bs = bs; b.x_pitch = P;
    b.bias = c->d_w + c->flow_post[f].b_off; b.bias_bs = 0;
    b.y = z + (flipped ? 0 : 96 * (size_t)P); b.y_bs = bs; b.y_pitch = P;
    b.lens_in = r.lens; b.lens_out = r.lens; b.mul_in = 1; b.mul_out = 1;
    b.slope = 1.f;
    b.sign = reverse ? -1.f : 1.f;
    TRY(launch(r, c->flow_post[f], b, T));
  }
  return OVC_OK;
}

static void drop_graphs(ovc_ctx* c) {
  for (auto& g : c->graphs)
    if (g.exec) cudaGraphExecDestroy(g.exec);
  c->graphs.clear();
}

__global__ void set_call_params_kernel(CallParams* p, unsigned long long seed, float tau, ItemParams items) {
  p->seed = seed;
  p->tau = tau;
  p->items = items;
}

static_assert(sizeof(ItemParams) == sizeof(ovc_item_params), "ItemParams mirrors ovc_item_params");
static ItemParams item_params(const ovc_item_params* p) {   // NULL -> every field NULL
  ItemParams r{};
  if (p) memcpy(&r, p, sizeof r);
  return r;
}
static void append_item_key(std::vector<uintptr_t>& key, const ItemParams& it) {
  for (const void* q : {(const void*)it.seed, (const void*)it.stream, (const void*)it.frame0, (const void*)it.tau,
                        (const void*)it.noise_scale, (const void*)it.noise_scale_w, (const void*)it.length_scale,
                        (const void*)it.sdp_ratio})
    key.push_back((uintptr_t)q);
}

// Run `body(stream)` -- a pure launch sequence -- directly, or replay it from a CUDA graph when the same signature `key`
// has been seen before (captured on the second sighting: a one-off call never pays for an instantiation).  Capture
// happens on an internal stream (the caller's may be the legacy default stream, which cannot be captured); the graph is
// launched into the caller's stream.
template <class Body>
static int run_graphed(ovc_ctx* c, const std::vector<uintptr_t>& key, cudaStream_t st, Body body) {
  if (!c->use_graph || c->prof || c->debug) return body(st);
  ovc_ctx::GraphEntry* e = nullptr;
  for (auto& g : c->graphs)
    if (g.key == key) { e = &g; break; }
  if (!e) {
    if (c->graphs.size() >= 16) {   // evict the least recently used signature
      size_t lru = 0;
      for (size_t i = 1; i < c->graphs.size(); ++i)
        if (c->graphs[i].stamp < c->graphs[lru].stamp) lru = i;
      if (c->graphs[lru].exec) cudaGraphExecDestroy(c->graphs[lru].exec);
      c->graphs.erase(c->graphs.begin() + lru);
    }
    c->graphs.emplace_back();
    e = &c->graphs.back();
    e->key = key;
  }
  e->stamp = ++c->graph_clock;
  e->seen++;
  if (e->exec) {
    CK(cudaGraphLaunch(e->exec, st));
    c->launches = e->launches;
    c->graph_replays++;
    return OVC_OK;
  }
  if (e->seen < 2) return body(st);
  if (!c->cap_stream) CK(cudaStreamCreateWithFlags(&c->cap_stream, cudaStreamNonBlocking));
  CK(cudaStreamBeginCapture(c->cap_stream, cudaStreamCaptureModeThreadLocal));
  const int rc = body(c->cap_stream);
  cudaGraph_t graph = nullptr;
  const cudaError_t ce = cudaStreamEndCapture(c->cap_stream, &graph);
  if (rc != OVC_OK || ce != cudaSuccess || !graph) {
    if (graph) cudaGraphDestroy(graph);
    cudaGetLastError();
    e->seen = -1000000;           // never try this signature again
    if (rc != OVC_OK) return rc;
    return body(st);
  }
  const cudaError_t ie = cudaGraphInstantiate(&e->exec, graph, 0);
  cudaGraphDestroy(graph);
  if (ie != cudaSuccess) {
    cudaGetLastError();
    e->exec = nullptr;
    e->seen = -1000000;
    return body(st);
  }
  e->launches = c->launches;
  CK(cudaGraphLaunch(e->exec, st));
  c->graph_replays++;
  return OVC_OK;
}

static int set_call_params(ovc_ctx* c, uint64_t seed, float tau, const ItemParams& items, cudaStream_t st) {
  if (!c->d_callp) CK(cudaMalloc(&c->d_callp, sizeof(CallParams)));
  set_call_params_kernel<<<1, 1, 0, st>>>(c->d_callp, seed, tau, items);
  CK(cudaGetLastError());
  return OVC_OK;
}
static uintptr_t option_bits(const ovc_ctx* c) {
  return (uintptr_t)c->precision | ((uintptr_t)c->use_pdl << 15) | ((uintptr_t)c->use_branches << 14) | ((uintptr_t)c->use_pair << 17) |
         ((uintptr_t)c->use_pair_occ << 18) | ((uintptr_t)c->use_staged_epi << 19);
}

static int ensure_ws(ovc_ctx* c, const WsLayout& W, int B, int Tmax, cudaStream_t st) {
  if (W.total <= c->ws_floats) return OVC_OK;
  CK(cudaStreamSynchronize(st));
  drop_graphs(c);               // captured launches point into the old workspace
  if (c->d_ws) CK(cudaFree(c->d_ws));
  c->d_ws = nullptr;
  c->ws_floats = 0;
  cudaError_t e = cudaMalloc(&c->d_ws, W.total * sizeof(float));
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail(OVC_ERR_NOMEM, "workspace of %.2f GB for B=%d Tmax=%d does not fit: %s", W.total * 4e-9, B, Tmax,
                cudaGetErrorString(e));
  }
  c->ws_floats = W.total;
  return OVC_OK;
}

// one side of a cond_kernel launch: [B][gin] per item, or [B][gin][Tmax] per frame
struct CondSide { const float* g; long long bs, cs, fs; };
static CondSide cond_side(const ovc_ctx* c, const float* g, bool per_frame, int Tmax) {
  const long long G = c->hp.gin_channels;
  return per_frame ? CondSide{g, G * Tmax, Tmax, 1} : CondSide{g, G, 1, 0};
}

// every speaker-conditioning 1x1 conv in one launch: the stacked list (cols NULL, n_out = cond_rows_out) or the
// per-frame columns `cols`, for `frames` frames of each of B items
static int launch_cond(ovc_ctx* c, cudaStream_t st, int B, int frames, const int* cols, int n_out, const CondSide& src,
                       const CondSide& tgt, float* out, long long out_bs, long long out_fs) {
  CondArgs a;
  a.w = c->d_w + c->cond_w_off; a.bias = c->d_w + c->cond_b_off;
  a.w_row = c->d_cond_wrow; a.sel = c->d_cond_sel; a.cols = cols;
  a.g_src = src.g; a.src_bs = src.bs; a.src_cs = src.cs; a.src_fs = src.fs;
  a.g_tgt = tgt.g; a.tgt_bs = tgt.bs; a.tgt_cs = tgt.cs; a.tgt_fs = tgt.fs;
  a.out = out; a.out_bs = out_bs; a.out_fs = out_fs;
  a.n_out = n_out; a.gin = c->hp.gin_channels; a.frames = frames;
  dim3 grid((n_out + COND_ROWS - 1) / COND_ROWS, B, (frames + COND_FCHUNK - 1) / COND_FCHUNK);
  cond_kernel<<<grid, 256, 0, st>>>(a);
  CK(cudaGetLastError());
  c->launches++;
  return OVC_OK;
}

// z (workspace, [B][192][P]) -> a caller tensor [B][192][Tmax], zero past each length
static int copy_latent_out(Run& r, const WsLayout& W, float* ws, float* dst) {
  if (!dst) return OVC_OK;
  dim3 grid((r.Tmax + 255) / 256, 192, r.B);
  copy_latent_kernel<<<grid, 256, 0, r.st>>>(ws + W.z, W.P, dst, r.Tmax, 192, r.lens);
  CK(cudaGetLastError());
  r.c->launches++;
  return OVC_OK;
}

// HiFi-GAN generator on the latent in ws.z (models.py:272-291): shared by voice_conversion and the TTS decode
static int run_dec(Run& r, const WsLayout& W, float* ws, const CondRef& cond, const long long* lens, float* o_hat) {
  ovc_ctx* c = r.c;
  cudaStream_t st = r.st;
  const int B = r.B, Tmax = r.Tmax, P = W.P;
  const long long bs192 = 192LL * P;
  // ---- generator (models.py:272-291).  Lengths: frames * cumulative upsampling.
  const bool pre_tc = c->precision >= 1 && c->tc_pre.TN != 0;
  if (!pre_tc) {
    ConvArgs a{};
    a.x = ws + W.z; a.x_bs = bs192; a.x_pitch = P;
    a.bias = cond.p; a.bias_bs = cond.bs; a.bias_ts = cond.ts;
    a.y = ws + W.dpre; a.y_bs = 512LL * P; a.y_pitch = P;
    a.lens_in = lens;          // z_hat * y_mask
    a.lens_out = r.glens; a.mul_in = 1; a.mul_out = 1;
    a.slope = 1.f; a.scale = 1.f;
    TRY(launch(r, c->dec_pre, a, Tmax));
    TRY(tap(r, "dec.pre", ws + W.dpre, 512, Tmax, P));
  }
  float* bufA = ws + W.bufA; float* bufB = ws + W.bufB; float* bufC = ws + W.bufC; float* bufD = ws + W.bufD;
  if (c->precision >= 1) {
    // ---- tensor-core generator: channels-last [t][C] from conv_pre's output to conv_post's input.
    // ConvTranspose1d = polyphase conv Cin -> s*Cout whose row n IS output rows s*n .. s*n+s-1 of the
    // channels-last result; ResBlock convs = tcconv with fused lrelu / bias / residual / MRF average.
    float* bufE = ws + W.bufE;
    float* bufF = ws + W.bufF;   // [C][T] scratch for debug taps
    auto tap_cl = [&](const char* nm, const float* cl, int C, int T_, int pitch) -> int {
      if (!c->debug) return OVC_OK;
      TRY(launch_transpose(r, cl, bufF, pitch, C));
      return tap(r, nm, bufF, C, T_, pitch);
    };
    if (pre_tc) {
      // conv_pre (192 -> 512, k 7) + cond(g) on the tensor cores too: z channels-last through bufA, result straight into
      // bufE; the input is cut at the frame lengths (z_hat * y_mask), the output runs over the generator's own limit
      TRY(launch_transpose(r, ws + W.z, bufA, 192, P));
      TcExtra e;
      e.bias = cond.p; e.bias_bs = cond.bs; e.bias_ts = cond.ts;
      e.lens_x = lens; e.has_lens_x = lens != nullptr;
      TRY(launch_tc(r, c->tc_pre, bufA, bufE, nullptr, Tmax, 1, 1.f, 1.f, 0, 0, e));
      TRY(tap_cl("dec.pre", bufE, 512, Tmax, P));
    } else {
      TRY(launch_transpose(r, ws + W.dpre, bufE, 512, P));
    }
    const float* stage_in = bufE;
    int cin = 512, up = 1;
    const bool par = W.branches && !c->prof && !c->debug;
    if (par && !c->br_stream[0]) {
      for (int j = 0; j < 2; ++j) CK(cudaStreamCreateWithFlags(&c->br_stream[j], cudaStreamNonBlocking));
      for (int j = 0; j < 4; ++j) CK(cudaEventCreateWithFlags(&c->br_ev[j], cudaEventDisableTiming));
    }
    for (int i = 0; i < 4; ++i) {
      const int s = c->hp.upsample_rates[i];
      const int cout = cin / 2, up_out = up * s;
      const int Tlen = Tmax * up_out, pitch_out = P * up_out;
      char nm[32];
      TRY(launch_tc(r, c->tc_ups[i], stage_in, bufA, nullptr, Tmax * up, up, 0.1f, 1.f, 0, 2));
      snprintf(nm, sizeof nm, "dec.ups%d", i);
      TRY(tap_cl(nm, bufA, cout, Tlen, pitch_out));
      if (!par) {
        for (int j = 0; j < 3; ++j) {
          bool fused = c->use_pair;
          for (int d = 0; d < 3; ++d) fused = fused && tc_pair_fuses(c->tc_c1[i * 3 + j][d], c->tc_c2[i * 3 + j][d]);
          if (fused) {
            // one kernel per conv pair; a pair never runs in place (its tiles read x with a halo), so the running
            // activation ping-pongs bufA -> bufB -> bufC -> bufD (bufC is free: the intermediate stays on chip)
            const float* xs[3] = {bufA, bufB, bufC};
            float* ys[3] = {bufB, bufC, bufD};
            for (int d = 0; d < 3; ++d)
              TRY(launch_pair(r, c->tc_c1[i * 3 + j][d], c->tc_c2[i * 3 + j][d], xs[d], ys[d], Tlen, up_out, 0.1f,
                              (d == 2 && j == 2) ? 1.0f / 3.0f : 1.f, (d == 2 && j > 0) ? 1 : 0));
            continue;
          }
          for (int d = 0; d < 3; ++d) {
            const float* xin = d == 0 ? bufA : bufB;
            float* yout = d < 2 ? bufB : bufD;
            TRY(launch_tc(r, c->tc_c1[i * 3 + j][d], xin, bufC, nullptr, Tlen, up_out, 0.1f, 1.f, 0, 1));
            TRY(launch_tc(r, c->tc_c2[i * 3 + j][d], bufC, yout, xin, Tlen, up_out, 0.1f,
                          (d == 2 && j == 2) ? 1.0f / 3.0f : 1.f, (d == 2 && j > 0) ? 1 : 0, 1));
          }
        }
      } else {
        // a latency-bound call: the three ResBlock branches (models.py:280-285) are independent up to their last conv,
        // so they run side by side -- branch 0 on the caller's stream, 1 and 2 on side streams, every kernel on a third
        // of the SMs.  The MRF sum keeps its order (the last conv of branch j waits for that of branch j - 1), so the
        // result is bit-identical to the sequential schedule.
        CK(cudaEventRecord(c->br_ev[3], r.st));
        TcExtra third;
        third.grid_div = 3;
        for (int j = 0; j < 3; ++j) {
          Run rj = r;
          if (j > 0) {
            rj.st = c->br_stream[j - 1];
            CK(cudaStreamWaitEvent(rj.st, c->br_ev[3], 0));
          }
          float* Bj = j == 0 ? bufB : ws + W.brB[j - 1];
          float* Cj = j == 0 ? bufC : ws + W.brC[j - 1];
          for (int d = 0; d < 3; ++d) {
            const float* xin = d == 0 ? bufA : Bj;
            TRY(launch_tc(rj, c->tc_c1[i * 3 + j][d], xin, Cj, nullptr, Tlen, up_out, 0.1f, 1.f, 0, 1, third));
            if (d == 2 && j > 0) CK(cudaStreamWaitEvent(rj.st, c->br_ev[j - 1], 0));   // xs so far is complete
            float* yout = d < 2 ? Bj : bufD;
            TRY(launch_tc(rj, c->tc_c2[i * 3 + j][d], Cj, yout, xin, Tlen, up_out, 0.1f,
                          (d == 2 && j == 2) ? 1.0f / 3.0f : 1.f, (d == 2 && j > 0) ? 1 : 0, 1, third));
          }
          CK(cudaEventRecord(c->br_ev[j], rj.st));
        }
        CK(cudaStreamWaitEvent(r.st, c->br_ev[2], 0));   // join (branch 1 is joined through branch 2's wait)
      }
      snprintf(nm, sizeof nm, "dec.stage%d", i);
      TRY(tap_cl(nm, bufD, cout, Tlen, pitch_out));
      stage_in = bufD;   // the next upsampling consumes xs before that stage's MRF rewrites bufD (stream order)
      cin = cout; up = up_out;
    }
    const int y_len = Tmax * up;
    dim3 grid((y_len + 255) / 256, B);
    conv_post_cl_kernel<32><<<grid, 256, 0, st>>>(stage_in, 32LL * P * up, c->d_w + c->post_w_off, o_hat, (long long)y_len,
                                                 y_len, r.glens, Tmax, up);
    CK(cudaGetLastError());
    c->launches++;
    return OVC_OK;
  }
  const float* stage_in = ws + W.dpre;
  int cin = 512, up = 1;
  for (int i = 0; i < 4; ++i) {
    const int s = c->hp.upsample_rates[i];
    const int cout = cin / 2;
    const int up_out = up * s;
    const int pitch_in = P * up, pitch_out = P * up_out;
    // leaky_relu(0.1) + ConvTranspose1d (models.py:278-279), polyphase
    {
      ConvArgs a{};
      a.x = stage_in; a.x_bs = (long long)cin * pitch_in; a.x_pitch = pitch_in;
      a.bias = c->d_w + c->dec_ups[i].b_off; a.bias_bs = 0;
      a.y = bufA; a.y_bs = (long long)cout * pitch_out; a.y_pitch = pitch_out;
      a.lens_in = r.glens; a.lens_out = r.glens; a.mul_in = up; a.mul_out = up;   // kernel time axis = input samples
      a.slope = 0.1f;
      TRY(launch(r, c->dec_ups[i], a, Tmax * up));
      char nm[32]; snprintf(nm, sizeof nm, "dec.ups%d", i);
      TRY(tap(r, nm, bufA, cout, Tmax * up_out, pitch_out));
    }
    // MRF: xs = sum_j ResBlock1_j(x) / 3 (models.py:280-286; ResBlock1 = modules.py:296-309)
    const long long bsC = (long long)cout * pitch_out;
    const int Tlen = Tmax * up_out;
    for (int j = 0; j < 3; ++j) {
      const int K = c->hp.resblock_kernel_sizes[j];
      for (int d = 0; d < 3; ++d) {
        const double fl = 2.0 * cout * cout * K * r.sum_len * up_out;
        const double by = 2.0 * cout * r.sum_len * up_out * 4.0;
        const float* xin = d == 0 ? bufA : bufB;
        ConvArgs a{};
        a.x = xin; a.x_bs = bsC; a.x_pitch = pitch_out;
        a.bias = c->d_w + c->rb_c1[i * 3 + j][d].b_off; a.bias_bs = 0;
        a.y = bufC; a.y_bs = bsC; a.y_pitch = pitch_out;
        a.lens_in = r.glens; a.lens_out = r.glens; a.mul_in = up_out; a.mul_out = up_out;
        a.slope = 0.1f; a.scale = 1.f;
        TRY(launch(r, c->rb_c1[i * 3 + j][d], a, Tlen, true, fl, by));
        ConvArgs b{};
        b.x = bufC; b.x_bs = bsC; b.x_pitch = pitch_out;
        b.bias = c->d_w + c->rb_c2[i * 3 + j][d].b_off; b.bias_bs = 0;
        b.r = xin; b.r_bs = bsC; b.r_pitch = pitch_out;
        b.lens_in = r.glens; b.lens_out = r.glens; b.mul_in = up_out; b.mul_out = up_out;
        b.slope = 0.1f; b.scale = 1.f;
        if (d < 2) {
          b.y = bufB; b.y_bs = bsC; b.y_pitch = pitch_out;
        } else {
          b.y = bufD; b.y_bs = bsC; b.y_pitch = pitch_out;
          if (j > 0) b.flags = F_ACCUM;
          if (j == 2) b.scale = 1.0f / 3.0f;   // xs / num_kernels (models.py:286), as a multiply
        }
        TRY(launch(r, c->rb_c2[i * 3 + j][d], b, Tlen, true, fl, by));
      }
    }
    char nm[32]; snprintf(nm, sizeof nm, "dec.stage%d", i);
    TRY(tap(r, nm, bufD, cout, Tlen, pitch_out));
    stage_in = bufD;
    cin = cout; up = up_out;
  }
  // leaky_relu(0.01) + conv_post + tanh (models.py:287-289)
  {
    const int y_len = Tmax * up;   // 256 * Tmax
    dim3 grid((y_len / 4 + 255) / 256, B);
    conv_post_kernel<32><<<grid, 256, 0, st>>>(stage_in, 32LL * P * up, P * up, c->d_w + c->post_w_off, o_hat,
                                              (long long)y_len, y_len, r.glens, Tmax, up);
    CK(cudaGetLastError());
    c->launches++;
  }
  return OVC_OK;
}

static int cond_pf_cols(const ovc_ctx* c, int se_frames) {
  return se_frames ? c->cond_pf_cols[c->precision >= 1][se_frames - 1] : 0;
}

// se_frames: OVC_SE_FRAMES_SRC / _TGT bits, the sides given per frame ([B][gin][Tmax]) rather than per item ([B][gin])
static int run_vc(ovc_ctx* c, const float* spec, int spec_pitch, const long long* lens, const float* g_src, const float* g_tgt,
                  int se_frames, const float* noise, uint64_t seed, float tau, int B, int Tmax, int ragged, float* o_hat,
                  float* z_out, float* zp_out, float* zh_out, cudaStream_t st) {
  const int n_pf = cond_pf_cols(c, se_frames);
  const WsLayout W = ws_layout(c, B, Tmax, n_pf);
  TRY(ensure_ws(c, W, B, Tmax, st));
  float* ws = c->d_ws;
  Run r{c, st, B, Tmax, W.P, lens, ragged ? lens : nullptr, (double)B * Tmax};
  c->launches = 0;
  const int P = W.P;
  const long long bs192 = 192LL * P;

  // ---- every speaker-conditioning 1x1 conv in one launch; with a time-varying side, a second launch computes the
  // sections that read it for every frame (the per-item vectors of those sections then go unread)
  const int o = c->precision >= 1;
  const bool src_pf = se_frames & OVC_SE_FRAMES_SRC, tgt_pf = se_frames & OVC_SE_FRAMES_TGT;
  TRY(launch_cond(c, st, B, 1, nullptr, c->cond_rows_out, cond_side(c, src_pf ? nullptr : g_src, false, Tmax),
                  cond_side(c, tgt_pf ? nullptr : g_tgt, false, Tmax), ws + W.cond, c->cond_rows_out, 0));
  if (n_pf)
    TRY(launch_cond(c, st, B, Tmax, c->d_cond_cols[o][se_frames - 1], n_pf, cond_side(c, src_pf ? g_src : nullptr, true, Tmax),
                    cond_side(c, tgt_pf ? g_tgt : nullptr, true, Tmax), ws + W.cond_pf, (long long)Tmax * n_pf, n_pf));
  const float* cond = ws + W.cond;
  TRY(tap(r, "cond", cond, 1, c->cond_rows_out, c->cond_rows_out));
  const int sec[2][4] = {{c->cond_off_enc, c->cond_off_fsrc, c->cond_off_ftgt, c->cond_off_dec},
                         {c->cond_off_enc_tc, c->cond_off_fsrc_tc, c->cond_off_ftgt_tc, c->cond_off_dec}};
  CondRef cr[4];   // enc, flow src, flow tgt, dec
  for (int k = 0; k < 4; ++k) {
    const int pf = n_pf ? c->cond_pf_off[o][se_frames - 1][k] : -1;
    cr[k] = pf < 0 ? CondRef{cond + sec[o][k], c->cond_rows_out, 0}
                   : CondRef{ws + W.cond_pf + pf, (long long)Tmax * n_pf, n_pf};
  }

  // ---- posterior encoder (models.py:212-221)
  {
    ConvArgs a{};
    a.x = spec; a.x_bs = (long long)c->hp.spec_channels * spec_pitch; a.x_pitch = spec_pitch;
    a.bias = c->d_w + c->enc_pre.b_off; a.bias_bs = 0;
    a.y = ws + W.x; a.y_bs = bs192; a.y_pitch = P;
    a.lens_in = lens; a.lens_out = lens; a.mul_in = 1; a.mul_out = 1;
    a.slope = 1.f; a.scale = 1.f;
    const bool aligned = (spec_pitch % 4 == 0) && ((reinterpret_cast<uintptr_t>(spec) & 15) == 0);
    TRY(launch(r, aligned ? c->enc_pre16 : c->enc_pre, a, Tmax));
    TRY(tap(r, "enc.pre", ws + W.x, 192, Tmax, P));
    if (c->precision >= 1) {
      TRY(run_wn_tc(r, c->enc_wn, ws + W.x, ws + W.skip, ws + W.acts, ws + W.bufA, ws + W.bufB, cr[0]));
    } else {
      TRY(run_wn(r, c->enc_wn, ws + W.x, ws + W.skip, ws + W.acts, cr[0]));
    }
    TRY(tap(r, "enc.wn", ws + W.skip, 192, Tmax, P));
    ConvArgs p{};
    p.x = ws + W.skip; p.x_bs = bs192; p.x_pitch = P;
    p.bias = c->d_w + c->enc_proj.b_off; p.bias_bs = 0;
    p.y = ws + W.z; p.y_bs = bs192; p.y_pitch = P;
    p.r = noise; p.r_bs = 192LL * Tmax; p.r_pitch = Tmax;
    p.lens_in = lens; p.lens_out = lens; p.mul_in = 1; p.mul_out = 1;
    p.slope = 1.f; p.tau = tau; p.seed = seed;
    p.callp = c->d_callp;       // set_call_params_kernel wrote (seed, tau, per-item arrays) there earlier on this stream
    TRY(launch(r, c->enc_proj, p, Tmax));
  }
  auto copy_latent = [&](float* dst) -> int { return copy_latent_out(r, W, ws, dst); };
  TRY(copy_latent(z_out));
  // ---- flow forward with g_src, reverse with g_tgt (models.py:496-497)
  TRY(run_flow(r, W, ws, false, cr[1]));
  TRY(copy_latent(zp_out));
  TRY(run_flow(r, W, ws, true, cr[2]));
  TRY(copy_latent(zh_out));
  if (!o_hat) return OVC_OK;   // the latent half alone (ovc_voice_conversion_frames with o_hat NULL)

  return run_dec(r, W, ws, cr[3], lens, o_hat);
}

// The generator half of run_vc: z_hat [B][192][Tmax] from the caller (zero from each length on, as the flow leaves it
// masked) through the same conditioning and run_dec, so a latent-half call followed by this one is run_vc bit for bit.
// Only the target side is read: the per-item launch computes every column (the source columns read zeros and go
// unread), a per-frame target only the generator's section of its per-frame columns.
static int run_gen(ovc_ctx* c, const float* z_hat, const long long* lens, const float* g_tgt, int se_frames, int B, int Tmax,
                   float* o_hat, cudaStream_t st) {
  const WsLayout W = ws_layout(c, B, Tmax, cond_pf_cols(c, se_frames));
  TRY(ensure_ws(c, W, B, Tmax, st));
  float* ws = c->d_ws;
  Run r{c, st, B, Tmax, W.P, lens, lens, (double)B * Tmax};
  c->launches = 0;
  const int o = c->precision >= 1;
  const bool tgt_pf = se_frames & OVC_SE_FRAMES_TGT;
  TRY(launch_cond(c, st, B, 1, nullptr, c->cond_rows_out, cond_side(c, nullptr, false, Tmax),
                  cond_side(c, tgt_pf ? nullptr : g_tgt, false, Tmax), ws + W.cond, c->cond_rows_out, 0));
  const int pf = tgt_pf ? c->cond_pf_off[o][OVC_SE_FRAMES_TGT - 1][3] : -1;   // -1: zero_g, the generator reads no g
  const int n_dec = 512;   // the generator's section: dec.cond rows (ovc_finalize_weights)
  if (pf >= 0)
    TRY(launch_cond(c, st, B, Tmax, c->d_cond_cols[o][OVC_SE_FRAMES_TGT - 1] + pf, n_dec, cond_side(c, nullptr, true, Tmax),
                    cond_side(c, g_tgt, true, Tmax), ws + W.cond_pf, (long long)Tmax * n_dec, n_dec));
  const CondRef cr = pf < 0 ? CondRef{ws + W.cond + c->cond_off_dec, c->cond_rows_out, 0}
                            : CondRef{ws + W.cond_pf, (long long)Tmax * n_dec, n_dec};
  dim3 grid((W.P + 255) / 256, 192, B);
  latent_in_kernel<<<grid, 256, 0, st>>>(z_hat, Tmax, ws + W.z, W.P, 192, lens);
  CK(cudaGetLastError());
  c->launches++;
  return run_dec(r, W, ws, cr, lens, o_hat);
}

#include "ovc_tts_run.inc"    // run_tts_encode() / run_tts_decode(): SynthesizerTrn.infer on the device

}  // namespace ovc

// =================================================================================================
// C ABI
// =================================================================================================
extern "C" {

int ovc_abi_version(void) { return OVC_ABI_VERSION; }

const char* ovc_last_error(void) { return ovc::g_err.c_str(); }

int ovc_create(const ovc_hparams* hp, int device, ovc_ctx** out) {
  if (!hp || !out) return fail(OVC_ERR_INVALID, "null argument");
  *out = nullptr;
  int rc = validate_hparams(hp);
  if (rc != OVC_OK) return rc;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    cudaGetLastError();
    return fail(OVC_ERR_CUDA, "no CUDA device available (%s); this library has no CPU path",
                e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
  }
  if (device < 0 || device >= n) return fail(OVC_ERR_INVALID, "device %d out of range (0..%d)", device, n - 1);
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)
    return fail(OVC_ERR_CUDA, "device %d is sm_%d%d; this library contains sm_90a code only", device, prop.major, prop.minor);
  ovc_ctx* c = new ovc_ctx();
  c->hp = *hp;
  c->device = device;
  c->sm_count = prop.multiProcessorCount;
  *out = c;
  return OVC_OK;
}

void ovc_destroy(ovc_ctx* c) {
  if (!c) return;
  DeviceGuard dev_guard_(c->device);
  if (c->d_w) cudaFree(c->d_w);
  if (c->d_ws) cudaFree(c->d_ws);
  if (c->d_tts) cudaFree(c->d_tts);
  if (c->d_cond_wrow) cudaFree(c->d_cond_wrow);
  if (c->d_cond_sel) cudaFree(c->d_cond_sel);
  for (auto& oc : c->d_cond_cols)
    for (int* p : oc)
      if (p) cudaFree(p);
  if (c->d_tcw) cudaFree(c->d_tcw);
  if (c->d_re) cudaFree(c->d_re);
  if (c->d_res) cudaFree(c->d_res);
  for (auto& kv : c->rs_banks) cudaFree(kv.second);
  if (c->d_rs_plans) cudaFree(c->d_rs_plans);
  if (c->d_tw) cudaFree(c->d_tw);
  if (c->d_win) cudaFree(c->d_win);
  drop_graphs(c);
  for (auto& q : c->br_stream)
    if (q) cudaStreamDestroy(q);
  for (auto& q : c->br_ev)
    if (q) cudaEventDestroy(q);
  if (c->cap_stream) cudaStreamDestroy(c->cap_stream);
  if (c->d_callp) cudaFree(c->d_callp);
  for (auto& e : c->ev) cudaEventDestroy(e);
  for (auto& kv : c->taps)
    if (kv.second.d) cudaFree(kv.second.d);
  delete c;
}

int ovc_load_tensor(ovc_ctx* c, const char* key, const float* data, const int64_t* shape, int ndim) {
  if (!c || !key || !data || !shape || ndim < 1 || ndim > 4) return fail(OVC_ERR_INVALID, "bad argument to ovc_load_tensor");
  const std::string k(key);
  if (!key_is_hot(k)) return 1;
  HostTensor t;
  t.shape.assign(shape, shape + ndim);
  const int64_t n = t.numel();
  if (n <= 0) return fail(OVC_ERR_INVALID, "tensor '%s' is empty", key);
  t.data.assign(data, data + n);
  c->sd[k] = std::move(t);
  c->finalized = false;
  return OVC_OK;
}

int ovc_finalize_weights(ovc_ctx* c) {
  if (!c) return fail(OVC_ERR_INVALID, "null context");
  return finalize(c);
}

size_t ovc_workspace_floats(const ovc_ctx* c, int B, int Tmax) {
  if (!c || B < 1 || Tmax < 1 || !c->finalized) return 0;
  return ws_layout(c, B, Tmax).total;
}

int ovc_voice_conversion(ovc_ctx* c, const float* spec, const int64_t* lengths, const float* g_src, const float* g_tgt,
                         const float* noise, uint64_t seed, float tau, int B, int Tmax, int ragged, float* o_hat, float* z,
                         float* z_p, float* z_hat, void* stream) {
  return ovc_voice_conversion_items(c, spec, lengths, g_src, g_tgt, noise, seed, tau, B, Tmax, ragged, o_hat, z, z_p, z_hat,
                                    stream, nullptr);
}

int ovc_voice_conversion_items(ovc_ctx* c, const float* spec, const int64_t* lengths, const float* g_src, const float* g_tgt,
                               const float* noise, uint64_t seed, float tau, int B, int Tmax, int ragged, float* o_hat,
                               float* z, float* z_p, float* z_hat, void* stream, const ovc_item_params* items) {
  return ovc_voice_conversion_frames(c, spec, lengths, g_src, g_tgt, 0, noise, seed, tau, B, Tmax, ragged, o_hat, z, z_p, z_hat,
                                     stream, items);
}

int ovc_voice_conversion_frames(ovc_ctx* c, const float* spec, const int64_t* lengths, const float* g_src, const float* g_tgt,
                                int se_frames, const float* noise, uint64_t seed, float tau, int B, int Tmax, int ragged,
                                float* o_hat, float* z, float* z_p, float* z_hat, void* stream, const ovc_item_params* items) {
  if (!c) return fail(OVC_ERR_INVALID, "null context");
  if (se_frames & ~(OVC_SE_FRAMES_SRC | OVC_SE_FRAMES_TGT)) return fail(OVC_ERR_INVALID, "unknown se_frames bits 0x%x", se_frames);
  if (!c->finalized) return fail(OVC_ERR_STATE, "ovc_finalize_weights has not been called");
  if (!spec || !lengths || !g_src || !g_tgt) return fail(OVC_ERR_INVALID, "null tensor argument");
  if (!o_hat && !z && !z_p && !z_hat) return fail(OVC_ERR_INVALID, "no output: o_hat, z, z_p and z_hat are all NULL");
  if (B < 1 || Tmax < 1) return fail(OVC_ERR_INVALID, "B and Tmax must be positive (got %d, %d)", B, Tmax);
  if ((long long)Tmax * 256 * 64 > 2000000000LL) return fail(OVC_ERR_INVALID, "Tmax %d too large for 32-bit indexing", Tmax);
  if (B > 65535) return fail(OVC_ERR_INVALID, "B %d exceeds the grid limit", B);
  ON_DEVICE(c);
  c->ev_used = c->prof ? c->ev_used : 0;
  cudaStream_t st = (cudaStream_t)stream;
  TRY(ensure_ws(c, ws_layout(c, B, Tmax, cond_pf_cols(c, se_frames)), B, Tmax, st));
  const ItemParams it = item_params(items);
  TRY(set_call_params(c, seed, tau, it, st));
  std::vector<uintptr_t> key = {1, (uintptr_t)spec, (uintptr_t)lengths, (uintptr_t)g_src, (uintptr_t)g_tgt, (uintptr_t)noise,
                                (uintptr_t)o_hat, (uintptr_t)z, (uintptr_t)z_p, (uintptr_t)z_hat, (uintptr_t)B, (uintptr_t)Tmax,
                                (uintptr_t)ragged, option_bits(c), (uintptr_t)se_frames};
  append_item_key(key, it);
  return run_graphed(c, key, st, [&](cudaStream_t s) {
    return run_vc(c, spec, Tmax, (const long long*)lengths, g_src, g_tgt, se_frames, noise, seed, tau, B, Tmax, ragged, o_hat, z,
                  z_p, z_hat, s);
  });
}

int ovc_generate_frames(ovc_ctx* c, const float* z_hat, const int64_t* lengths, const float* g_tgt, int se_frames, int B,
                        int Tmax, float* o_hat, void* stream) {
  if (!c) return fail(OVC_ERR_INVALID, "null context");
  if (se_frames & ~OVC_SE_FRAMES_TGT)
    return fail(OVC_ERR_INVALID, "ovc_generate_frames: se_frames 0x%x (the generator reads the target side only)", se_frames);
  if (!c->finalized) return fail(OVC_ERR_STATE, "ovc_finalize_weights has not been called");
  if (!z_hat || !lengths || !g_tgt || !o_hat) return fail(OVC_ERR_INVALID, "null tensor argument");
  if (B < 1 || Tmax < 1) return fail(OVC_ERR_INVALID, "B and Tmax must be positive (got %d, %d)", B, Tmax);
  if ((long long)Tmax * 256 * 64 > 2000000000LL) return fail(OVC_ERR_INVALID, "Tmax %d too large for 32-bit indexing", Tmax);
  if (B > 65535) return fail(OVC_ERR_INVALID, "B %d exceeds the grid limit", B);
  ON_DEVICE(c);
  c->ev_used = c->prof ? c->ev_used : 0;
  cudaStream_t st = (cudaStream_t)stream;
  TRY(ensure_ws(c, ws_layout(c, B, Tmax, cond_pf_cols(c, se_frames)), B, Tmax, st));
  const std::vector<uintptr_t> key = {4, (uintptr_t)z_hat, (uintptr_t)lengths, (uintptr_t)g_tgt, (uintptr_t)o_hat, (uintptr_t)B,
                                      (uintptr_t)Tmax, option_bits(c), (uintptr_t)se_frames};
  return run_graphed(c, key, st, [&](cudaStream_t s) {
    return run_gen(c, z_hat, (const long long*)lengths, g_tgt, se_frames, B, Tmax, o_hat, s);
  });
}

static int launch_stft(ovc_ctx* c, const float* wav, const int64_t* wav_lengths, int B, int Lmax, int Tmax, float* spec,
                       int spec_pitch, long long* frames, cudaStream_t st) {
  if (c->hp.spec_channels != STFT_N / 2 + 1 || c->hp.hop_length != 256)
    return fail(OVC_ERR_INVALID, "the STFT kernel is specialised for n_fft = win_length = 1024, hop 256");
  dim3 grid((Tmax + STFT_FR - 1) / STFT_FR, B);
  stft_mag_kernel<<<grid, 256, 0, st>>>(wav, (long long)Lmax, (const long long*)wav_lengths, c->hp.hop_length, spec,
                                        (long long)c->hp.spec_channels * spec_pitch, spec_pitch, Tmax, c->d_tw, c->d_win,
                                        frames);
  CK(cudaGetLastError());
  return OVC_OK;
}

int ovc_spectrogram(ovc_ctx* c, const float* wav, const int64_t* wav_lengths, int B, int Lmax, int Tmax, float* spec,
                    int64_t* frames, void* stream) {
  if (!c) return fail(OVC_ERR_INVALID, "null context");
  if (!c->finalized) return fail(OVC_ERR_STATE, "ovc_finalize_weights has not been called");
  if (!wav || !wav_lengths || !spec) return fail(OVC_ERR_INVALID, "null tensor argument");
  if (B < 1 || Lmax < 1 || Tmax < 1 || B > 65535) return fail(OVC_ERR_INVALID, "bad sizes B=%d Lmax=%d Tmax=%d", B, Lmax, Tmax);
  ON_DEVICE(c);
  return launch_stft(c, wav, wav_lengths, B, Lmax, Tmax, spec, Tmax, (long long*)frames, (cudaStream_t)stream);
}

static_assert(RING_OPEN == INT64_MAX, "ovc_spectrogram_ring: INT64_MAX marks an open stream");

int ovc_spectrogram_ring(ovc_ctx* c, const float* rings, int ring_rows, int64_t ring_cap, const int64_t* row,
                         const int64_t* frame_lo, const int64_t* frames, const int64_t* stream_len, int B, int Tmax,
                         float* spec, void* stream) {
  if (!c) return fail(OVC_ERR_INVALID, "null context");
  if (!c->finalized) return fail(OVC_ERR_STATE, "ovc_finalize_weights has not been called");
  if (!rings || !row || !frame_lo || !frames || !stream_len || !spec) return fail(OVC_ERR_INVALID, "null tensor argument");
  if (B < 1 || Tmax < 1 || B > 65535 || ring_rows < 1)
    return fail(OVC_ERR_INVALID, "bad sizes B=%d Tmax=%d ring_rows=%d", B, Tmax, ring_rows);
  if (ring_cap < STFT_N) return fail(OVC_ERR_INVALID, "ring_cap %lld is below one FFT frame (%d)", (long long)ring_cap, STFT_N);
  if (c->hp.spec_channels != STFT_N / 2 + 1 || c->hp.hop_length != 256)
    return fail(OVC_ERR_INVALID, "the STFT kernel is specialised for n_fft = win_length = 1024, hop 256");
  ON_DEVICE(c);
  dim3 grid((Tmax + STFT_FR - 1) / STFT_FR, B);
  stft_ring_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(rings, (long long)ring_cap, ring_rows, (const long long*)row,
                                                           (const long long*)frame_lo, (const long long*)frames,
                                                           (const long long*)stream_len, c->hp.hop_length, spec, Tmax,
                                                           c->d_tw, c->d_win);
  CK(cudaGetLastError());
  return OVC_OK;
}

int ovc_convert_waveform(ovc_ctx* c, const float* wav, const int64_t* wav_lengths, int B, int Lmax, const float* g_src,
                         const float* g_tgt, const float* noise, uint64_t seed, float tau, float* o_hat, int64_t* frames,
                         void* stream) {
  return ovc_convert_waveform_items(c, wav, wav_lengths, B, Lmax, g_src, g_tgt, noise, seed, tau, o_hat, frames, stream, nullptr);
}

int ovc_convert_waveform_items(ovc_ctx* c, const float* wav, const int64_t* wav_lengths, int B, int Lmax, const float* g_src,
                               const float* g_tgt, const float* noise, uint64_t seed, float tau, float* o_hat, int64_t* frames,
                               void* stream, const ovc_item_params* items) {
  return ovc_convert_waveform_frames(c, wav, wav_lengths, B, Lmax, g_src, g_tgt, 0, noise, seed, tau, o_hat, frames, stream, items);
}

int ovc_convert_waveform_frames(ovc_ctx* c, const float* wav, const int64_t* wav_lengths, int B, int Lmax, const float* g_src,
                                const float* g_tgt, int se_frames, const float* noise, uint64_t seed, float tau, float* o_hat,
                                int64_t* frames, void* stream, const ovc_item_params* items) {
  if (!c) return fail(OVC_ERR_INVALID, "null context");
  if (se_frames & ~(OVC_SE_FRAMES_SRC | OVC_SE_FRAMES_TGT)) return fail(OVC_ERR_INVALID, "unknown se_frames bits 0x%x", se_frames);
  if (!c->finalized) return fail(OVC_ERR_STATE, "ovc_finalize_weights has not been called");
  if (!wav || !wav_lengths || !g_src || !g_tgt || !o_hat) return fail(OVC_ERR_INVALID, "null tensor argument");
  const int Tmax = Lmax / c->hp.hop_length;
  if (B < 1 || Tmax < 1 || B > 65535) return fail(OVC_ERR_INVALID, "bad sizes B=%d Lmax=%d", B, Lmax);
  if ((long long)Tmax * 256 * 64 > 2000000000LL) return fail(OVC_ERR_INVALID, "Lmax %d too large for 32-bit indexing", Lmax);
  ON_DEVICE(c);
  cudaStream_t st = (cudaStream_t)stream;
  const WsLayout W = ws_layout(c, B, Tmax, cond_pf_cols(c, se_frames));
  TRY(ensure_ws(c, W, B, Tmax, st));
  const ItemParams it = item_params(items);
  TRY(set_call_params(c, seed, tau, it, st));
  std::vector<uintptr_t> key = {2, (uintptr_t)wav, (uintptr_t)wav_lengths, (uintptr_t)g_src, (uintptr_t)g_tgt, (uintptr_t)noise,
                                (uintptr_t)o_hat, (uintptr_t)frames, (uintptr_t)B, (uintptr_t)Lmax, option_bits(c),
                                (uintptr_t)se_frames};
  append_item_key(key, it);
  return run_graphed(c, key, st, [&](cudaStream_t s) {
    float* spec = c->d_ws + W.spec;
    long long* fr = reinterpret_cast<long long*>(c->d_ws + W.frames);
    TRY(launch_stft(c, wav, wav_lengths, B, Lmax, Tmax, spec, W.P, fr, s));
    if (frames) CK(cudaMemcpyAsync(frames, fr, (size_t)B * sizeof(long long), cudaMemcpyDeviceToDevice, s));
    const int rc = run_vc(c, spec, W.P, fr, g_src, g_tgt, se_frames, noise, seed, tau, B, Tmax, 1, o_hat, nullptr, nullptr,
                          nullptr, s);
    c->launches += 1;
    return rc;
  });
}

int ovc_tone_track_expand(ovc_ctx* c, const int64_t* key_frame, const float* key_se, int64_t n_keys, const int64_t* key0,
                          const int64_t* nkeys, const int64_t* frame0, const int64_t* frames, int B, int Tmax, float* out,
                          void* stream) {
  if (!c) return fail(OVC_ERR_INVALID, "null context");
  if (!key_frame || !key_se || !key0 || !nkeys || !frame0 || !frames || !out) return fail(OVC_ERR_INVALID, "null tensor argument");
  if (n_keys < 1 || B < 1 || B > 65535 || Tmax < 1) return fail(OVC_ERR_INVALID, "bad sizes n_keys=%lld B=%d Tmax=%d", (long long)n_keys, B, Tmax);
  const int G = c->hp.gin_channels;
  if (G > 65535) return fail(OVC_ERR_INVALID, "gin_channels %d exceeds the grid limit", G);
  ON_DEVICE(c);
  dim3 grid((Tmax + 255) / 256, G, B);
  tone_track_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const long long*)key_frame, key_se, (long long)n_keys,
                                                            (const long long*)key0, (const long long*)nkeys,
                                                            (const long long*)frame0, (const long long*)frames, G, Tmax, out);
  CK(cudaGetLastError());
  return OVC_OK;
}

// ovc_reference_encoder (lengths == nullptr: every item T frames) and ovc_reference_encoder_ragged
static int run_refenc(ovc_ctx* c, const float* spec, const long long* lengths, int N, int T, float* out, void* stream) {
  if (!c) return fail(OVC_ERR_INVALID, "null context");
  if (!c->finalized) return fail(OVC_ERR_STATE, "ovc_finalize_weights has not been called");
  if (!c->has_refenc) return fail(OVC_ERR_MISSING, "the checkpoint had no ref_enc.* tensors");
  if (!spec || !out || N < 1 || T < 1) return fail(OVC_ERR_INVALID, "bad argument to ovc_reference_encoder");
  ON_DEVICE(c);
  cudaStream_t st = (cudaStream_t)stream;
  const int F = c->hp.spec_channels, G = c->hp.gin_channels;
  static const int filt[7] = {1, 32, 32, 64, 64, 128, 128};
  int H[7], W[7];
  H[0] = T; W[0] = F;
  size_t maxact = (size_t)N * T * F;
  for (int i = 0; i < 6; ++i) {
    H[i + 1] = (H[i] - 1) / 2 + 1; W[i + 1] = (W[i] - 1) / 2 + 1;
    maxact = std::max(maxact, (size_t)N * filt[i + 1] * H[i + 1] * W[i + 1]);
  }
  if (128 * W[6] != c->re_gru_in)
    return fail(OVC_ERR_INVALID, "ref_enc.gru.weight_ih_l0 takes %d inputs but spec_channels %d gives %d", c->re_gru_in, F, 128 * W[6]);
  const size_t gi_floats = (size_t)N * H[6] * 384;
  const size_t need = 2 * round_up(maxact, 64) + round_up(gi_floats, 64);
  if (need > c->re_floats) {
    CK(cudaStreamSynchronize(st));
    if (c->d_re) CK(cudaFree(c->d_re));
    c->d_re = nullptr; c->re_floats = 0;
    CK(cudaMalloc(&c->d_re, need * sizeof(float)));
    c->re_floats = need;
  }
  float* a0 = c->d_re;
  float* a1 = a0 + round_up(maxact, 64);
  float* gi = a1 + round_up(maxact, 64);
  {
    const int warps = N * T;
    refenc_layernorm_kernel<<<(warps * 32 + 255) / 256, 256, 0, st>>>(spec, c->d_w + c->re_lng, c->d_w + c->re_lnb, a0, N, F, T,
                                                                      (const int64_t*)lengths);
    CK(cudaGetLastError());
  }
  float* cur = a0; float* nxt = a1;
  for (int i = 0; i < 6; ++i) {
    const long long total = (long long)N * filt[i + 1] * H[i + 1] * W[i + 1];
    refenc_conv_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(cur, c->d_w + c->re_conv_w[i], c->d_w + c->re_conv_b[i], nxt, N,
                                                                        filt[i], H[i], W[i], filt[i + 1], H[i + 1], W[i + 1],
                                                                        (const int64_t*)lengths, T, i);
    CK(cudaGetLastError());
    std::swap(cur, nxt);
  }
  {
    const long long warps = (long long)N * H[6] * 384;
    refenc_gru_in_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, st>>>(cur, c->d_w + c->re_wih, c->d_w + c->re_bih, gi, N, 128,
                                                                              H[6], W[6], 384, (const int64_t*)lengths, T);
    CK(cudaGetLastError());
    refenc_gru_kernel<<<N, 128, 0, st>>>(gi, c->d_w + c->re_whh, c->d_w + c->re_bhh, c->d_w + c->re_pw, c->d_w + c->re_pb, out, H[6], G,
                                         (const int64_t*)lengths, T);
    CK(cudaGetLastError());
  }
  return OVC_OK;
}

int ovc_reference_encoder(ovc_ctx* c, const float* spec, int N, int T, float* out, void* stream) {
  return run_refenc(c, spec, nullptr, N, T, out, stream);
}

int ovc_reference_encoder_ragged(ovc_ctx* c, const float* spec, const int64_t* lengths, int N, int Tmax, float* out,
                                 void* stream) {
  if (!lengths) return fail(OVC_ERR_INVALID, "null lengths in ovc_reference_encoder_ragged");
  return run_refenc(c, spec, (const long long*)lengths, N, Tmax, out, stream);
}

size_t ovc_reference_encoder_stream_state_floats(const ovc_ctx* c) {
  if (!c || !c->finalized || !c->has_refenc) return 0;
  return (size_t)ovc_re::geom(c->hp.spec_channels).floats;
}

int ovc_reference_encoder_stream(ovc_ctx* c, const float* rings, int ring_rows, int64_t ring_cap, float* state, int state_rows,
                                 const int64_t* desc, int B, int max_new_frames, float* out, void* stream) {
  if (!c) return fail(OVC_ERR_INVALID, "null context");
  if (!c->finalized) return fail(OVC_ERR_STATE, "ovc_finalize_weights has not been called");
  if (!c->has_refenc) return fail(OVC_ERR_MISSING, "the checkpoint had no ref_enc.* tensors");
  if (!rings || !state || !desc || !out) return fail(OVC_ERR_INVALID, "null tensor argument");
  if (B < 1 || B > 65535 || ring_rows < 1 || state_rows < 1)
    return fail(OVC_ERR_INVALID, "bad sizes B=%d ring_rows=%d state_rows=%d", B, ring_rows, state_rows);
  if (max_new_frames < 1 || max_new_frames > ovc_re::MAX_NEW)
    return fail(OVC_ERR_INVALID, "max_new_frames %d outside [1, %d]", max_new_frames, ovc_re::MAX_NEW);
  if (ring_cap < STFT_N) return fail(OVC_ERR_INVALID, "ring_cap %lld is below one FFT frame (%d)", (long long)ring_cap, STFT_N);
  if (c->hp.spec_channels != STFT_N / 2 + 1 || c->hp.hop_length != 256)
    return fail(OVC_ERR_INVALID, "the STFT kernel is specialised for n_fft = win_length = 1024, hop 256");
  const int F = c->hp.spec_channels, G = c->hp.gin_channels;
  const ovc_re::Geom geo = ovc_re::geom(F);
  if (ovc_re::filt(ovc_re::LAYERS) * geo.W[ovc_re::LAYERS] != c->re_gru_in)
    return fail(OVC_ERR_INVALID, "ref_enc.gru.weight_ih_l0 takes %d inputs but spec_channels %d gives %d", c->re_gru_in, F,
                ovc_re::filt(ovc_re::LAYERS) * geo.W[ovc_re::LAYERS]);
  ON_DEVICE(c);
  cudaStream_t st = (cudaStream_t)stream;
  const int Tcols = max_new_frames + ovc_re::TAIL;
  const size_t spec_floats = round_up((size_t)B * F * Tcols, 64);
  const size_t item = (size_t)ovc_re::ws_floats(max_new_frames, F);
  const size_t need = spec_floats + (size_t)B * item;
  if (need > c->res_floats) {   // grows outside capture only: a captured call keeps the addresses it was captured with
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    CK(cudaStreamIsCapturing(st, &cs));
    if (cs != cudaStreamCaptureStatusNone)
      return fail(OVC_ERR_STATE, "ovc_reference_encoder_stream: B=%d max_new_frames=%d needs a larger workspace; make one such "
                  "call outside stream capture first", B, max_new_frames);
    CK(cudaStreamSynchronize(st));
    if (c->d_res) CK(cudaFree(c->d_res));
    c->d_res = nullptr; c->res_floats = 0;
    CK(cudaMalloc(&c->d_res, need * sizeof(float)));
    c->res_floats = need;
  }
  float* spec = c->d_res;
  dim3 grid((Tcols + STFT_FR - 1) / STFT_FR, B);
  stft_refenc_kernel<<<grid, 256, 0, st>>>(rings, (long long)ring_cap, ring_rows, state, state_rows, (long long)geo.floats, desc,
                                           max_new_frames, c->hp.hop_length, spec, Tcols, c->d_tw, c->d_win);
  CK(cudaGetLastError());
  RefencWeights P;
  P.ln_g = c->d_w + c->re_lng; P.ln_b = c->d_w + c->re_lnb;
  for (int i = 0; i < 6; ++i) { P.conv_w[i] = c->d_w + c->re_conv_w[i]; P.conv_b[i] = c->d_w + c->re_conv_b[i]; }
  P.w_ih = c->d_w + c->re_wih; P.b_ih = c->d_w + c->re_bih; P.w_hh = c->d_w + c->re_whh; P.b_hh = c->d_w + c->re_bhh;
  P.pw = c->d_w + c->re_pw; P.pb = c->d_w + c->re_pb;
  refenc_stream_kernel<<<B, 256, 0, st>>>(P, spec, Tcols, state, state_rows, desc, ring_rows, max_new_frames, c->hp.hop_length, F, G,
                                          spec + spec_floats, (long long)item, out);
  CK(cudaGetLastError());
  return OVC_OK;
}

static int resample_plan(int sr_in, int sr_out, ovc_rs::Plan* p) {
  if (ovc_rs::make_plan(sr_in, sr_out, p) != 0)
    return fail(OVC_ERR_INVALID, "cannot resample %d Hz -> %d Hz: both rates must be positive and the reduced ratio "
                "up/down must have max(up, down) <= %lld", sr_in, sr_out, (long long)ovc_rs::MAX_M);
  return OVC_OK;
}

int ovc_resample_span(int sr_in, int sr_out, int64_t n_in, int64_t m0, int64_t m1, int64_t* out4) {
  ovc_rs::Plan p;
  TRY(resample_plan(sr_in, sr_out, &p));
  if (!out4 || n_in < 0 || m0 < 0 || m1 <= m0) return fail(OVC_ERR_INVALID, "bad argument to ovc_resample_span");
  int64_t lo, hi;
  ovc_rs::span(p, m0, m1, &lo, &hi);
  out4[0] = ovc_rs::n_out(p, n_in);
  out4[1] = ovc_rs::n_ready(p, n_in);
  out4[2] = lo;
  out4[3] = hi;
  return OVC_OK;
}

static constexpr int64_t RS_SMEM_MAX = 200 * 1024;   // opt-in dynamic shared memory of the resample kernels

// stage a tile of plan p as doubles when one output's span fits shared memory as doubles
static bool resample_stage_dbl(const ovc_rs::Plan& p) {
  return resample_stage_len(p, 1) * (int64_t)sizeof(double) <= RS_SMEM_MAX;
}

// the context's bank of p, built and uploaded on first use (waits for `stream`)
static int resample_bank(ovc_ctx* c, const ovc_rs::Plan& p, double** out, cudaStream_t stream) {
  double*& bank = c->rs_banks[{p.up, p.down}];
  if (!bank) {
    const std::vector<double> h = ovc_rs::design_bank(p);
    CK(cudaMalloc(&bank, h.size() * sizeof(double)));
    // ordered on the call's stream (a non-blocking stream does not wait for the legacy default stream) and finished
    // before the pageable source goes out of scope
    CK(cudaMemcpyAsync(bank, h.data(), h.size() * sizeof(double), cudaMemcpyHostToDevice, stream));
    CK(cudaStreamSynchronize(stream));
  }
  *out = bank;
  return OVC_OK;
}

int ovc_resample(ovc_ctx* c, int sr_in, int sr_out, const float* in, const int64_t* in_lengths, int B, int64_t in_pitch,
                 int64_t in_start, float* out, int64_t out_pitch, int64_t out_start, void* stream) {
  if (!c) return fail(OVC_ERR_INVALID, "null context");
  ovc_rs::Plan p;
  TRY(resample_plan(sr_in, sr_out, &p));
  if (!in || !in_lengths || !out) return fail(OVC_ERR_INVALID, "null tensor argument");
  if (B < 1 || B > 65535 || in_pitch < 0 || out_pitch < 0 || out_start < 0)
    return fail(OVC_ERR_INVALID, "bad sizes B=%d in_pitch=%lld out_pitch=%lld out_start=%lld", B, (long long)in_pitch,
                (long long)out_pitch, (long long)out_start);
  if (out_pitch == 0) return OVC_OK;
  ON_DEVICE(c);
  double* bank = nullptr;
  TRY(resample_bank(c, p, &bank, (cudaStream_t)stream));
  // tile of up to 256 outputs whose staged span fits the opt-in shared memory; staged as doubles when one output's does
  const int64_t smem_max = RS_SMEM_MAX;
  const bool dbl = resample_stage_dbl(p);
  const int64_t elem = dbl ? sizeof(double) : sizeof(float);
  int tile = 256;
  while (tile > 1 && resample_stage_len(p, tile) * elem > smem_max) tile /= 2;
  const size_t smem = (size_t)(resample_stage_len(p, tile) * elem);
  const int64_t tiles = (out_pitch + tile - 1) / tile;
  if (tiles > 0x7fffffffLL) return fail(OVC_ERR_INVALID, "out_pitch %lld too large", (long long)out_pitch);
  const dim3 grid((unsigned)tiles, B);
  const int threads = std::min(256, (tile + 31) / 32 * 32);
  cudaStream_t st = (cudaStream_t)stream;
  if (!c->rs_smem_opt_in) {
    CK(cudaFuncSetAttribute(resample_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max));
    CK(cudaFuncSetAttribute(resample_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max));
    c->rs_smem_opt_in = true;
  }
  if (dbl) {
    resample_kernel<double><<<grid, threads, smem, st>>>(p, bank, in, in_pitch, in_start, (const int64_t*)in_lengths, out,
                                                         out_pitch, out_start, tile);
  } else {
    resample_kernel<float><<<grid, threads, smem, st>>>(p, bank, in, in_pitch, in_start, (const int64_t*)in_lengths, out,
                                                        out_pitch, out_start, tile);
  }
  CK(cudaGetLastError());
  return OVC_OK;
}

int ovc_resample_plan(ovc_ctx* c, int sr_in, int sr_out, int32_t* id, void* stream) {
  if (!c || !id) return fail(OVC_ERR_INVALID, "null argument to ovc_resample_plan");
  ovc_rs::Plan p;
  TRY(resample_plan(sr_in, sr_out, &p));
  for (size_t i = 0; i < c->rs_plans.size(); ++i)
    if (c->rs_plans[i].p.up == p.up && c->rs_plans[i].p.down == p.down) {
      *id = (int32_t)i;
      return OVC_OK;
    }
  ON_DEVICE(c);
  cudaStream_t st = (cudaStream_t)stream;
  RsRingPlan e;
  e.p = p;
  double* bank = nullptr;
  TRY(resample_bank(c, p, &bank, st));
  e.bank = bank;
  e.dbl = resample_stage_dbl(p) ? 1 : 0;
  std::vector<RsRingPlan> plans = c->rs_plans;
  plans.push_back(e);
  // one tile for every plan of the table: the largest (up to 256) whose staged span fits each plan's staging type
  auto bytes = [](const RsRingPlan& q, int tile) {
    return resample_stage_len(q.p, tile) * (int64_t)(q.dbl ? sizeof(double) : sizeof(float));
  };
  int tile = 256;
  for (;;) {
    bool fits = true;
    for (const RsRingPlan& q : plans) fits = fits && bytes(q, tile) <= RS_SMEM_MAX;
    if (fits || tile == 1) break;
    tile /= 2;
  }
  int64_t smem = 0;
  for (const RsRingPlan& q : plans) smem = std::max(smem, bytes(q, tile));
  RsRingPlan* table = nullptr;
  CK(cudaMalloc(&table, plans.size() * sizeof(RsRingPlan)));
  const cudaError_t up = cudaMemcpyAsync(table, plans.data(), plans.size() * sizeof(RsRingPlan), cudaMemcpyHostToDevice, st);
  const cudaError_t done = up == cudaSuccess ? cudaStreamSynchronize(st) : up;
  if (done != cudaSuccess) {
    cudaFree(table);
    return fail(OVC_ERR_CUDA, "ovc_resample_plan: %s", cudaGetErrorString(done));
  }
  CK(cudaFuncSetAttribute(resample_ring_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)RS_SMEM_MAX));
  if (c->d_rs_plans) CK(cudaFree(c->d_rs_plans));   // synchronises the device: no launch still reads the old table
  c->d_rs_plans = table;
  c->rs_plans = plans;
  c->rs_ring_tile = tile;
  c->rs_ring_smem = (size_t)smem;
  *id = (int32_t)(plans.size() - 1);
  return OVC_OK;
}

int ovc_resample_rings(ovc_ctx* c, const int32_t* plan, const float* in, int in_rows, int64_t in_cap,
                       const int64_t* in_row, const int64_t* in_len, const int64_t* m0, const int64_t* count, float* out,
                       int out_rows, int64_t out_cap, const int64_t* out_row, const int64_t* out_off, int B,
                       int64_t max_count, void* stream) {
  if (!c) return fail(OVC_ERR_INVALID, "null context");
  if (c->rs_plans.empty()) return fail(OVC_ERR_STATE, "ovc_resample_rings: no plan has been built (ovc_resample_plan)");
  if (B < 0 || B > 65535 || max_count < 0 || max_count > 0x7fffffffLL)
    return fail(OVC_ERR_INVALID, "ovc_resample_rings: bad sizes B=%d max_count=%lld", B, (long long)max_count);
  if (in_rows < 1 || in_cap < 1 || out_rows < 1 || out_cap < 1 || in_cap > (INT64_MAX / 4) / in_rows ||
      out_cap > (INT64_MAX / 4) / out_rows)
    return fail(OVC_ERR_INVALID, "ovc_resample_rings: bad rings (in %d x %lld, out %d x %lld)", in_rows,
                (long long)in_cap, out_rows, (long long)out_cap);
  if (B == 0 || max_count == 0) return OVC_OK;
  if (!plan || !in || !in_row || !in_len || !m0 || !count || !out || !out_row || !out_off)
    return fail(OVC_ERR_INVALID, "null tensor argument");
  ON_DEVICE(c);
  const int tile = c->rs_ring_tile;
  const dim3 grid((unsigned)((max_count + tile - 1) / tile), B);
  const int threads = std::min(256, (tile + 31) / 32 * 32);
  resample_ring_kernel<<<grid, threads, c->rs_ring_smem, (cudaStream_t)stream>>>(
      c->d_rs_plans, (int)c->rs_plans.size(), plan, in, in_rows, in_cap, in_row, in_len, m0, count, out, out_rows,
      out_cap, out_row, out_off, max_count, tile);
  CK(cudaGetLastError());
  return OVC_OK;
}

int ovc_tts_info(const ovc_ctx* c, int32_t* out8) {
  if (!c || !out8) return fail(OVC_ERR_INVALID, "null argument");
  if (!c->finalized) return fail(OVC_ERR_STATE, "ovc_finalize_weights has not been called");
  const TtsLayers& L = c->tts;
  const int32_t v[8] = {L.ready ? 1 : 0, L.n_vocab, L.n_speakers, L.heads, L.n_layers, L.window, L.Fc, L.D};
  for (int i = 0; i < 8; ++i) out8[i] = v[i];
  return OVC_OK;
}

int ovc_tts_encode(ovc_ctx* c, const int64_t* tokens, const int64_t* x_lengths, const int64_t* sid, const float* noise_w,
                   uint64_t seed, float noise_scale_w, float length_scale, float sdp_ratio, int B, int T, int64_t* y_lengths,
                   float* w_ceil, float* logw, void* stream) {
  return ovc_tts_encode_items(c, tokens, x_lengths, sid, noise_w, seed, noise_scale_w, length_scale, sdp_ratio, B, T, y_lengths,
                              w_ceil, logw, stream, nullptr);
}

// Per-token speaker vectors condition the flow reverse and the generator per frame; both sections must read the target
// embedding (a zero_g checkpoint's generator does not, and its section has no per-frame columns).
static int check_tts_per_frame_cond(const ovc_ctx* c) {
  const int tc = c->precision >= 1, m = OVC_SE_FRAMES_TGT - 1;
  if (c->cond_pf_off[tc][m][2] < 0 || c->cond_pf_off[tc][m][3] < 0)
    return fail(OVC_ERR_INVALID, "per-token speaker vectors need a flow and a generator conditioned on g (zero_g is not)");
  return OVC_OK;
}

// the TTS encode with speaker ids (sid) or caller-supplied vectors (g, per row or with g_tokens per token)
static int tts_encode_any(ovc_ctx* c, const int64_t* tokens, const int64_t* x_lengths, const int64_t* sid, const float* g,
                          int g_tokens, const float* noise_w, uint64_t seed, float noise_scale_w, float length_scale,
                          float sdp_ratio, int B, int T, int64_t* y_lengths, float* w_ceil, float* logw, void* stream,
                          const ovc_item_params* items, const ovc_tts_fit* fit = nullptr) {
  if (!c) return fail(OVC_ERR_INVALID, "null context");
  if (!c->finalized) return fail(OVC_ERR_STATE, "ovc_finalize_weights has not been called");
  if (!c->tts.ready) return fail(OVC_ERR_STATE, "the checkpoint has no TTS members (enc_p / dp / sdp / emb_g): not a V1 base speaker");
  if (!tokens || !x_lengths || !(sid || g) || !y_lengths) return fail(OVC_ERR_INVALID, "null tensor argument");
  if (g_tokens != 0 && g_tokens != 1) return fail(OVC_ERR_INVALID, "g_tokens must be 0 or 1 (got %d)", g_tokens);
  if (g_tokens) TRY(check_tts_per_frame_cond(c));
  if (B < 1 || T < 1) return fail(OVC_ERR_INVALID, "B and T must be positive (got %d, %d)", B, T);
  if (B > 65535 || (long long)T * T > 2000000000LL / 256) return fail(OVC_ERR_INVALID, "B %d / T %d exceed the grid limits", B, T);
  if (!(length_scale > 0.f)) return fail(OVC_ERR_INVALID, "length_scale must be positive");
  TtsFit tf{};
  if (fit) {
    if (fit->G < 1 || fit->G > B) return fail(OVC_ERR_INVALID, "fit: G = %d groups for B = %d rows (1 <= G <= B)", fit->G, B);
    if (!fit->row0 || !fit->row1 || !fit->target_frames || !fit->length_scale) return fail(OVC_ERR_INVALID, "fit: null array");
    if (!(fit->scale_lo > 0.f && fit->scale_lo <= fit->scale_hi && std::isfinite(fit->scale_hi)))
      return fail(OVC_ERR_INVALID, "fit: scale range [%g, %g] must satisfy 0 < lo <= hi < inf", fit->scale_lo, fit->scale_hi);
    tf = TtsFit{(const long long*)fit->row0, (const long long*)fit->row1, (const long long*)fit->target_frames, fit->G,
                fit->scale_lo, fit->scale_hi, fit->length_scale};
  }
  ON_DEVICE(c);
  c->ev_used = c->prof ? c->ev_used : 0;
  return run_tts_encode(c, (const long long*)tokens, (const long long*)x_lengths, (const long long*)sid, g, g_tokens, noise_w,
                        seed, noise_scale_w, length_scale, sdp_ratio, B, T, (long long*)y_lengths, w_ceil, logw,
                        item_params(items), (cudaStream_t)stream, fit ? &tf : nullptr);
}

int ovc_tts_encode_items(ovc_ctx* c, const int64_t* tokens, const int64_t* x_lengths, const int64_t* sid, const float* noise_w,
                         uint64_t seed, float noise_scale_w, float length_scale, float sdp_ratio, int B, int T,
                         int64_t* y_lengths, float* w_ceil, float* logw, void* stream, const ovc_item_params* items) {
  if (!sid) return fail(OVC_ERR_INVALID, "null tensor argument");
  return tts_encode_any(c, tokens, x_lengths, sid, nullptr, 0, noise_w, seed, noise_scale_w, length_scale, sdp_ratio, B, T,
                        y_lengths, w_ceil, logw, stream, items);
}

int ovc_tts_encode_g(ovc_ctx* c, const int64_t* tokens, const int64_t* x_lengths, const float* g, int g_tokens,
                     const float* noise_w, uint64_t seed, float noise_scale_w, float length_scale, float sdp_ratio, int B, int T,
                     int64_t* y_lengths, float* w_ceil, float* logw, void* stream, const ovc_item_params* items) {
  if (!g) return fail(OVC_ERR_INVALID, "null tensor argument");
  return tts_encode_any(c, tokens, x_lengths, nullptr, g, g_tokens, noise_w, seed, noise_scale_w, length_scale, sdp_ratio, B,
                        T, y_lengths, w_ceil, logw, stream, items);
}

int ovc_tts_encode_fit(ovc_ctx* c, const int64_t* tokens, const int64_t* x_lengths, const int64_t* sid, const float* g,
                       int g_tokens, const float* noise_w, uint64_t seed, float noise_scale_w, float length_scale,
                       float sdp_ratio, int B, int T, int64_t* y_lengths, float* w_ceil, float* logw, void* stream,
                       const ovc_item_params* items, const ovc_tts_fit* fit) {
  if (!sid == !g) return fail(OVC_ERR_INVALID, "ovc_tts_encode_fit takes exactly one of sid and g");
  if (!fit) return fail(OVC_ERR_INVALID, "null fit");
  return tts_encode_any(c, tokens, x_lengths, sid, g, sid ? 0 : g_tokens, noise_w, seed, noise_scale_w, length_scale,
                        sdp_ratio, B, T, y_lengths, w_ceil, logw, stream, items, fit);
}

int ovc_tts_decode(ovc_ctx* c, const float* noise, uint64_t seed, float noise_scale, int B, int Ymax, int max_len, int ragged,
                   float* o, float* z, float* z_p, void* stream) {
  return ovc_tts_decode_items(c, noise, seed, noise_scale, B, Ymax, max_len, ragged, o, z, z_p, stream, nullptr);
}

int ovc_tts_decode_items(ovc_ctx* c, const float* noise, uint64_t seed, float noise_scale, int B, int Ymax, int max_len,
                         int ragged, float* o, float* z, float* z_p, void* stream, const ovc_item_params* items) {
  if (!c) return fail(OVC_ERR_INVALID, "null context");
  if (!c->finalized || !c->tts.ready) return fail(OVC_ERR_STATE, "no finalized TTS checkpoint");
  if (c->tts_B < 1) return fail(OVC_ERR_STATE, "ovc_tts_decode needs a preceding ovc_tts_encode");
  if (B != c->tts_B) return fail(OVC_ERR_INVALID, "B = %d but the pending ovc_tts_encode had B = %d", B, c->tts_B);
  if (!o) return fail(OVC_ERR_INVALID, "null tensor argument");
  if (Ymax < 1) return fail(OVC_ERR_INVALID, "Ymax must be positive");
  if ((long long)Ymax * 256 * 64 > 2000000000LL) return fail(OVC_ERR_INVALID, "Ymax %d too large for 32-bit indexing", Ymax);
  ON_DEVICE(c);
  c->ev_used = c->prof ? c->ev_used : 0;
  if (max_len < 0) return fail(OVC_ERR_INVALID, "max_len must be >= 0 (0 = no limit)");
  return run_tts_decode(c, noise, seed, noise_scale, B, Ymax, max_len, ragged, o, z, z_p, item_params(items),
                        (cudaStream_t)stream);
}

// g_tok: the caller's g is [B][gin][T] and the pending encode must have taken per-token vectors; else [B][gin] and it
// must not (either mismatch is OVC_ERR_STATE: a per-token encode never yields one vector per row)
static int tts_encode_state(ovc_ctx* c, float* stats, int32_t* cum, float* g, bool g_tok, void* stream) {
  if (!c) return fail(OVC_ERR_INVALID, "null context");
  if (!c->finalized || !c->tts.ready) return fail(OVC_ERR_STATE, "no finalized TTS checkpoint");
  if (c->tts_B < 1) return fail(OVC_ERR_STATE, "ovc_tts_encode_state needs a preceding ovc_tts_encode");
  if (c->tts_gtok != g_tok)
    return fail(OVC_ERR_STATE, g_tok ? "ovc_tts_encode_state_tokens needs a per-token encode (ovc_tts_encode_g, g_tokens = 1)"
                                     : "the pending encode took per-token speaker vectors: use ovc_tts_encode_state_tokens");
  if (!stats || !cum || !g) return fail(OVC_ERR_INVALID, "null tensor argument");
  ON_DEVICE(c);
  const int B = c->tts_B, T = c->tts_T;
  const TtsWs TW = tts_ws_layout(c, B, T, g_tok);
  cudaStream_t st = (cudaStream_t)stream;
  CK(cudaMemcpyAsync(stats, c->d_tts + TW.STATS, (size_t)B * T * 2 * c->tts.C * sizeof(float), cudaMemcpyDeviceToDevice, st));
  CK(cudaMemcpyAsync(cum, c->d_tts + TW.cum, (size_t)B * T * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  CK(cudaMemcpyAsync(g, c->d_tts + (g_tok ? TW.gtok : TW.g), (size_t)B * c->hp.gin_channels * (g_tok ? T : 1) * sizeof(float),
                     cudaMemcpyDeviceToDevice, st));
  return OVC_OK;
}

int ovc_tts_encode_state(ovc_ctx* c, float* stats, int32_t* cum, float* g, void* stream) {
  return tts_encode_state(c, stats, cum, g, false, stream);
}

int ovc_tts_encode_state_tokens(ovc_ctx* c, float* stats, int32_t* cum, float* g, void* stream) {
  return tts_encode_state(c, stats, cum, g, true, stream);
}

// g_tok: g [B][gin][T] -> d_g [N][gin][Tp] (tts_state_rows_g_kernel); else g [B][gin] -> d_g [N][gin]
static int tts_state_rows(ovc_ctx* c, const float* stats, const int* cum, const float* g, bool g_tok, const long long* y_len,
                          int B, int T, const int64_t* dst_row, int N, int Tp, float* d_stats, int32_t* d_cum, float* d_g,
                          int64_t* d_ylen, cudaStream_t st) {
  if (!dst_row || !d_stats || !d_cum || !d_g || !d_ylen) return fail(OVC_ERR_INVALID, "null tensor argument");
  if (N < 1 || Tp < T) return fail(OVC_ERR_INVALID, "pool of %d rows at pitch %d cannot take rows of %d tokens", N, Tp, T);
  const int gin = g_tok ? 0 : c->hp.gin_channels;   // per token: the g part is the second kernel's
  const long long per_row = (long long)Tp * 2 * c->tts.C + Tp + gin + 1;
  const int gx = (int)std::max(1LL, std::min((per_row + 255) / 256, std::max(1LL, 4LL * c->sm_count / B)));
  tts_state_rows_kernel<<<dim3(gx, std::min(B, 65535)), 256, 0, st>>>(stats, cum, g, y_len, B, T, 2 * c->tts.C, gin,
                                                     (const long long*)dst_row, N, Tp, d_stats, d_cum, d_g,
                                                     (long long*)d_ylen);
  CK(cudaGetLastError());
  if (g_tok) {
    const long long n = (long long)c->hp.gin_channels * Tp;
    const int gx2 = (int)std::max(1LL, std::min((n + 255) / 256, std::max(1LL, 4LL * c->sm_count / B)));
    tts_state_rows_g_kernel<<<dim3(gx2, std::min(B, 65535)), 256, 0, st>>>(g, B, T, c->hp.gin_channels,
                                                                           (const long long*)dst_row, N, Tp, d_g);
    CK(cudaGetLastError());
  }
  return OVC_OK;
}

static int tts_encode_state_rows(ovc_ctx* c, bool g_tok, const int64_t* dst_row, int N, int Tp, float* stats, int32_t* cum,
                                 float* g, int64_t* y_lengths, void* stream) {
  if (!c) return fail(OVC_ERR_INVALID, "null context");
  if (!c->finalized || !c->tts.ready) return fail(OVC_ERR_STATE, "no finalized TTS checkpoint");
  if (c->tts_B < 1) return fail(OVC_ERR_STATE, "ovc_tts_encode_state_rows needs a preceding ovc_tts_encode");
  if (c->tts_gtok != g_tok)
    return fail(OVC_ERR_STATE, g_tok ? "ovc_tts_encode_state_rows_tokens needs a per-token encode (ovc_tts_encode_g, g_tokens = 1)"
                                     : "the pending encode took per-token speaker vectors: use ovc_tts_encode_state_rows_tokens");
  ON_DEVICE(c);
  const int B = c->tts_B, T = c->tts_T;
  const TtsWs TW = tts_ws_layout(c, B, T, g_tok);
  return tts_state_rows(c, c->d_tts + TW.STATS, reinterpret_cast<const int*>(c->d_tts + TW.cum),
                        c->d_tts + (g_tok ? TW.gtok : TW.g), g_tok, reinterpret_cast<const long long*>(c->d_tts + TW.ylen),
                        B, T, dst_row, N, Tp, stats, cum, g, y_lengths, (cudaStream_t)stream);
}

int ovc_tts_encode_state_rows(ovc_ctx* c, const int64_t* dst_row, int N, int Tp, float* stats, int32_t* cum, float* g,
                              int64_t* y_lengths, void* stream) {
  return tts_encode_state_rows(c, false, dst_row, N, Tp, stats, cum, g, y_lengths, stream);
}

int ovc_tts_encode_state_rows_tokens(ovc_ctx* c, const int64_t* dst_row, int N, int Tp, float* stats, int32_t* cum, float* g,
                                     int64_t* y_lengths, void* stream) {
  return tts_encode_state_rows(c, true, dst_row, N, Tp, stats, cum, g, y_lengths, stream);
}

static int tts_state_rows_from(ovc_ctx* c, bool g_tok, const float* stats, const int32_t* cum, const float* g,
                               const int64_t* y_lengths, int B, int T, const int64_t* dst_row, int N, int Tp, float* d_stats,
                               int32_t* d_cum, float* d_g, int64_t* d_y_lengths, void* stream) {
  if (!c) return fail(OVC_ERR_INVALID, "null context");
  if (!c->finalized || !c->tts.ready) return fail(OVC_ERR_STATE, "no finalized TTS checkpoint");
  if (!stats || !cum || !g || !y_lengths) return fail(OVC_ERR_INVALID, "null tensor argument");
  if (B < 1 || T < 1) return fail(OVC_ERR_INVALID, "B and T must be positive (got %d, %d)", B, T);
  ON_DEVICE(c);
  return tts_state_rows(c, stats, cum, g, g_tok, (const long long*)y_lengths, B, T, dst_row, N, Tp, d_stats, d_cum, d_g,
                        d_y_lengths, (cudaStream_t)stream);
}

int ovc_tts_state_rows(ovc_ctx* c, const float* stats, const int32_t* cum, const float* g, const int64_t* y_lengths, int B,
                       int T, const int64_t* dst_row, int N, int Tp, float* d_stats, int32_t* d_cum, float* d_g,
                       int64_t* d_y_lengths, void* stream) {
  return tts_state_rows_from(c, false, stats, cum, g, y_lengths, B, T, dst_row, N, Tp, d_stats, d_cum, d_g, d_y_lengths, stream);
}

int ovc_tts_state_rows_tokens(ovc_ctx* c, const float* stats, const int32_t* cum, const float* g, const int64_t* y_lengths,
                              int B, int T, const int64_t* dst_row, int N, int Tp, float* d_stats, int32_t* d_cum, float* d_g,
                              int64_t* d_y_lengths, void* stream) {
  return tts_state_rows_from(c, true, stats, cum, g, y_lengths, B, T, dst_row, N, Tp, d_stats, d_cum, d_g, d_y_lengths, stream);
}

static int tts_decode_windows(ovc_ctx* c, const float* stats, const int32_t* cum, const float* g, bool g_tok,
                              const int64_t* y_lengths, int N, int T, const int64_t* row, const int64_t* frame0,
                              const int64_t* len, int W, int Wmax, const uint64_t* seed, const int64_t* stream,
                              const float* noise_scale, float* o, float* z_p, void* cuda_stream) {
  if (!c) return fail(OVC_ERR_INVALID, "null context");
  if (!c->finalized || !c->tts.ready) return fail(OVC_ERR_STATE, "no finalized TTS checkpoint");
  if (!stats || !cum || !g || !y_lengths || !row || !frame0 || !len || !seed || !stream || !noise_scale || !o)
    return fail(OVC_ERR_INVALID, "null tensor argument");
  if (N < 1 || T < 1 || W < 1 || Wmax < 1)
    return fail(OVC_ERR_INVALID, "N, T, W and Wmax must be positive (got %d, %d, %d, %d)", N, T, W, Wmax);
  if (W > 65535) return fail(OVC_ERR_INVALID, "W %d exceeds the grid limit", W);
  if (g_tok) TRY(check_tts_per_frame_cond(c));
  if ((long long)Wmax * 256 * 64 > 2000000000LL) return fail(OVC_ERR_INVALID, "Wmax %d too large for 32-bit indexing", Wmax);
  ON_DEVICE(c);
  c->ev_used = c->prof ? c->ev_used : 0;
  cudaStream_t st = (cudaStream_t)cuda_stream;
  TRY(ensure_ws(c, tts_windows_ws(c, W, Wmax, g_tok), W, Wmax, st));
  ItemParams it{};
  it.seed = (const unsigned long long*)seed; it.stream = (const long long*)stream; it.noise_scale = noise_scale;
  const TtsWindows win{(const long long*)row, (const long long*)frame0, (const long long*)len, N};
  std::vector<uintptr_t> key = {3, (uintptr_t)stats, (uintptr_t)cum, (uintptr_t)g, (uintptr_t)y_lengths, (uintptr_t)N,
                                (uintptr_t)T, (uintptr_t)row, (uintptr_t)frame0, (uintptr_t)len, (uintptr_t)W, (uintptr_t)Wmax,
                                (uintptr_t)o, (uintptr_t)z_p, option_bits(c), (uintptr_t)g_tok};
  append_item_key(key, it);
  return run_graphed(c, key, st, [&](cudaStream_t s) {
    return run_tts_decode_windows(c, stats, cum, g, g_tok, (const long long*)y_lengths, T, win, W, Wmax, it, o, z_p, s);
  });
}

int ovc_tts_decode_windows(ovc_ctx* c, const float* stats, const int32_t* cum, const float* g, const int64_t* y_lengths,
                           int N, int T, const int64_t* row, const int64_t* frame0, const int64_t* len, int W, int Wmax,
                           const uint64_t* seed, const int64_t* stream, const float* noise_scale, float* o, float* z_p,
                           void* cuda_stream) {
  return tts_decode_windows(c, stats, cum, g, false, y_lengths, N, T, row, frame0, len, W, Wmax, seed, stream, noise_scale, o,
                            z_p, cuda_stream);
}

int ovc_tts_decode_windows_tokens(ovc_ctx* c, const float* stats, const int32_t* cum, const float* g, const int64_t* y_lengths,
                                  int N, int T, const int64_t* row, const int64_t* frame0, const int64_t* len, int W, int Wmax,
                                  const uint64_t* seed, const int64_t* stream, const float* noise_scale, float* o, float* z_p,
                                  void* cuda_stream) {
  return tts_decode_windows(c, stats, cum, g, true, y_lengths, N, T, row, frame0, len, W, Wmax, seed, stream, noise_scale, o,
                            z_p, cuda_stream);
}

int ovc_philox_normals(uint64_t seed, int64_t stream, int64_t c0, int C, int64_t frame0, int T, float* out, void* cuda_stream) {
  if (!out || C < 1 || T < 1 || C > 65535) return fail(OVC_ERR_INVALID, "bad argument to ovc_philox_normals (C=%d, T=%d)", C, T);
  philox_normals_kernel<<<dim3((T + 127) / 128, C), 128, 0, (cudaStream_t)cuda_stream>>>(
      seed, (uint32_t)stream, (uint32_t)c0, (uint32_t)frame0, T, out);
  CK(cudaGetLastError());
  return OVC_OK;
}

static_assert(OVC_SPLICE_PCM16 == ovc_sp::PCM16 && OVC_SPLICE_SRC_WRAP == ovc_sp::SRC_WRAP, "ovc_splice flags");

int ovc_splice(const float* src, int64_t src_rows, int64_t src_pitch, float* dst, int64_t dst_rows, int64_t dst_cap,
               const int64_t* seg, int S, int flags, void* stream) {
  if (S < 0 || (S > 0 && !seg)) return fail(OVC_ERR_INVALID, "ovc_splice: bad segment table (S=%d)", S);
  if (!dst || dst_rows < 1 || dst_cap < 1)
    return fail(OVC_ERR_INVALID, "ovc_splice: bad destination (rows %lld, cap %lld)", (long long)dst_rows, (long long)dst_cap);
  if (src_rows < 0 || (src_rows > 0 && (!src || src_pitch < 1)))
    return fail(OVC_ERR_INVALID, "ovc_splice: bad source (rows %lld, pitch %lld)", (long long)src_rows, (long long)src_pitch);
  if (flags & ~(OVC_SPLICE_PCM16 | OVC_SPLICE_SRC_WRAP)) return fail(OVC_ERR_INVALID, "ovc_splice: unknown flags %d", flags);
  if (S == 0) return OVC_OK;
  const int gy = S < 65535 ? S : 65535;
  const int gx = std::max(1, std::min(1024, 2048 / gy));
  ovc_sp::splice_kernel<<<dim3(gx, gy), 256, 0, (cudaStream_t)stream>>>(src, src_rows, src_pitch, seg, S, dst, dst_rows,
                                                                         dst_cap, flags);
  CK(cudaGetLastError());
  return OVC_OK;
}

int ovc_set_precision(ovc_ctx* c, int mode) {
  if (!c) return fail(OVC_ERR_INVALID, "null context");
  if (mode < 0 || mode > 2) return fail(OVC_ERR_INVALID, "precision mode must be 0 (fp32 FFMA), 1 (3xFP16 tensor cores) or 2 (single-pass fp16)");
  c->precision = mode;
  return OVC_OK;
}

int ovc_set_option(ovc_ctx* c, int key, int value) {
  if (!c) return fail(OVC_ERR_INVALID, "null context");
  switch (key) {
    case OVC_OPT_TTS_SIMPLE: c->tts_simple = value != 0; return OVC_OK;
    case OVC_OPT_GRAPH: c->use_graph = value != 0; return OVC_OK;
    case OVC_OPT_PDL:
      if (value < 0 || value > 2) return fail(OVC_ERR_INVALID, "pdl must be 0, 1 or 2");
      c->use_pdl = value;
      return OVC_OK;
    case OVC_OPT_BRANCHES: c->use_branches = value != 0; return OVC_OK;
    case OVC_OPT_PAIR: c->use_pair = value != 0; return OVC_OK;
    case OVC_OPT_PAIR_OCC: c->use_pair_occ = value != 0; return OVC_OK;
    case OVC_OPT_STAGED_EPI: c->use_staged_epi = value != 0; return OVC_OK;
    default: return fail(OVC_ERR_INVALID, "unknown option %d", key);
  }
}

int ovc_last_launch_count(const ovc_ctx* c) { return c ? c->launches : 0; }

int ovc_graph_replays(const ovc_ctx* c) { return c ? c->graph_replays : 0; }

int ovc_profile_enable(ovc_ctx* c, int enable) {
  if (!c) return fail(OVC_ERR_INVALID, "null context");
  c->prof = enable != 0;
  c->ev_used = 0;
  c->ev_flops.clear();
  c->ev_bytes.clear();
  c->ev_variant.clear();
  c->ev_family.clear();
  c->ev_tag.clear();
  return OVC_OK;
}

int ovc_profile_read(ovc_ctx* c, double* ms, int64_t* launches, double* flops, double* bytes) {
  if (!c) return fail(OVC_ERR_INVALID, "null context");
  double tms = 0, tf = 0, tb = 0;
  int64_t n = 0;
  for (size_t i = 0; i + 1 < c->ev_used; i += 2) {
    if (!c->ev_family[i / 2]) continue;
    float m = 0;
    CK(cudaEventElapsedTime(&m, c->ev[i], c->ev[i + 1]));
    tms += m;
    tf += c->ev_flops[i / 2];
    tb += c->ev_bytes[i / 2];
    ++n;
  }
  if (ms) *ms = tms;
  if (launches) *launches = n;
  if (flops) *flops = tf;
  if (bytes) *bytes = tb;
  c->ev_used = 0;
  c->ev_flops.clear();
  c->ev_bytes.clear();
  c->ev_variant.clear();
  c->ev_family.clear();
  c->ev_tag.clear();
  return OVC_OK;
}

int ovc_profile_detail(ovc_ctx* c, int max, char* names /* max x 16 */, double* ms, double* flops, double* bytes, int* family) {
  if (!c) return fail(OVC_ERR_INVALID, "null context");
  int n = 0;
  for (size_t i = 0; i + 1 < c->ev_used && n < max; i += 2, ++n) {
    float m = 0;
    CK(cudaEventElapsedTime(&m, c->ev[i], c->ev[i + 1]));
    if (names) {
      const int tag = c->ev_tag[i / 2], v = c->ev_variant[i / 2];
      // the C = 128 pair is named T128P...: per-kernel tables group names by their first four characters
      if (tag && v == V_TCPAIR128) snprintf(names + 16 * n, 16, "T128Pk%dd%d", (tag >> 8) & 255, tag & 255);
      else if (tag && (v == V_TCPAIR64 || v == V_TCPAIR32)) snprintf(names + 16 * n, 16, "P%dk%dd%d", tag >> 16, (tag >> 8) & 255, tag & 255);
      else if (tag) snprintf(names + 16 * n, 16, "T%dc%dk%dd%d", v == V_TC128 ? 128 : v == V_TC64 ? 64 : 32, tag >> 16, (tag >> 8) & 255, tag & 255);
      else { strncpy(names + 16 * n, variant_name(v), 15); names[16 * n + 15] = 0; }
    }
    if (ms) ms[n] = m;
    if (flops) flops[n] = c->ev_flops[i / 2];
    if (bytes) bytes[n] = c->ev_bytes[i / 2];
    if (family) family[n] = c->ev_family[i / 2];
  }
  return n;
}

int ovc_debug_enable(ovc_ctx* c, int enable) {
  if (!c) return fail(OVC_ERR_INVALID, "null context");
  c->debug = enable != 0;
  return OVC_OK;
}

int ovc_debug_fetch(ovc_ctx* c, const char* name, float* host_out, size_t max_floats, int64_t* shape4) {
  if (!c || !name) return fail(OVC_ERR_INVALID, "null argument");
  auto it = c->taps.find(name);
  if (it == c->taps.end()) return fail(OVC_ERR_INVALID, "no debug tap named '%s' (enable debug and run a call first)", name);
  const DebugBuf& d = it->second;
  const size_t n = (size_t)d.shape[0] * d.shape[1] * d.shape[3];
  if (shape4) memcpy(shape4, d.shape, sizeof d.shape);
  if (host_out) {
    if (max_floats < n) return fail(OVC_ERR_INVALID, "buffer too small for tap '%s': need %zu floats", name, n);
    ON_DEVICE(c);
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(host_out, d.d, n * sizeof(float), cudaMemcpyDeviceToHost));
  }
  return OVC_OK;
}

}  // extern "C"
