// kc_staged.cu -- test harness of the staged-epilogue kernels (tcconv_kernel<128, PAIR, 1, 2, true>, OVC_OPT_STAGED_EPI):
// a single conv or a fused pair with the staged or the unstaged epilogue, the rule the library stages by
// (tc_stage_pays), and the staged configs' budgets.
//
// Compiled together with kc_pair.cu (included below), so libovc_kc_staged.so exports everything libovc_kc_pair.so does
// and its launches share that harness's stream and checks.  Built by `make -C openvoice_b200/csrc kernelcheck` into
// tests/kernelcheck/libovc_kc_staged.so; tests/test_gpu_staged_epilogue.py is its ctypes front end.
#include "kc_pair.cu"

namespace {

// one launch of a tcconv_kernel instantiation at its own block size and shared memory
int launch_kernel(const TcKernel& k, const KcConv* kc, const TcGrid& g) {
  if (!k.fn) return fail("no kernel for this configuration");
  KC_CK(cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k.smem));
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)g.grid_x, g.ncol, 1);
  cfg.blockDim = dim3((unsigned)k.threads, 1, 1);
  cfg.dynamicSmemBytes = k.smem;
  cfg.stream = g_stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = kc->pdl ? 1 : 0;
  KC_CK(cudaLaunchKernelEx(&cfg, k.fn, to_args(kc), g.n_tt, g.total));
  KC_CK(cudaGetLastError());
  return 0;
}

}  // namespace

extern "C" {

// host only: whether the library stages a TN = 128 conv / C = 128 pair of k taps in this pass mode
__attribute__((visibility("default"))) int kc_stage_pays(int K, int passes) { return tc_stage_pays(K, passes) ? 1 : 0; }

// host only: the staged configs (TcnCfg<128, pair, 1, 2, true>) -> out[0..7] = threads, shared memory bytes, staging
// tile bytes, its own buffer's bytes (0: it overlays the conv-2 operand), conv-2 operand bytes, producer / MMA / store
// registers per thread
__attribute__((visibility("default"))) void kc_staged_cfg(int pair, long long* out) {
  auto put = [&](auto cfg) {
    using Cfg = decltype(cfg);
    const long long v[8] = {Cfg::THREADS, (long long)Cfg::SMEM_BYTES, Cfg::STAGE_BYTES, Cfg::SBUF_BYTES, Cfg::A2_BYTES,
                            Cfg::PROD_REGS, Cfg::MMA_REGS, Cfg::STORE_REGS};
    for (int i = 0; i < 8; ++i) out[i] = v[i];
  };
  if (pair) put(TcnCfg<128, true, 1, 2, true>());
  else put(TcnCfg<128, false, 1, 2, true>());
}

// one conv (PAIR = false), checked like kc_conv; staged: TN = 128 runs the staged epilogue, 0 the unstaged kernel
__attribute__((visibility("default"))) int kc_conv_staged(const KcConv* k, int staged) {
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
  return launch_kernel(tc_conv_kernel(TN, staged != 0), k, g);
}

// one fused ResBlock conv pair, checked like kc_pair_fused; staged: C = 128 runs the staged epilogue
__attribute__((visibility("default"))) int kc_pair_fused_staged(const KcConv* k, int staged) {
  if (setup()) return -1;
  const int TN = tc_tile_n(k->Ntot, k->Cin, k->K, k->DIL);
  if (check_common(k, TN)) return -1;
  TcGeom a1, a2;
  a1.Cin = k->Cin; a1.Ntot = k->Ntot; a1.K = k->K; a1.DIL = k->DIL; a1.TN = TN;
  a2 = a1; a2.DIL = 1; a2.TN = tc_tile_n(k->Ntot, k->Cin, k->K, 1);
  if (!tc_pair_fuses(a1, a2)) return fail("the pair C %d, k %d, dilation %d is not fused", k->Cin, k->K, k->DIL);
  if (!k->w2 || !k->bias2) return fail("pair: w2 and bias2 are required");
  if (k->epi != 0 || k->r || k->has_lens_x || k->y_ld != TN) return fail("pair: linear epilogue, residual = x, y_ld = C only");
  const TcGrid g = tc_pair_grid(k->tmax * k->mul, k->B, k->K, g_sms);
  return launch_kernel(tc_pair_kernel(TN, TcPairOcc(), staged != 0), k, g);
}

}  // extern "C"
