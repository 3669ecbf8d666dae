// kc_pair.cu -- test harness of the fused ResBlock conv pair as the library runs it (tc_pair_fuses, ovc_tcpack.h):
// every square C = 32 / 64 / 128 pair, with resident or streamed weights.
//
// Compiled together with kc_tcconv.cu (included below), so libovc_kc_pair.so exports everything libovc_kc.so does and
// its single-conv launches share the pair's stream and checks.  Built by `make -C openvoice_b200/csrc kernelcheck` into
// tests/kernelcheck/libovc_kc_pair.so; the ctypes front end is tests/kernelcheck/kc_pair.py.
#include "kc_tcconv.cu"

extern "C" {

__attribute__((visibility("default"))) int kc_pair_fuses(int C1, int N1, int K1, int D1, int C2, int N2, int K2, int D2) {
  TcGeom a, b;
  a.Cin = C1; a.Ntot = N1; a.K = K1; a.DIL = D1; a.TN = tc_tile_n(N1, C1, K1, D1);
  b.Cin = C2; b.Ntot = N2; b.K = K2; b.DIL = D2; b.TN = tc_tile_n(N2, C2, K2, D2);
  return tc_pair_fuses(a, b) ? 1 : 0;
}

// one ResBlock conv pair the library fuses: w / bias conv 1 (dilation DIL), w2 / bias2 conv 2 (dilation 1),
// residual = x, y_ld = C
__attribute__((visibility("default"))) int kc_pair_fused(const KcConv* k) {
  if (setup()) return -1;
  static bool attr_done = false;
  if (!attr_done) {
    KC_CK(cudaFuncSetAttribute(tcconv_kernel<128, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TcnCfg<128, true>::SMEM_BYTES));
    attr_done = true;
  }
  const int TN = tc_tile_n(k->Ntot, k->Cin, k->K, k->DIL);
  if (check_common(k, TN)) return -1;
  TcGeom a1, a2;
  a1.Cin = k->Cin; a1.Ntot = k->Ntot; a1.K = k->K; a1.DIL = k->DIL; a1.TN = TN;
  a2 = a1; a2.DIL = 1; a2.TN = tc_tile_n(k->Ntot, k->Cin, k->K, 1);
  if (!tc_pair_fuses(a1, a2)) return fail("the pair C %d, k %d, dilation %d is not fused", k->Cin, k->K, k->DIL);
  if (!k->w2 || !k->bias2) return fail("pair: w2 and bias2 are required");
  if (k->epi != 0 || k->r || k->has_lens_x || k->y_ld != TN) return fail("pair: linear epilogue, residual = x, y_ld = C only");
  const TcGrid g = tc_pair_grid(k->tmax * k->mul, k->B, k->K, g_sms);
  const TcConvArgs a = to_args(k);
  const dim3 pg((unsigned)g.grid_x, 1, 1);
  const bool pdl = k->pdl != 0;
  if (TN == 128) KC_CK(launch_ex(tcconv_kernel<128, true>, pg, TcnCfg<128, true>::SMEM_BYTES, pdl, a, g.n_tt, g.total));
  else if (TN == 64) KC_CK(launch_ex(tcconv_kernel<64, true>, pg, TcnCfg<64, true>::SMEM_BYTES, pdl, a, g.n_tt, g.total));
  else KC_CK(launch_ex(tcconv_kernel<32, true>, pg, TcnCfg<32, true>::SMEM_BYTES, pdl, a, g.n_tt, g.total));
  KC_CK(cudaGetLastError());
  return 0;
}

}  // extern "C"
