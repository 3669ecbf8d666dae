// kc_pair_occ.cu -- test harness of the conv pairs at two CTAs per SM (tc_pair_occ, ovc_tcpack.h): the config the
// library picks per pair, the device's occupancy of each two-CTA kernel, and a pair launch at one or two CTAs per SM.
//
// Compiled together with kc_pair.cu (included below), so libovc_kc_pair_occ.so exports everything libovc_kc_pair.so
// does.  Built by `make -C openvoice_b200/csrc kernelcheck` into tests/kernelcheck/libovc_kc_pair_occ.so; the ctypes
// front end is tests/kernelcheck/kc_pair_occ.py.
#include "kc_pair.cu"

extern "C" {

// host only: the config tc_pair_occ picks for the square pair (C, k, dilation) -> out[0..4] = CTAs per SM, operand
// buffers, ring slots, shared memory bytes per CTA, resident (both convs' weights fit the ring); -1 if not fused
__attribute__((visibility("default"))) int kc_pair_occ(int C, int K, int D, long long* out) {
  TcGeom a, b;
  a.Cin = C; a.Ntot = C; a.K = K; a.DIL = D; a.TN = tc_tile_n(C, C, K, D);
  b = a; b.DIL = 1; b.TN = tc_tile_n(C, C, K, 1);
  if (!tc_pair_fuses(a, b)) return fail("the pair C %d, k %d, dilation %d is not fused", C, K, D);
  const TcPairOcc o = tc_pair_occ(a, b);
  const int ring = tc_pair_ring(a.TN, o.occ, o.nabuf);
  out[0] = o.occ; out[1] = o.nabuf; out[2] = ring;
  out[3] = (long long)tc_pair_smem(a.TN, o.nabuf, ring);
  out[4] = 2 * (C / 16) * K <= ring;
  return 0;
}

// cudaOccupancyMaxActiveBlocksPerMultiprocessor of the pair kernel (C, occ, nabuf) at its shared memory
__attribute__((visibility("default"))) int kc_pair_occupancy(int C, int occ, int nabuf) {
  if (setup()) return -1;
  const TcPairKernel pk = tc_pair_kernel(C, TcPairOcc{occ, nabuf});
  if (!pk.fn) return fail("no pair kernel C %d, occ %d, nabuf %d", C, occ, nabuf);
  KC_CK(cudaFuncSetAttribute(pk.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pk.smem));
  int blocks = 0;
  KC_CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, pk.fn, TCN_THREADS, pk.smem));
  return blocks;
}

// kc_pair_fused at a chosen occupancy: occ = 1 one CTA per SM (the kernel kc_pair_fused runs), occ = 2 the two-CTA
// config tc_pair_occ picks for the pair (an error where it picks one CTA), on a grid of occ CTAs per SM
__attribute__((visibility("default"))) int kc_pair_fused_occ(const KcConv* k, int occ) {
  if (setup()) return -1;
  const int TN = tc_tile_n(k->Ntot, k->Cin, k->K, k->DIL);
  if (check_common(k, TN)) return -1;
  TcGeom a1, a2;
  a1.Cin = k->Cin; a1.Ntot = k->Ntot; a1.K = k->K; a1.DIL = k->DIL; a1.TN = TN;
  a2 = a1; a2.DIL = 1; a2.TN = tc_tile_n(k->Ntot, k->Cin, k->K, 1);
  if (!tc_pair_fuses(a1, a2)) return fail("the pair C %d, k %d, dilation %d is not fused", k->Cin, k->K, k->DIL);
  if (!k->w2 || !k->bias2) return fail("pair: w2 and bias2 are required");
  if (k->epi != 0 || k->r || k->has_lens_x || k->y_ld != TN) return fail("pair: linear epilogue, residual = x, y_ld = C only");
  TcPairOcc o;
  if (occ == 2) {
    o = tc_pair_occ(a1, a2);
    if (o.occ != 2) return fail("tc_pair_occ runs the pair C %d, k %d one CTA per SM", k->Cin, k->K);
  } else if (occ != 1) {
    return fail("occ must be 1 or 2, not %d", occ);
  }
  const TcPairKernel pk = tc_pair_kernel(TN, o);
  if (!pk.fn) return fail("no pair kernel C %d, occ %d, nabuf %d", TN, o.occ, o.nabuf);
  KC_CK(cudaFuncSetAttribute(pk.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pk.smem));
  const TcGrid g = tc_pair_grid(k->tmax * k->mul, k->B, k->K, g_sms, o.occ);
  const TcConvArgs a = to_args(k);
  KC_CK(launch_ex(pk.fn, dim3((unsigned)g.grid_x, 1, 1), pk.smem, k->pdl != 0, a, g.n_tt, g.total));
  KC_CK(cudaGetLastError());
  return 0;
}

}  // extern "C"
