"""ctypes front end of libovc_kc_pair_occ.so (kc_pair_occ.cu): the kc_pair.py harness plus the two-CTA-per-SM conv-pair
configs of the library (tc_pair_occ), the occupancy query and a pair launch at a chosen occupancy."""
import ctypes as C
import importlib.util
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libovc_kc_pair_occ.so")

_spec = importlib.util.spec_from_file_location("kc_pair", os.path.join(HERE, "kc_pair.py"))
kc_pair = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(kc_pair)
kc = kc_pair.kc


class PairOccHarness(kc_pair.PairHarness):
    def __init__(self, path=LIB_PATH):
        super().__init__(path)
        self.lib.kc_pair_fused_occ.argtypes = [C.POINTER(kc.KcConv), C.c_int]
        self.lib.kc_pair_occ.argtypes = [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_longlong)]
        self.lib.kc_pair_occupancy.argtypes = [C.c_int, C.c_int, C.c_int]

    def pair_occ(self, C_, K, D):
        """The config tc_pair_occ picks for a fused square pair: dict(occ, nabuf, ring, smem, resident)."""
        out = (C.c_longlong * 5)()
        self._check(self.lib.kc_pair_occ(C_, K, D, out))
        return dict(occ=out[0], nabuf=out[1], ring=out[2], smem=out[3], resident=bool(out[4]))

    def pair_occupancy(self, C_, occ, nabuf):
        """CTAs per SM the device fits of the pair kernel (C, occ, nabuf) (cudaOccupancyMaxActiveBlocksPerMultiprocessor)."""
        n = self.lib.kc_pair_occupancy(C_, occ, nabuf)
        self._check(n if n < 0 else 0)
        return n

    def pair_at(self, occ, x, w, bias, w2, bias2, y, sync=True, **kw):
        """pair() at occ CTAs per SM: 1 the one-CTA kernel, 2 the config tc_pair_occ picks."""
        import torch
        a = self._args(x, w, bias, y, w2=w2, bias2=bias2, Ntot=x.shape[2], **kw)
        torch.cuda.current_stream().synchronize()
        self._check(self.lib.kc_pair_fused_occ(C.byref(a), occ))
        if sync:
            self.sync()
