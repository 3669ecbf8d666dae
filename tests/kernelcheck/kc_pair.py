"""ctypes front end of libovc_kc_pair.so (kc_pair.cu): the kc.py harness plus the pair fusion rule of the library
(tc_pair_fuses) and a pair launch that accepts every pair it fuses, resident or streamed weights."""
import ctypes as C
import importlib.util
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libovc_kc_pair.so")

_spec = importlib.util.spec_from_file_location("kc", os.path.join(HERE, "kc.py"))
kc = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(kc)


class PairHarness(kc.Harness):
    def __init__(self, path=LIB_PATH):
        super().__init__(path)
        self.lib.kc_pair_fused.argtypes = [C.POINTER(kc.KcConv)]

    def pair_fuses(self, C1, K1, D1, C2=None, K2=None, D2=1, N1=None, N2=None):
        """The pairs the library runs as one kernel (pair() launches exactly these)."""
        C2 = C1 if C2 is None else C2
        K2 = K1 if K2 is None else K2
        return bool(self.lib.kc_pair_fuses(C1, C1 if N1 is None else N1, K1, D1, C2, C2 if N2 is None else N2, K2, D2))

    def pair(self, x, w, bias, w2, bias2, y, sync=True, **kw):
        """One fused ResBlock conv pair: y = (c2(lrelu(c1(lrelu(x)) + bias)) + bias2 + x [+ y_old]) * scale."""
        import torch
        a = self._args(x, w, bias, y, w2=w2, bias2=bias2, Ntot=x.shape[2], **kw)
        torch.cuda.current_stream().synchronize()   # inputs written by torch are in place
        self._check(self.lib.kc_pair_fused(C.byref(a)))
        if sync:
            self.sync()
