"""ctypes front end of libovc_kc.so (kc_tcconv.cu): the library's tensor-core conv kernel and packing code, one launch
at a time, on torch tensors.  Activations are channels-last [B][L][C] fp32 CUDA tensors; every launch is refused on
the host (RuntimeError) when the fit rules refuse it or a buffer is too small for what the kernel would touch."""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libovc_kc.so")

P = C.c_void_p


class KcConv(C.Structure):
    _fields_ = [(n, P) for n in ("x", "w", "bias", "y", "r", "s", "lens", "lens_x", "w2", "bias2")] + \
               [(n, C.c_longlong) for n in ("x_bs", "bias_bs", "y_bs", "s_bs")] + \
               [(n, C.c_int) for n in ("y_ld", "epi", "split", "first", "tmax", "mul", "has_lens_x", "Cin", "Ntot", "K", "DIL",
                                       "accumulate", "passes", "grid_div", "pdl", "B")] + \
               [("slope", C.c_float), ("scale", C.c_float)]


def _ptr(a):
    return a.ctypes.data_as(P)


class Harness:
    def __init__(self, path=LIB_PATH):
        if not os.path.exists(path):
            raise FileNotFoundError(f"{path} is missing: build it with `make -C openvoice_b200/csrc kernelcheck` "
                                    "(__graft_entry__.build() does)")
        L = self.lib = C.CDLL(path)
        L.kc_error.restype = C.c_char_p
        L.kc_packed_halfs.restype = C.c_longlong
        L.kc_pack.argtypes = [P, C.c_int, C.c_int, C.c_int, C.c_int, P]
        L.kc_ups_weights.argtypes = [P, C.c_int, C.c_int, C.c_int, C.c_int, P]
        L.kc_grid.argtypes = [C.c_int] * 8 + [P]
        L.kc_corrupt.argtypes = [P] + [C.c_int] * 7
        L.kc_conv.argtypes = [C.POINTER(KcConv)]
        L.kc_pair.argtypes = [C.POINTER(KcConv)]

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError(self.lib.kc_error().decode())

    # ---- host only
    def tile_n(self, Ntot, Cin, K, DIL=1):
        return self.lib.kc_tile_n(Ntot, Cin, K, DIL)

    def ring_slots(self, TN, pair=False):
        return self.lib.kc_ring_slots(TN, int(pair))

    def pair_fits(self, C1, K1, D1, C2=None, K2=None, D2=1, N1=None, N2=None):
        C2 = C1 if C2 is None else C2
        K2 = K1 if K2 is None else K2
        return bool(self.lib.kc_pair_fits(C1, C1 if N1 is None else N1, K1, D1, C2, C2 if N2 is None else N2, K2, D2))

    def grid(self, t_len, B, Ntot, TN, sm_count, grid_div=1, pair=False, K=1):
        out = (C.c_int * 4)()
        self.lib.kc_grid(t_len, B, Ntot, TN, sm_count, grid_div, int(pair), K, C.cast(out, P))
        return tuple(out)

    def pack(self, w, DIL=1):
        """w: [Ntot][Cin][K] -> (packed uint16 array, TN); ValueError when the conv does not fit."""
        w = np.ascontiguousarray(w, dtype=np.float32)
        N, Cin, K = w.shape
        TN = self.tile_n(N, Cin, K, DIL)
        if not TN:
            raise ValueError(f"conv {Cin} -> {N} (k {K}, dilation {DIL}) does not fit the tensor-core kernel")
        out = np.zeros(self.lib.kc_packed_halfs(N, Cin, K, TN), np.uint16)
        assert self.lib.kc_pack(_ptr(w), N, Cin, K, DIL, _ptr(out)) == TN
        return out, TN

    def ups_weights(self, raw, s):
        """ConvTranspose1d weight [cin][cout][kk] of stride s -> unpacked polyphase weight [s*cout][cin][3]."""
        raw = np.ascontiguousarray(raw, dtype=np.float32)
        cin, cout, kk = raw.shape
        out = np.empty((s * cout, cin, 3), np.float32)
        self.lib.kc_ups_weights(_ptr(raw), cin, cout, kk, s, _ptr(out))
        return out

    def corrupt(self, packed, Ntot, Cin, K, TN, kind, i=0, j=0):
        """kind 'lo' zeroes every lo row, 'swap' swaps the slots of taps i and j, 'slot' zeroes 16-channel slot i of
        column tile j.  Returns a corrupted copy."""
        p = packed.copy()
        self._check(self.lib.kc_corrupt(_ptr(p), Ntot, Cin, K, TN, {"lo": 0, "swap": 1, "slot": 2}[kind], i, j))
        return p

    # ---- device
    def sm_count(self):
        n = self.lib.kc_sm_count()
        if n < 0:
            raise RuntimeError(self.lib.kc_error().decode())
        return n

    @staticmethod
    def upload(packed):
        import torch
        return torch.from_numpy(packed.view(np.int16)).cuda()

    def _args(self, x, w, bias, y, *, Ntot, K, DIL=1, tmax, mul=1, lens=None, lens_x=None, r=None, s=None, bias_bs=0,
              epi=0, split=0, first=0, slope=1.0, scale=1.0, accumulate=False, passes=3, grid_div=1, pdl=False, w2=None,
              bias2=None):
        import torch
        for name, t in (("x", x), ("bias", bias), ("y", y), ("r", r), ("s", s), ("bias2", bias2)):
            if t is not None:
                assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous(), name
        B, L, Cin = x.shape
        rows = tmax * mul
        assert L >= rows and y.shape[0] == B and y.shape[1] >= rows, "buffers shorter than tmax * mul"
        y_ld = y.shape[2]
        need_y = {0: Ntot, 1: Ntot // 2, 2: max(split, Ntot - split)}[epi]
        assert y_ld >= need_y, "output row narrower than the epilogue writes"
        if r is not None:
            assert r.shape == y.shape
        if s is not None:
            assert s.shape == y.shape
        assert bias.numel() >= (B - 1) * bias_bs + Ntot
        TN = self.tile_n(Ntot, Cin, K, DIL)
        if TN:
            assert w.numel() >= self.lib.kc_packed_halfs(Ntot, Cin, K, TN)
        for ln in (lens, lens_x):
            if ln is not None:
                assert ln.is_cuda and ln.dtype == torch.int64 and ln.numel() >= B
        a = KcConv()
        a.x, a.w, a.bias, a.y = x.data_ptr(), w.data_ptr(), bias.data_ptr(), y.data_ptr()
        a.r = r.data_ptr() if r is not None else None
        a.s = s.data_ptr() if s is not None else None
        a.lens = lens.data_ptr() if lens is not None else None
        a.lens_x = lens_x.data_ptr() if lens_x is not None else None
        a.w2 = w2.data_ptr() if w2 is not None else None
        a.bias2 = bias2.data_ptr() if bias2 is not None else None
        a.x_bs, a.bias_bs, a.y_bs, a.s_bs = L * Cin, bias_bs, y.shape[1] * y_ld, y.shape[1] * y_ld
        a.y_ld, a.epi, a.split, a.first = y_ld, epi, split, int(first)
        a.tmax, a.mul, a.has_lens_x = tmax, mul, int(lens_x is not None)
        a.Cin, a.Ntot, a.K, a.DIL = Cin, Ntot, K, DIL
        a.accumulate, a.passes, a.grid_div, a.pdl, a.B = int(accumulate), passes, grid_div, int(pdl), B
        a.slope, a.scale = slope, scale
        return a

    def conv(self, x, w, bias, y, sync=True, **kw):
        """One tcconv launch.  x [B][L][Cin], y [B][L][y_ld] (and r, s like y); w packed (upload()); bias [Ntot] or
        per utterance with bias_bs; lens / lens_x int64 [B]."""
        import torch
        a = self._args(x, w, bias, y, **kw)
        torch.cuda.current_stream().synchronize()   # inputs written by torch are in place
        self._check(self.lib.kc_conv(C.byref(a)))
        if sync:
            self.sync()

    def pair(self, x, w, bias, w2, bias2, y, sync=True, **kw):
        """One ResBlock conv pair: y = (c2(lrelu(c1(lrelu(x)) + bias)) + bias2 + x [+ y_old]) * scale."""
        import torch
        a = self._args(x, w, bias, y, w2=w2, bias2=bias2, Ntot=x.shape[2], **kw)
        torch.cuda.current_stream().synchronize()   # inputs written by torch are in place
        self._check(self.lib.kc_pair(C.byref(a)))
        if sync:
            self.sync()

    def sync(self):
        self._check(self.lib.kc_sync())
