"""ctypes front end of libovc_kc_f32.so (kc_f32.cu): the library's fp32 CUDA-core conv instantiations, its packing code
and the two conv_post kernels, one launch at a time, on torch tensors.  Activations are [B][C][pitch] fp32 CUDA tensors
(time fastest); every launch is refused on the host (RuntimeError) when the harness's checks refuse it."""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libovc_kc_f32.so")

P = C.c_void_p
EPI = {"LINEAR": 0, "GATE": 1, "RESSKIP": 2, "PROJ": 3, "COUPLE": 4, "UPS8": 5, "UPS2": 6}
F_ACCUM, F_FIRST = 1, 2


class KcF32(C.Structure):
    _fields_ = [(n, P) for n in ("x", "w", "bias", "y", "r", "s", "lens_in", "lens_out", "it_seed", "it_stream",
                                 "it_frame0", "it_tau")] + \
               [(n, C.c_longlong) for n in ("x_bs", "bias_bs", "y_bs", "r_bs", "s_bs", "x_n", "w_n", "bias_n", "y_n",
                                            "r_n", "s_n")] + \
               [("seed", C.c_ulonglong), ("cp_seed", C.c_ulonglong)] + \
               [(n, C.c_int) for n in ("variant", "x_pitch", "cin", "rows", "y_pitch", "r_pitch", "s_pitch", "tmax",
                                       "mul_in", "mul_out", "flags", "split", "t_len", "B", "lens_in_n", "lens_out_n",
                                       "items_n", "use_callp")] + \
               [(n, C.c_float) for n in ("slope", "scale", "tau", "sign", "cp_tau")]


class KcPost(C.Structure):
    _fields_ = [(n, P) for n in ("x", "w", "y", "lens")] + \
               [(n, C.c_longlong) for n in ("x_bs", "x_n", "w_n", "y_bs", "y_n")] + \
               [(n, C.c_int) for n in ("x_pitch", "y_len", "tmax", "mul", "B", "lens_n", "channels_last")]


class VariantInfo:
    def __init__(self, idx, name, f):
        self.idx, self.name = idx, name
        self.K, self.DIL, self.CO_T, self.T_T, self.CI_CH, epi, self.NG, self.XALIGN = f
        self.epi = {v: k for k, v in EPI.items()}[epi]


def _ptr(a):
    return a.ctypes.data_as(P)


def _dptr(t):
    return None if t is None else t.data_ptr()


class Harness:
    def __init__(self, path=LIB_PATH):
        if not os.path.exists(path):
            raise FileNotFoundError(f"{path} is missing: build it with `make -C openvoice_b200/csrc kernelcheck` "
                                    "(__graft_entry__.build() does)")
        L = self.lib = C.CDLL(path)
        L.kc_error.restype = C.c_char_p
        L.kc_variant.restype = C.c_char_p
        L.kc_variant.argtypes = [C.c_int, P]
        L.kc_packed_floats.restype = C.c_longlong
        L.kc_pack.argtypes = [C.c_int, P, C.c_int, C.c_int, C.c_int, P]
        L.kc_pack_ups.argtypes = [C.c_int, P] + [C.c_int] * 4 + [P]
        L.kc_corrupt.argtypes = [C.c_int, P] + [C.c_int] * 5
        L.kc_conv.argtypes = [C.POINTER(KcF32)]
        L.kc_conv_post.argtypes = [C.POINTER(KcPost)]
        self.variants = {}
        for i in range(L.kc_variant_count()):
            f = (C.c_int * 8)()
            name = L.kc_variant(i, C.cast(f, P)).decode()
            self.variants[name] = VariantInfo(i, name, tuple(f))

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError(self.lib.kc_error().decode())

    # ---- host only
    def paired_row(self, p, half):
        return self.lib.kc_paired_row(p, half)

    def ups_kidx(self, s, kk, row, tap):
        return self.lib.kc_ups_kidx(s, kk, row, tap)

    def tap_is_zero(self, s, k, r):
        return bool(self.lib.kc_tap_is_zero(s, k, r))

    def packed_floats(self, name, rows, cin):
        return self.lib.kc_packed_floats(self.variants[name].idx, rows, cin)

    def pack(self, name, w, paired=False):
        """w: [rows][cin][K] natural order -> packed float32 array ([row_tile][ci_pad][K][CO_T])."""
        w = np.ascontiguousarray(w, dtype=np.float32)
        rows, cin, K = w.shape
        assert K == self.variants[name].K, (name, K)
        out = np.zeros(self.packed_floats(name, rows, cin), np.float32)
        self._check(self.lib.kc_pack(self.variants[name].idx, _ptr(w), rows, cin, int(paired), _ptr(out)))
        return out

    def pack_ups(self, name, raw, s):
        """raw ConvTranspose1d weight [cin][cout][kk] of stride s -> the packed polyphase conv."""
        raw = np.ascontiguousarray(raw, dtype=np.float32)
        cin, cout, kk = raw.shape
        out = np.zeros(self.packed_floats(name, cout * s, cin), np.float32)
        self._check(self.lib.kc_pack_ups(self.variants[name].idx, _ptr(raw), cin, cout, kk, s, _ptr(out)))
        return out

    def corrupt(self, name, packed, rows, cin, kind, i=0, j=0):
        """kind 'swap' swaps taps i and j; 'chunk' zeroes ci-chunk i of row tile j.  Returns a corrupted copy."""
        p = packed.copy()
        self._check(self.lib.kc_corrupt(self.variants[name].idx, _ptr(p), rows, cin, {"swap": 0, "chunk": 1}[kind], i, j))
        return p

    # ---- device
    def setup(self):
        self._check(self.lib.kc_setup())

    def conv(self, name, x, w, bias, y, *, rows, cin=None, tmax, mul_in=1, mul_out=1, t_len=None, lens_in=None,
             lens_out=None, r=None, s=None, bias_bs=0, slope=1.0, scale=1.0, tau=0.0, sign=1.0, flags=0, split=0, seed=0,
             callp=None, sync=True):
        """One conv1d_f32 launch of variant `name`.  x [B][cin'][x_pitch] (or any flat tensor with explicit strides
        given as (tensor, bs, pitch)), w a packed CUDA tensor, bias flat, y / r / s like x.  callp: None, or
        dict(seed=, tau=, items=dict(seed=, stream=, frame0=, tau=) of [B] CUDA tensors or None)."""
        import torch
        a = KcF32()
        a.variant = self.variants[name].idx

        def buf(t):
            if t is None:
                return None, 0, 0, 0
            if isinstance(t, tuple):
                t, bs, pitch = t
            else:
                bs, pitch = t.shape[1] * t.shape[2], t.shape[2]
            assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()
            return t.data_ptr(), bs, pitch, t.numel()

        a.x, a.x_bs, a.x_pitch, a.x_n = buf(x)
        a.y, a.y_bs, a.y_pitch, a.y_n = buf(y)
        a.r, a.r_bs, a.r_pitch, a.r_n = buf(r)
        a.s, a.s_bs, a.s_pitch, a.s_n = buf(s)
        B = (x[0] if isinstance(x, tuple) else x).shape[0]
        a.cin = cin if cin is not None else (x[0] if isinstance(x, tuple) else x).shape[1]
        assert w.is_cuda and w.dtype == torch.float32 and bias.is_cuda and bias.dtype == torch.float32
        a.w, a.w_n, a.bias, a.bias_n, a.bias_bs = w.data_ptr(), w.numel(), bias.data_ptr(), bias.numel(), bias_bs
        for nm, ln in (("lens_in", lens_in), ("lens_out", lens_out)):
            if ln is not None:
                assert ln.is_cuda and ln.dtype == torch.int64
                setattr(a, nm, ln.data_ptr())
                setattr(a, nm + "_n", ln.numel())
        if callp is not None:
            a.use_callp, a.cp_seed, a.cp_tau = 1, callp["seed"], callp["tau"]
            items = callp.get("items") or {}
            n = []
            for k, dt in (("seed", torch.int64), ("stream", torch.int64), ("frame0", torch.int64), ("tau", torch.float32)):
                t = items.get(k)
                if t is not None:
                    assert t.is_cuda and t.dtype == dt
                    setattr(a, "it_" + k, t.data_ptr())
                    n.append(t.numel())
            a.items_n = min(n) if n else 0
        a.rows, a.tmax, a.mul_in, a.mul_out = rows, tmax, mul_in, mul_out
        a.t_len = t_len if t_len is not None else tmax * mul_out
        a.B, a.flags, a.split, a.seed = B, flags, split, seed
        a.slope, a.scale, a.tau, a.sign = slope, scale, tau, sign
        torch.cuda.current_stream().synchronize()   # inputs written by torch are in place
        self._check(self.lib.kc_conv(C.byref(a)))
        if sync:
            self.sync()

    def conv_post(self, x, w, y, *, y_len, tmax, mul, lens=None, channels_last=False, x_pitch=None, sync=True):
        """conv_post_kernel<32> (x [B][32][pitch]) or conv_post_cl_kernel<32> (x [B][T][32]); y [B][y_pitch]."""
        import torch
        for t in (x, w, y):
            assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()
        a = KcPost()
        a.x, a.w, a.y = x.data_ptr(), w.data_ptr(), y.data_ptr()
        a.x_bs, a.x_n, a.w_n = x[0].numel(), x.numel(), w.numel()
        a.y_bs, a.y_n = y.shape[1], y.numel()
        a.x_pitch = 0 if channels_last else (x_pitch or x.shape[2])
        a.y_len, a.tmax, a.mul, a.B, a.channels_last = y_len, tmax, mul, x.shape[0], int(channels_last)
        if lens is not None:
            assert lens.is_cuda and lens.dtype == torch.int64
            a.lens, a.lens_n = lens.data_ptr(), lens.numel()
        torch.cuda.current_stream().synchronize()
        self._check(self.lib.kc_conv_post(C.byref(a)))
        if sync:
            self.sync()

    def sync(self):
        self._check(self.lib.kc_sync())
