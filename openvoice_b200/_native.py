"""ctypes binding of libovc_b200.so (C ABI: include/ovc.h).

PyTorch is used for device memory and streams only; every tensor crosses the boundary as a raw
device pointer.  If the library is missing or no sm_90 GPU is present this module raises --
there is no fallback path of any kind.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, Iterable, Optional, Tuple

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libovc_b200.so")

ABI_VERSION = 18
EXPORTS = (
    "ovc_abi_version", "ovc_last_error", "ovc_create", "ovc_destroy", "ovc_load_tensor",
    "ovc_finalize_weights", "ovc_workspace_floats", "ovc_voice_conversion", "ovc_last_launch_count",
    "ovc_profile_enable", "ovc_profile_read", "ovc_profile_detail", "ovc_debug_enable", "ovc_debug_fetch",
    "ovc_spectrogram", "ovc_convert_waveform", "ovc_set_precision", "ovc_reference_encoder",
    "ovc_tts_info", "ovc_tts_encode", "ovc_tts_decode", "ovc_set_option", "ovc_graph_replays",
    "ovc_reference_encoder_ragged", "ovc_resample", "ovc_resample_span", "ovc_voice_conversion_items",
    "ovc_convert_waveform_items", "ovc_tts_encode_items", "ovc_tts_decode_items", "ovc_philox_normals",
    "ovc_tts_encode_state", "ovc_tts_decode_windows", "ovc_spectrogram_ring", "ovc_splice",
    "ovc_tts_encode_state_rows", "ovc_tts_state_rows", "ovc_resample_plan", "ovc_resample_rings",
    "ovc_voice_conversion_frames", "ovc_convert_waveform_frames", "ovc_tone_track_expand",
    "ovc_tts_encode_g", "ovc_tts_encode_state_tokens", "ovc_tts_decode_windows_tokens", "ovc_tts_encode_state_rows_tokens",
    "ovc_tts_state_rows_tokens", "ovc_reference_encoder_stream", "ovc_reference_encoder_stream_state_floats",
    "ovc_generate_frames", "ovc_tts_encode_fit",
)

STREAM_OPEN = 2 ** 63 - 1   # ovc_resample / ovc_spectrogram_ring length of a stream that has not ended
SPLICE_PCM16 = 1            # ovc_splice flag: the 16-bit PCM round trip of every copied value
SPLICE_SRC_WRAP = 2         # ovc_splice flag: source rows are rings, src_off + i wraps mod the source pitch
SE_FRAMES_SRC, SE_FRAMES_TGT = 1, 2   # ovc_*_frames: the side's embedding is given per frame


def se_arg(g, B: int, gin: int, T: int, what: str):
    """(float32 contiguous [B, gin] or [B, gin, T] tensor, per_frame) of a speaker embedding: B * gin values (any
    shape: one embedding per item) or a [B, gin, T] tensor (one per frame, T > 1).  Anything else raises ValueError,
    so an embedding is never read as some other layout.  A 3-D tensor with gin rows and more than one column is a
    per-frame embedding and must be exactly [B, gin, T]; it is never reinterpreted as per-item values."""
    if g.dim() == 3 and g.shape[-2] == gin and g.shape[-1] > 1:
        if T > 1 and tuple(g.shape) == (B, gin, T):
            return g.contiguous().float(), True
    elif g.numel() == B * gin:
        return g.reshape(B, gin).contiguous().float(), False
    raise ValueError(f"{what} has shape {tuple(g.shape)}: expected {B} x {gin} values (one embedding per item) or "
                     f"[{B}, {gin}, {T}] (one per frame)")


class OvcHParams(C.Structure):
    """struct ovc_hparams of include/ovc.h."""
    _fields_ = [
        ("spec_channels", C.c_int32), ("inter_channels", C.c_int32), ("hidden_channels", C.c_int32),
        ("gin_channels", C.c_int32), ("resblock", C.c_int32), ("n_resblock_kernels", C.c_int32),
        ("resblock_kernel_sizes", C.c_int32 * 4), ("resblock_dilations", (C.c_int32 * 3) * 4),
        ("n_upsamples", C.c_int32), ("upsample_rates", C.c_int32 * 4),
        ("upsample_kernel_sizes", C.c_int32 * 4), ("upsample_initial_channel", C.c_int32),
        ("zero_g", C.c_int32), ("hop_length", C.c_int32),
    ]


class ItemParams(C.Structure):
    """struct ovc_item_params of include/ovc.h: per-item device arrays ([B] each, NULL = the call's value)."""
    _fields_ = [
        ("seed", C.c_void_p), ("stream", C.c_void_p), ("frame0", C.c_void_p), ("tau", C.c_void_p),
        ("noise_scale", C.c_void_p), ("noise_scale_w", C.c_void_p), ("length_scale", C.c_void_p),
        ("sdp_ratio", C.c_void_p),
    ]


class TtsFit(C.Structure):
    """struct ovc_tts_fit of include/ovc.h: fit groups of ovc_tts_encode_fit (device arrays)."""
    _fields_ = [
        ("row0", C.c_void_p), ("row1", C.c_void_p), ("target_frames", C.c_void_p), ("G", C.c_int),
        ("scale_lo", C.c_float), ("scale_hi", C.c_float), ("length_scale", C.c_void_p),
    ]


# dtype of each ItemParams field's device array (seeds travel as int64 holding the uint64 bit pattern)
ITEM_FIELDS = {"seed": "int64", "stream": "int64", "frame0": "int64", "tau": "float32", "noise_scale": "float32",
               "noise_scale_w": "float32", "length_scale": "float32", "sdp_ratio": "float32"}


def item_params(items: Optional[dict], B: int) -> Optional[ItemParams]:
    """ItemParams from ``{field: [B] cuda tensor or None}`` (None -> no struct: the entry point without items).  Each
    tensor must be contiguous, on the device and of the field's dtype (``ITEM_FIELDS``); the caller keeps the tensors
    alive until the call's kernels have run."""
    if items is None:
        return None
    import torch
    s = ItemParams()
    for k, t in items.items():
        if k not in ITEM_FIELDS:
            raise ValueError(f"unknown item parameter {k!r} (known: {sorted(ITEM_FIELDS)})")
        if t is None:
            continue
        assert t.is_cuda and t.is_contiguous() and t.dtype == getattr(torch, ITEM_FIELDS[k]), k
        if tuple(t.shape) != (B,):
            raise ValueError(f"item parameter {k!r} has shape {tuple(t.shape)}, expected ({B},)")
        setattr(s, k, t.data_ptr())
    return s


def _items_ref(s: Optional[ItemParams]):
    return C.byref(s) if s is not None else None


PRECISIONS = {"fp32": 0, "f16x3": 1, "f16": 2}


class OvcError(RuntimeError):
    pass


_lib = None


def load_library(path: Optional[str] = None):
    """dlopen the CUDA library (once).  Raises OvcError when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    path = path or os.environ.get("OVC_B200_LIB", LIB_PATH)
    if not os.path.exists(path):
        raise OvcError(
            f"{path} not found: build the sm_90a extension first "
            "(python -c 'import __graft_entry__ as g; g.build()' or make -C openvoice_b200/csrc). "
            "openvoice_b200 has no CPU / PyTorch fallback.")
    lib = C.CDLL(path)
    lib.ovc_abi_version.restype = C.c_int
    lib.ovc_last_error.restype = C.c_char_p
    lib.ovc_create.argtypes = [C.POINTER(OvcHParams), C.c_int, C.POINTER(C.c_void_p)]
    lib.ovc_destroy.argtypes = [C.c_void_p]
    lib.ovc_destroy.restype = None
    lib.ovc_load_tensor.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.POINTER(C.c_int64), C.c_int]
    lib.ovc_finalize_weights.argtypes = [C.c_void_p]
    lib.ovc_workspace_floats.argtypes = [C.c_void_p, C.c_int, C.c_int]
    lib.ovc_workspace_floats.restype = C.c_size_t
    lib.ovc_voice_conversion.argtypes = [
        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_float,
        C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.ovc_last_launch_count.argtypes = [C.c_void_p]
    lib.ovc_graph_replays.argtypes = [C.c_void_p]
    lib.ovc_graph_replays.restype = C.c_int
    lib.ovc_set_precision.argtypes = [C.c_void_p, C.c_int]
    lib.ovc_set_option.argtypes = [C.c_void_p, C.c_int, C.c_int]
    lib.ovc_reference_encoder.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lib.ovc_reference_encoder_ragged.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                                 C.c_void_p]
    lib.ovc_profile_enable.argtypes = [C.c_void_p, C.c_int]
    lib.ovc_profile_read.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int64),
                                     C.POINTER(C.c_double), C.POINTER(C.c_double)]
    lib.ovc_profile_detail.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.POINTER(C.c_double), C.POINTER(C.c_double),
                                       C.POINTER(C.c_double), C.POINTER(C.c_int)]
    lib.ovc_debug_enable.argtypes = [C.c_void_p, C.c_int]
    lib.ovc_debug_fetch.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_int64)]
    lib.ovc_spectrogram.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                    C.c_void_p, C.c_void_p]
    lib.ovc_spectrogram_ring.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lib.ovc_convert_waveform.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_uint64, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.ovc_tts_info.argtypes = [C.c_void_p, C.POINTER(C.c_int32)]
    lib.ovc_tts_encode.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_float,
                                   C.c_float, C.c_float, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.ovc_tts_decode.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_float, C.c_int, C.c_int, C.c_int, C.c_int,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.ovc_resample.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int64,
                                 C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]
    lib.ovc_resample_span.argtypes = [C.c_int, C.c_int, C.c_int64, C.c_int64, C.c_int64, C.POINTER(C.c_int64)]
    P = C.POINTER(ItemParams)
    lib.ovc_voice_conversion_items.argtypes = lib.ovc_voice_conversion.argtypes + [P]
    lib.ovc_convert_waveform_items.argtypes = lib.ovc_convert_waveform.argtypes + [P]
    lib.ovc_tts_encode_items.argtypes = lib.ovc_tts_encode.argtypes + [P]
    lib.ovc_tts_decode_items.argtypes = lib.ovc_tts_decode.argtypes + [P]
    lib.ovc_philox_normals.argtypes = [C.c_uint64, C.c_int64, C.c_int64, C.c_int, C.c_int64, C.c_int, C.c_void_p,
                                       C.c_void_p]
    lib.ovc_tts_encode_state.argtypes = [C.c_void_p] * 5
    lib.ovc_tts_encode_state_tokens.argtypes = [C.c_void_p] * 5
    lib.ovc_tts_encode_g.argtypes = lib.ovc_tts_encode.argtypes[:4] + [C.c_int] + lib.ovc_tts_encode.argtypes[4:] + [P]
    lib.ovc_tts_decode_windows.argtypes = ([C.c_void_p] * 5 + [C.c_int, C.c_int] + [C.c_void_p] * 3 + [C.c_int, C.c_int]
                                           + [C.c_void_p] * 6)
    lib.ovc_tts_decode_windows_tokens.argtypes = lib.ovc_tts_decode_windows.argtypes
    lib.ovc_splice.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int,
                               C.c_int, C.c_void_p]
    lib.ovc_tts_encode_state_rows.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 5
    lib.ovc_tts_state_rows.argtypes = ([C.c_void_p] * 5 + [C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int]
                                       + [C.c_void_p] * 5)
    lib.ovc_tts_encode_state_rows_tokens.argtypes = lib.ovc_tts_encode_state_rows.argtypes
    lib.ovc_tts_state_rows_tokens.argtypes = lib.ovc_tts_state_rows.argtypes
    lib.ovc_voice_conversion_frames.argtypes = (lib.ovc_voice_conversion.argtypes[:5] + [C.c_int]
                                                + lib.ovc_voice_conversion.argtypes[5:] + [P])
    lib.ovc_convert_waveform_frames.argtypes = (lib.ovc_convert_waveform.argtypes[:7] + [C.c_int]
                                                + lib.ovc_convert_waveform.argtypes[7:] + [P])
    lib.ovc_tone_track_expand.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64] + [C.c_void_p] * 4 + [
        C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lib.ovc_resample_plan.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int32), C.c_void_p]
    lib.ovc_resample_rings.argtypes = ([C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int64] + [C.c_void_p] * 5
                                       + [C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_void_p])
    lib.ovc_reference_encoder_stream_state_floats.restype = C.c_size_t
    lib.ovc_reference_encoder_stream_state_floats.argtypes = [C.c_void_p]
    lib.ovc_reference_encoder_stream.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_int, C.c_void_p,
                                                 C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lib.ovc_generate_frames.argtypes = [C.c_void_p] * 4 + [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lib.ovc_tts_encode_fit.argtypes = (lib.ovc_tts_encode.argtypes[:4] + [C.c_void_p, C.c_int]
                                       + lib.ovc_tts_encode.argtypes[4:] + [P, C.POINTER(TtsFit)])
    if lib.ovc_abi_version() != ABI_VERSION:
        raise OvcError(f"ABI mismatch: library {lib.ovc_abi_version()} vs binding {ABI_VERSION}")
    _lib = lib
    return lib


def _check(lib, rc: int, what: str):
    if rc < 0:
        msg = lib.ovc_last_error().decode("utf-8", "replace")
        if rc == -1:
            raise ValueError(f"{what}: {msg}")
        raise OvcError(f"{what}: {msg} (status {rc})")


def hparams_struct(hps) -> OvcHParams:
    """Build struct ovc_hparams from the reference-style config tree (utils.HParams or dict)."""
    def get(obj, k, default=None):
        if isinstance(obj, dict):
            return obj.get(k, default)
        return getattr(obj, k, default)

    model, data = get(hps, "model"), get(hps, "data")
    s = OvcHParams()
    s.spec_channels = int(get(data, "filter_length")) // 2 + 1
    s.inter_channels = int(get(model, "inter_channels"))
    s.hidden_channels = int(get(model, "hidden_channels"))
    s.gin_channels = int(get(model, "gin_channels", 256))
    rb = str(get(model, "resblock"))
    s.resblock = 1 if rb == "1" else 2
    ks = list(get(model, "resblock_kernel_sizes"))
    ds = [list(d) for d in get(model, "resblock_dilation_sizes")]
    if len(ks) > 4 or any(len(d) != 3 for d in ds) or len(ds) != len(ks):
        raise ValueError("unsupported resblock configuration")
    s.n_resblock_kernels = len(ks)
    for i, k in enumerate(ks):
        s.resblock_kernel_sizes[i] = int(k)
        for j in range(3):
            s.resblock_dilations[i][j] = int(ds[i][j])
    ur, uk = list(get(model, "upsample_rates")), list(get(model, "upsample_kernel_sizes"))
    if len(ur) > 4 or len(ur) != len(uk):
        raise ValueError("unsupported upsample configuration")
    s.n_upsamples = len(ur)
    for i in range(len(ur)):
        s.upsample_rates[i] = int(ur[i])
        s.upsample_kernel_sizes[i] = int(uk[i])
    s.upsample_initial_channel = int(get(model, "upsample_initial_channel"))
    s.zero_g = 1 if get(model, "zero_g", False) else 0
    s.hop_length = int(get(data, "hop_length"))
    return s


def philox_normals(seed: int, stream: int, c0: int, channels: int, frame0: int, T: int, device=None, stream_obj=None):
    """[channels, T] float32 cuda tensor of the in-kernel Philox draws at (key = seed; stream, c0 + c, frame0 + t)
    (include/ovc.h: ovc_philox_normals): the noise a per-item-keyed call draws, as an explicit tensor."""
    import torch
    lib = load_library()
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    out = torch.empty(int(channels), int(T), device=dev, dtype=torch.float32)
    st = stream_obj if stream_obj is not None else torch.cuda.current_stream(dev)
    with torch.cuda.device(dev):
        rc = lib.ovc_philox_normals(C.c_uint64(int(seed) & (2 ** 64 - 1)), int(stream), int(c0), int(channels),
                                    int(frame0), int(T), C.c_void_p(out.data_ptr()), C.c_void_p(st.cuda_stream))
    _check(lib, rc, "ovc_philox_normals")
    return out


def resample_span(sr_in: int, sr_out: int, n_in: int = 0, m0: int = 0, m1: int = 1) -> Tuple[int, int, int, int]:
    """Geometry of ``NativeConverter.resample`` (include/ovc.h: ovc_resample_span), computed on the host:
    (n_out(n_in), outputs a stream of n_in samples can emit, and the input samples [lo, hi) outputs [m0, m1) read).
    Raises ValueError naming both rates for a pair the resampler refuses."""
    lib = load_library()
    out = (C.c_int64 * 4)()
    _check(lib, lib.ovc_resample_span(int(sr_in), int(sr_out), int(n_in), int(m0), int(m1), out), "ovc_resample_span")
    return int(out[0]), int(out[1]), int(out[2]), int(out[3])


class NativeConverter:
    """Owns one ovc_ctx (one per device)."""

    def __init__(self, hps, device_index: int):
        self.lib = load_library()
        self.hp = hparams_struct(hps)
        h = C.c_void_p()
        _check(self.lib, self.lib.ovc_create(C.byref(self.hp), int(device_index), C.byref(h)), "ovc_create")
        self.handle = h
        self.device_index = int(device_index)
        self.finalized = False

    def close(self):
        if getattr(self, "handle", None):
            self.lib.ovc_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- weights ---------------------------------------------------------------------------
    def load_state_dict(self, sd: Dict[str, "object"]) -> Tuple[list, list]:
        """Feed a reference-schema state dict; returns (used_keys, ignored_keys)."""
        import numpy as np
        used, ignored = [], []
        for k, v in sd.items():
            a = v.detach().cpu().float().contiguous().numpy() if hasattr(v, "detach") else np.ascontiguousarray(v, dtype=np.float32)
            if a.ndim == 0 or a.ndim > 4:
                ignored.append(k)
                continue
            shape = (C.c_int64 * a.ndim)(*a.shape)
            rc = self.lib.ovc_load_tensor(self.handle, k.encode(), a.ctypes.data_as(C.c_void_p), shape, a.ndim)
            _check(self.lib, rc, f"ovc_load_tensor({k})")
            (ignored if rc == 1 else used).append(k)
        self.finalized = False
        return used, ignored

    def finalize(self):
        _check(self.lib, self.lib.ovc_finalize_weights(self.handle), "ovc_finalize_weights")
        self.finalized = True

    def set_precision(self, mode: str):
        """'fp32' (CUDA-core FFMA), 'f16x3' (split-precision fp16 tensor-core convs, fp32-grade) or 'f16' (single pass)."""
        m = PRECISIONS[mode]
        _check(self.lib, self.lib.ovc_set_precision(self.handle, m), "ovc_set_precision")
        self.precision = mode

    def set_option(self, key: str, value: int):
        """Tuning switches of include/ovc.h: 'tts_simple', 'graph', 'pdl' (0/1/2), 'branches', 'pair', 'pair_occ', 'staged_epi' (0/1)."""
        k = {"tts_simple": 2, "graph": 3, "pdl": 5, "branches": 7, "pair": 8, "pair_occ": 9, "staged_epi": 10}[key]
        _check(self.lib, self.lib.ovc_set_option(self.handle, k, int(value)), "ovc_set_option")

    # ---- hot path --------------------------------------------------------------------------
    def voice_conversion(self, spec, lengths, g_src, g_tgt, noise=None, tau: float = 0.3, seed: int = 0,
                         ragged: bool = False, latents: bool = True, stream=None, items: Optional[dict] = None, out=None):
        """spec [B,S,T] f32 cuda, lengths [B] i64 cuda, g_* [B,gin(,1)] (per item) or [B,gin,T] (per frame) f32 cuda.
        Returns (o_hat [B,1,hop*T], (z, z_p, z_hat) or None).  Asynchronous on `stream`.  ``items``: per-item
        parameters ``{"seed", "stream", "frame0", "tau": [B] cuda tensor}`` (see ``item_params``), or None.  ``out``:
        a caller-owned o_hat buffer of B * hop * T floats (a repeated call on stable buffers replays its CUDA graph)."""
        import torch
        assert spec.is_cuda and spec.dtype == torch.float32 and spec.is_contiguous()
        assert lengths.is_cuda and lengths.dtype == torch.int64 and lengths.is_contiguous()
        B, S, T = spec.shape
        gs, fs = se_arg(g_src, B, self.hp.gin_channels, T, "g_src")
        gt, ft = se_arg(g_tgt, B, self.hp.gin_channels, T, "g_tgt")
        if noise is not None:
            noise = noise.contiguous().float()
            assert tuple(noise.shape) == (B, self.hp.inter_channels, T)
        hop = self.hp.hop_length
        if out is not None:
            assert out.is_cuda and out.dtype == torch.float32 and out.is_contiguous() and out.numel() == B * hop * T
            o = out.view(B, 1, hop * T)
        else:
            o = torch.empty(B, 1, hop * T, device=spec.device, dtype=torch.float32)
        lat = None
        if latents:
            lat = tuple(torch.empty(B, self.hp.inter_channels, T, device=spec.device, dtype=torch.float32)
                        for _ in range(3))
        st = stream if stream is not None else torch.cuda.current_stream(spec.device)
        p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
        it = item_params(items, B)
        rc = self.lib.ovc_voice_conversion_frames(
            self.handle, p(spec), p(lengths), p(gs), p(gt), (SE_FRAMES_SRC if fs else 0) | (SE_FRAMES_TGT if ft else 0),
            p(noise), C.c_uint64(seed & (2 ** 64 - 1)),
            C.c_float(tau), B, T, 1 if ragged else 0, p(o),
            p(lat[0]) if lat else None, p(lat[1]) if lat else None, p(lat[2]) if lat else None,
            C.c_void_p(st.cuda_stream), _items_ref(it))
        _check(self.lib, rc, "ovc_voice_conversion")
        return o, lat

    def latent(self, spec, lengths, g_src, g_tgt, items: Optional[dict] = None, out=None, stream=None):
        """The latent half of ``voice_conversion`` (ragged): posterior encoder, flow forward with g_src, flow reverse
        with g_tgt, and no generator (``ovc_voice_conversion_frames`` with o_hat NULL).  Arguments as there; ``out``: a
        caller-owned z_hat buffer of B * inter * T floats.  Returns z_hat [B, inter, T], bit for bit the z_hat
        ``voice_conversion(..., ragged=True)`` returns.  Asynchronous on `stream`."""
        import torch
        assert spec.is_cuda and spec.dtype == torch.float32 and spec.is_contiguous()
        assert lengths.is_cuda and lengths.dtype == torch.int64 and lengths.is_contiguous()
        B, S, T = spec.shape
        gs, fs = se_arg(g_src, B, self.hp.gin_channels, T, "g_src")
        gt, ft = se_arg(g_tgt, B, self.hp.gin_channels, T, "g_tgt")
        C_ = self.hp.inter_channels
        if out is not None:
            assert out.is_cuda and out.dtype == torch.float32 and out.is_contiguous() and out.numel() == B * C_ * T
            z = out.view(B, C_, T)
        else:
            z = torch.empty(B, C_, T, device=spec.device, dtype=torch.float32)
        st = stream if stream is not None else torch.cuda.current_stream(spec.device)
        p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
        rc = self.lib.ovc_voice_conversion_frames(
            self.handle, p(spec), p(lengths), p(gs), p(gt), (SE_FRAMES_SRC if fs else 0) | (SE_FRAMES_TGT if ft else 0),
            None, C.c_uint64(0), C.c_float(0.3), B, T, 1, None, None, None, p(z), C.c_void_p(st.cuda_stream),
            _items_ref(item_params(items, B)))
        _check(self.lib, rc, "ovc_voice_conversion_frames (latent half)")
        return z

    def generate(self, z_hat, lengths, g_tgt, out=None, stream=None):
        """The generator half (``ovc_generate_frames``): z_hat [B, inter, T] f32 cuda, lengths [B] i64 cuda (each item at
        its own length), g_tgt [B, gin(,1)] per item or [B, gin, T] per frame.  ``out``: a caller-owned o_hat buffer of
        B * hop * T floats.  Returns o_hat [B, 1, hop * T]; on ``latent``'s z_hat it equals ``voice_conversion(...,
        ragged=True)``'s o_hat bit for bit.  Asynchronous on `stream`."""
        import torch
        assert z_hat.is_cuda and z_hat.dtype == torch.float32 and z_hat.is_contiguous()
        assert lengths.is_cuda and lengths.dtype == torch.int64 and lengths.is_contiguous()
        B, _, T = z_hat.shape
        assert z_hat.shape[1] == self.hp.inter_channels
        gt, ft = se_arg(g_tgt, B, self.hp.gin_channels, T, "g_tgt")
        hop = self.hp.hop_length
        if out is not None:
            assert out.is_cuda and out.dtype == torch.float32 and out.is_contiguous() and out.numel() == B * hop * T
            o = out.view(B, 1, hop * T)
        else:
            o = torch.empty(B, 1, hop * T, device=z_hat.device, dtype=torch.float32)
        st = stream if stream is not None else torch.cuda.current_stream(z_hat.device)
        p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
        rc = self.lib.ovc_generate_frames(self.handle, p(z_hat), p(lengths), p(gt), SE_FRAMES_TGT if ft else 0, B, T, p(o),
                                          C.c_void_p(st.cuda_stream))
        _check(self.lib, rc, "ovc_generate_frames")
        return o

    def spectrogram(self, wav, wav_lengths, stream=None):
        """wav [B, Lmax] f32 cuda (zero padded), wav_lengths [B] i64 cuda (samples) ->
        (spec [B, S, Lmax // hop], frames [B] i64): spectrogram_torch on device, per-item reflect padding."""
        import torch
        assert wav.is_cuda and wav.dtype == torch.float32 and wav.is_contiguous() and wav.dim() == 2
        assert wav_lengths.is_cuda and wav_lengths.dtype == torch.int64
        B, L = wav.shape
        T = L // self.hp.hop_length
        spec = torch.empty(B, self.hp.spec_channels, T, device=wav.device, dtype=torch.float32)
        frames = torch.empty(B, device=wav.device, dtype=torch.int64)
        st = stream if stream is not None else torch.cuda.current_stream(wav.device)
        rc = self.lib.ovc_spectrogram(self.handle, C.c_void_p(wav.data_ptr()), C.c_void_p(wav_lengths.data_ptr()), B, L, T,
                                      C.c_void_p(spec.data_ptr()), C.c_void_p(frames.data_ptr()), C.c_void_p(st.cuda_stream))
        _check(self.lib, rc, "ovc_spectrogram")
        return spec, frames

    def spectrogram_ring(self, rings, row, frame_lo, frames, stream_len, Tmax: int, out=None, stream=None):
        """Spectrogram windows of streams held in device audio rings (include/ovc.h: ovc_spectrogram_ring).
        rings [R, cap] f32 cuda: sample s of the stream in row r at rings[r, s % cap].  row, frame_lo, frames,
        stream_len: [B] i64 cuda; item b is frames [frame_lo[b], frame_lo[b] + frames[b]) of row[b], with reflect padding
        at the end only when stream_len[b] != STREAM_OPEN.  Returns spec [B, S, Tmax] (zeros past frames[b]), written
        into ``out`` when given.  Asynchronous on `stream`."""
        import torch
        assert rings.is_cuda and rings.dtype == torch.float32 and rings.is_contiguous() and rings.dim() == 2
        B = row.numel()
        for t in (row, frame_lo, frames, stream_len):
            assert t.is_cuda and t.dtype == torch.int64 and t.is_contiguous()
            if tuple(t.shape) != (B,):
                raise ValueError(f"spectrogram_ring: per-item arrays need shape ({B},), got {tuple(t.shape)}")
        shape = (B, self.hp.spec_channels, int(Tmax))
        if out is None:
            out = torch.empty(shape, device=rings.device, dtype=torch.float32)
        assert out.is_cuda and out.dtype == torch.float32 and out.is_contiguous() and tuple(out.shape) == shape
        st = stream if stream is not None else torch.cuda.current_stream(rings.device)
        p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
        rc = self.lib.ovc_spectrogram_ring(self.handle, p(rings), int(rings.shape[0]), int(rings.shape[1]), p(row),
                                           p(frame_lo), p(frames), p(stream_len), B, int(Tmax), p(out),
                                           C.c_void_p(st.cuda_stream))
        _check(self.lib, rc, "ovc_spectrogram_ring")
        return out

    def convert_waveform(self, wav, wav_lengths, g_src, g_tgt, noise=None, tau: float = 0.3, seed: int = 0, stream=None,
                         out=None, frames_out=None, items: Optional[dict] = None):
        """The device work of ToneColorConverter.convert for a batch: wav [B, Lmax] f32 cuda ->
        (o_hat [B, hop * (Lmax // hop)], frames [B]).  Asynchronous on `stream`.  ``out`` / ``frames_out`` let the
        caller supply the result buffers: with every buffer at a stable address, a repeated call is replayed from a
        CUDA graph (include/ovc.h: OVC_OPT_GRAPH).  ``items`` as in ``voice_conversion``; ``g_*`` per item or
        [B, gin, Lmax // hop] per frame."""
        import torch
        assert wav.is_cuda and wav.dtype == torch.float32 and wav.is_contiguous() and wav.dim() == 2
        assert wav_lengths.is_cuda and wav_lengths.dtype == torch.int64
        B, L = wav.shape
        T = L // self.hp.hop_length
        gs, fs = se_arg(g_src, B, self.hp.gin_channels, T, "g_src")
        gt, ft = se_arg(g_tgt, B, self.hp.gin_channels, T, "g_tgt")
        if noise is not None:
            noise = noise.contiguous().float()
            assert tuple(noise.shape) == (B, self.hp.inter_channels, T)
        if out is not None:
            assert out.is_cuda and out.dtype == torch.float32 and out.is_contiguous() and out.numel() == B * self.hp.hop_length * T
            o = out.view(B, self.hp.hop_length * T)
        else:
            o = torch.empty(B, self.hp.hop_length * T, device=wav.device, dtype=torch.float32)
        if frames_out is not None:
            assert frames_out.is_cuda and frames_out.dtype == torch.int64 and frames_out.numel() == B
            frames = frames_out
        else:
            frames = torch.empty(B, device=wav.device, dtype=torch.int64)
        st = stream if stream is not None else torch.cuda.current_stream(wav.device)
        it = item_params(items, B)
        rc = self.lib.ovc_convert_waveform_frames(
            self.handle, C.c_void_p(wav.data_ptr()), C.c_void_p(wav_lengths.data_ptr()), B, L, C.c_void_p(gs.data_ptr()),
            C.c_void_p(gt.data_ptr()), (SE_FRAMES_SRC if fs else 0) | (SE_FRAMES_TGT if ft else 0), C.c_void_p(noise.data_ptr()) if noise is not None else None,
            C.c_uint64(seed & (2 ** 64 - 1)), C.c_float(tau), C.c_void_p(o.data_ptr()), C.c_void_p(frames.data_ptr()),
            C.c_void_p(st.cuda_stream), _items_ref(it))
        _check(self.lib, rc, "ovc_convert_waveform")
        return o, frames

    def tone_track_expand(self, key_frame, key_se, key0, nkeys, frame0, frames, Tmax: int, out=None, stream=None):
        """Per-frame embeddings [B, gin, Tmax] from keyframe tracks (include/ovc.h: ovc_tone_track_expand).
        key_frame [K] i64, key_se [K, gin] f32, key0 / nkeys / frame0 / frames [B] i64, all cuda and contiguous; item b
        is track keys [key0[b], key0[b] + nkeys[b]) evaluated at frames frame0[b] + t, t < frames[b] (zeros after).
        Written into ``out`` when given.  Asynchronous on `stream`."""
        import torch
        gin = self.hp.gin_channels
        K = key_frame.numel()
        assert key_frame.is_cuda and key_frame.dtype == torch.int64 and key_frame.is_contiguous()
        assert key_se.is_cuda and key_se.dtype == torch.float32 and key_se.is_contiguous()
        if tuple(key_se.shape) != (K, gin):
            raise ValueError(f"key_se has shape {tuple(key_se.shape)}, expected ({K}, {gin})")
        B = key0.numel()
        for t in (key0, nkeys, frame0, frames):
            assert t.is_cuda and t.dtype == torch.int64 and t.is_contiguous()
            if tuple(t.shape) != (B,):
                raise ValueError(f"tone_track_expand: per-item arrays need shape ({B},), got {tuple(t.shape)}")
        shape = (B, gin, int(Tmax))
        if out is None:
            out = torch.empty(shape, device=key_se.device, dtype=torch.float32)
        assert out.is_cuda and out.dtype == torch.float32 and out.is_contiguous() and tuple(out.shape) == shape
        st = stream if stream is not None else torch.cuda.current_stream(key_se.device)
        p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
        rc = self.lib.ovc_tone_track_expand(self.handle, p(key_frame), p(key_se), K, p(key0), p(nkeys), p(frame0), p(frames),
                                            B, int(Tmax), p(out), C.c_void_p(st.cuda_stream))
        _check(self.lib, rc, "ovc_tone_track_expand")
        return out

    def reference_encoder(self, spec, lengths=None, stream=None):
        """spec [N, S, T] f32 cuda (ovc_spectrogram layout) -> tone-colour embedding [N, gin]
        (ReferenceEncoder.forward, openvoice/models.py:339-359).  ``lengths`` ([N] int64 cuda, frames, or None): every
        item is encoded at its own length and row n equals a call on ``spec[n:n+1, :, :lengths[n]]`` bit for bit; the
        frames past it are never read.  The ``frames`` output of ``spectrogram`` can be passed as is (no host sync)."""
        import torch
        assert spec.is_cuda and spec.dtype == torch.float32 and spec.is_contiguous() and spec.dim() == 3
        N, S, T = spec.shape
        if S != self.hp.spec_channels:
            raise ValueError(f"reference_encoder: spec has {S} channels, the model has spec_channels {self.hp.spec_channels}")
        if lengths is not None:
            assert lengths.is_cuda and lengths.dtype == torch.int64 and lengths.is_contiguous()
            if tuple(lengths.shape) != (N,):
                raise ValueError(f"reference_encoder: lengths has shape {tuple(lengths.shape)}, expected ({N},)")
        out = torch.empty(N, self.hp.gin_channels, device=spec.device, dtype=torch.float32)
        st = stream if stream is not None else torch.cuda.current_stream(spec.device)
        if lengths is None:
            rc = self.lib.ovc_reference_encoder(self.handle, C.c_void_p(spec.data_ptr()), N, T, C.c_void_p(out.data_ptr()),
                                                C.c_void_p(st.cuda_stream))
            _check(self.lib, rc, "ovc_reference_encoder")
        else:
            rc = self.lib.ovc_reference_encoder_ragged(self.handle, C.c_void_p(spec.data_ptr()), C.c_void_p(lengths.data_ptr()),
                                                       N, T, C.c_void_p(out.data_ptr()), C.c_void_p(st.cuda_stream))
            _check(self.lib, rc, "ovc_reference_encoder_ragged")
        return out

    @property
    def refenc_state_floats(self) -> int:
        """Floats of one ``reference_encoder_stream`` state row (0 without ref_enc.* tensors)."""
        return int(self.lib.ovc_reference_encoder_stream_state_floats(self.handle))

    def reference_encoder_stream(self, rings, state, desc, max_new_frames: int, out=None, stream=None):
        """Advance streams' reference encoders and take snapshots (include/ovc.h: ovc_reference_encoder_stream).
        rings [R, cap] f32 cuda (sample s of row r at rings[r, s % cap]); state [S, refenc_state_floats] f32 cuda, one
        row per stream, all zeros for a fresh one, updated in place; desc [B, 4] int64 cuda rows (state_row, ring_row,
        n_adv, n_snap).  Returns out [B, gin]: row b is the embedding of the stream's first n_snap samples (NaN when it
        cannot be produced; untouched when n_snap <= 0).  Asynchronous on `stream`; ValueError for bad shapes before any
        launch."""
        import torch
        gin = self.hp.gin_channels
        for name, t, dt in (("rings", rings, torch.float32), ("state", state, torch.float32), ("desc", desc, torch.int64)):
            if not (t.is_cuda and t.dtype == dt and t.is_contiguous() and t.dim() == 2):
                raise ValueError(f"reference_encoder_stream: {name} must be a contiguous 2-D {dt} cuda tensor")
        F = self.refenc_state_floats
        if F == 0:
            raise ValueError("reference_encoder_stream: the checkpoint has no ref_enc.* tensors")
        if state.shape[1] != F:
            raise ValueError(f"reference_encoder_stream: state rows have {state.shape[1]} floats, expected {F}")
        B = desc.shape[0]
        if desc.shape[1] != 4 or B < 1:
            raise ValueError(f"reference_encoder_stream: desc has shape {tuple(desc.shape)}, expected (B >= 1, 4)")
        if rings.shape[1] < 1024 or rings.shape[0] < 1 or state.shape[0] < 1:
            raise ValueError(f"reference_encoder_stream: rings {tuple(rings.shape)} / state {tuple(state.shape)} too small")
        if not 1 <= int(max_new_frames) <= 65536:
            raise ValueError(f"reference_encoder_stream: max_new_frames {max_new_frames} outside [1, 65536]")
        if out is None:
            out = torch.empty(B, gin, device=rings.device, dtype=torch.float32)
        if not (out.is_cuda and out.dtype == torch.float32 and out.is_contiguous() and out.numel() == B * gin):
            raise ValueError(f"reference_encoder_stream: out must be a contiguous float32 cuda tensor of {B} x {gin}")
        st = stream if stream is not None else torch.cuda.current_stream(rings.device)
        p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
        rc = self.lib.ovc_reference_encoder_stream(self.handle, p(rings), int(rings.shape[0]), int(rings.shape[1]), p(state),
                                                   int(state.shape[0]), p(desc), B, int(max_new_frames), p(out),
                                                   C.c_void_p(st.cuda_stream))
        _check(self.lib, rc, "ovc_reference_encoder_stream")
        return out

    def resample(self, x, in_lengths, sr_in: int, sr_out: int, out=None, out_pitch: Optional[int] = None,
                 in_start: int = 0, out_start: int = 0, stream=None):
        """Polyphase resampling on the device (scipy.signal.resample_poly arithmetic, include/ovc.h: ovc_resample).
        x [B, in_pitch] f32 cuda: row b holds samples [in_start, in_start + in_pitch) of item b; in_lengths [B] int64
        cuda: each item's whole input length (STREAM_OPEN: not ended).  Returns out [B, out_pitch] with
        y_b[out_start, out_start + out_pitch), zero past each item's n_out; out_pitch defaults to
        n_out(in_start + in_pitch) - out_start, computed on the host.  Asynchronous on `stream`."""
        import torch
        assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 2
        assert in_lengths.is_cuda and in_lengths.dtype == torch.int64 and in_lengths.is_contiguous()
        B, pitch = x.shape
        if tuple(in_lengths.shape) != (B,):
            raise ValueError(f"resample: in_lengths has shape {tuple(in_lengths.shape)}, expected ({B},)")
        if out_pitch is None:
            out_pitch = (out.shape[1] if out is not None else
                         max(0, resample_span(sr_in, sr_out, in_start + pitch)[0] - out_start))
        if out is None:
            out = torch.empty(B, out_pitch, device=x.device, dtype=torch.float32)
        assert out.is_cuda and out.dtype == torch.float32 and out.is_contiguous() and tuple(out.shape) == (B, out_pitch)
        if out_pitch == 0:
            return out
        st = stream if stream is not None else torch.cuda.current_stream(x.device)
        rc = self.lib.ovc_resample(self.handle, int(sr_in), int(sr_out), C.c_void_p(x.data_ptr()),
                                   C.c_void_p(in_lengths.data_ptr()), B, pitch, int(in_start), C.c_void_p(out.data_ptr()),
                                   int(out_pitch), int(out_start), C.c_void_p(st.cuda_stream))
        _check(self.lib, rc, "ovc_resample")
        return out

    def resample_plan(self, sr_in: int, sr_out: int, stream=None) -> int:
        """Plan id of sr_in -> sr_out for ``resample_rings`` (include/ovc.h: ovc_resample_plan).  Builds the pair's filter
        bank on first use and WAITS for the stream: call it at set-up.  ValueError for a pair the resampler refuses."""
        import torch
        dev = torch.device("cuda", self.device_index)
        st = stream if stream is not None else torch.cuda.current_stream(dev)
        out = C.c_int32(-1)
        with torch.cuda.device(dev):
            rc = self.lib.ovc_resample_plan(self.handle, int(sr_in), int(sr_out), C.byref(out), C.c_void_p(st.cuda_stream))
        _check(self.lib, rc, "ovc_resample_plan")
        return int(out.value)

    def resample_rings(self, plan, x, in_row, in_len, m0, count, out, out_row, out_off, max_count: int, stream=None):
        """Many streams' resampling in one launch (include/ovc.h: ovc_resample_rings): item b computes outputs
        [m0[b], m0[b] + count[b]) of plan[b], reading x[in_row[b], j % cap] (0 outside [0, in_len[b])) and writing output
        m to out[out_row[b], (out_off[b] + m - m0[b]) % out_cap].  plan [B] int32, the rest [B] int64, all cuda; x and
        out 2-D f32 cuda.  Asynchronous on `stream`; returns ``out``."""
        import torch
        for t in (x, out):
            assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.dim() == 2
        B = plan.numel()
        assert plan.is_cuda and plan.dtype == torch.int32 and plan.is_contiguous()
        for t in (in_row, in_len, m0, count, out_row, out_off):
            assert t.is_cuda and t.dtype == torch.int64 and t.is_contiguous()
            if t.numel() != B:
                raise ValueError(f"resample_rings: per-item arrays need {B} values, got {t.numel()}")
        st = stream if stream is not None else torch.cuda.current_stream(out.device)
        p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
        rc = self.lib.ovc_resample_rings(self.handle, p(plan), p(x), int(x.shape[0]), int(x.shape[1]), p(in_row),
                                         p(in_len), p(m0), p(count), p(out), int(out.shape[0]), int(out.shape[1]),
                                         p(out_row), p(out_off), B, int(max_count), C.c_void_p(st.cuda_stream))
        _check(self.lib, rc, "ovc_resample_rings")
        return out

    def splice(self, src, seg, dst, pcm16: bool = False, stream=None, src_wrap: bool = False):
        """Copy sample runs between device buffers in one launch (include/ovc.h: ovc_splice).  src [rows, pitch] f32
        cuda, or None when every segment is a gap; seg [S, 5] int64 cuda, rows (src_row, src_off, count, dst_row,
        dst_off); dst [rows, cap] f32 cuda, written in place: segment s puts src[src_row, src_off + i] (0 when src_row
        < 0) at dst[dst_row, (dst_off + i) % cap], i < count.  ``pcm16``: every copied value takes the 16-bit PCM round
        trip (``SPLICE_PCM16``).  ``src_wrap``: the source rows are rings too, segment s reads
        src[src_row, (src_off + i) % pitch] (``SPLICE_SRC_WRAP``).  Asynchronous on `stream`; returns ``dst``."""
        import torch
        assert dst.is_cuda and dst.dtype == torch.float32 and dst.is_contiguous() and dst.dim() == 2
        assert seg.is_cuda and seg.dtype == torch.int64 and seg.is_contiguous()
        if seg.dim() != 2 or seg.shape[1] != 5:
            raise ValueError(f"splice: seg needs shape (S, 5), got {tuple(seg.shape)}")
        if src is not None:
            assert src.is_cuda and src.dtype == torch.float32 and src.is_contiguous() and src.dim() == 2
            assert src.device == dst.device
        rows, pitch = (0, 0) if src is None else (int(src.shape[0]), int(src.shape[1]))
        st = stream if stream is not None else torch.cuda.current_stream(dst.device)
        with torch.cuda.device(dst.device):
            rc = self.lib.ovc_splice(None if src is None else C.c_void_p(src.data_ptr()), rows, pitch,
                                     C.c_void_p(dst.data_ptr()), int(dst.shape[0]), int(dst.shape[1]),
                                     C.c_void_p(seg.data_ptr()), int(seg.shape[0]),
                                     (SPLICE_PCM16 if pcm16 else 0) | (SPLICE_SRC_WRAP if src_wrap else 0),
                                     C.c_void_p(st.cuda_stream))
        _check(self.lib, rc, "ovc_splice")
        return dst

    # ---- V1 TTS front half (SynthesizerTrn.infer, openvoice/models.py:467-490) ----------------
    def tts_info(self) -> dict:
        out = (C.c_int32 * 8)()
        _check(self.lib, self.lib.ovc_tts_info(self.handle, out), "ovc_tts_info")
        keys = ("has_tts", "n_vocab", "n_speakers", "n_heads", "n_layers", "window", "filter_channels", "dp_filter")
        return dict(zip(keys, (int(v) for v in out)))

    def tts_encode(self, tokens, x_lengths, sid, noise_w=None, seed: int = 0, noise_scale_w: float = 1.0,
                   length_scale: float = 1.0, sdp_ratio: float = 0.2, stream=None, items: Optional[dict] = None,
                   g=None, fit=None):
        """tokens [B,T] i64 cuda, x_lengths [B] i64 cuda, sid [B] i64 cuda, noise_w [B,2,T] or None (Philox).
        Returns (y_lengths [B] i64, w_ceil [B,T], logw [B,T]), all on the device; asynchronous on `stream`.
        ``items``: per-item ``{"seed", "stream", "noise_scale_w", "length_scale", "sdp_ratio"}`` (``item_params``).
        ``g``: speaker vectors instead of ``sid`` (which is then ignored), f32 cuda [B, gin] or per token [B, gin, T]
        (include/ovc.h: ovc_tts_encode_g).
        ``fit``: ``(row0, row1, target_frames, scale_lo, scale_hi)``, the first three [G] i64 cuda tensors (include/ovc.h:
        ovc_tts_encode_fit); the return then ends with each row's length scale, [B] f32 on the device."""
        import torch
        for t in (tokens, x_lengths) + ((sid,) if g is None else ()):
            assert t.is_cuda and t.dtype == torch.int64 and t.is_contiguous()
        B, T = tokens.shape
        if g is not None:
            gin = self.hp.gin_channels
            assert g.is_cuda and g.dtype == torch.float32 and g.is_contiguous()
            assert tuple(g.shape) in ((B, gin), (B, gin, T)), tuple(g.shape)
        if noise_w is not None:
            noise_w = noise_w.contiguous().float()
            assert tuple(noise_w.shape) == (B, 2, T)
        y_lengths = torch.empty(B, device=tokens.device, dtype=torch.int64)
        w_ceil = torch.empty(B, T, device=tokens.device, dtype=torch.float32)
        logw = torch.empty(B, T, device=tokens.device, dtype=torch.float32)
        st = stream if stream is not None else torch.cuda.current_stream(tokens.device)
        p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
        it = item_params(items, B)
        rest = (p(noise_w), C.c_uint64(seed & (2 ** 64 - 1)), C.c_float(noise_scale_w), C.c_float(length_scale),
                C.c_float(sdp_ratio), B, T, p(y_lengths), p(w_ceil), p(logw), C.c_void_p(st.cuda_stream), _items_ref(it))
        if fit is not None:
            row0, row1, target, lo, hi = fit
            for t in (row0, row1, target):
                assert t.is_cuda and t.dtype == torch.int64 and t.is_contiguous() and t.shape == row0.shape
            scale = torch.empty(B, device=tokens.device, dtype=torch.float32)
            f = TtsFit(p(row0), p(row1), p(target), int(row0.numel()), lo, hi, p(scale))
            rc = self.lib.ovc_tts_encode_fit(self.handle, p(tokens), p(x_lengths), p(sid) if g is None else None, p(g),
                                             1 if g is not None and g.dim() == 3 else 0, *rest, C.byref(f))
            _check(self.lib, rc, "ovc_tts_encode_fit")
            return y_lengths, w_ceil, logw, scale
        if g is None:
            rc = self.lib.ovc_tts_encode_items(self.handle, p(tokens), p(x_lengths), p(sid), *rest)
        else:
            rc = self.lib.ovc_tts_encode_g(self.handle, p(tokens), p(x_lengths), p(g), 1 if g.dim() == 3 else 0, *rest)
        _check(self.lib, rc, "ovc_tts_encode")
        return y_lengths, w_ceil, logw

    def tts_decode(self, B: int, y_max: int, device, noise=None, seed: int = 0, noise_scale: float = 1.0,
                   ragged: bool = False, latents: bool = False, max_len: Optional[int] = None, stream=None,
                   items: Optional[dict] = None):
        """Second half of infer() for the last tts_encode.  Returns (o [B,1,hop*min(y_max, max_len)], (z, z_p) or None).
        ``items``: per-item ``{"seed" (the decode key), "stream", "noise_scale"}`` (``item_params``)."""
        import torch
        C_ = self.hp.inter_channels
        if noise is not None:
            noise = noise.contiguous().float()
            assert noise.is_cuda and tuple(noise.shape) == (B, C_, y_max)
        cut = int(max_len) if max_len is not None and 0 < int(max_len) < y_max else 0
        o = torch.empty(B, 1, self.hp.hop_length * (cut or y_max), device=device, dtype=torch.float32)
        lat = tuple(torch.empty(B, C_, y_max, device=device, dtype=torch.float32) for _ in range(2)) if latents else None
        st = stream if stream is not None else torch.cuda.current_stream(device)
        p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
        it = item_params(items, B)
        rc = self.lib.ovc_tts_decode_items(self.handle, p(noise), C.c_uint64(seed & (2 ** 64 - 1)), C.c_float(noise_scale),
                                           B, int(y_max), cut, 1 if ragged else 0, p(o), p(lat[0]) if lat else None,
                                           p(lat[1]) if lat else None, C.c_void_p(st.cuda_stream), _items_ref(it))
        _check(self.lib, rc, "ovc_tts_decode")
        return o, lat

    def tts_encode_state(self, B: int, T: int, device, stream=None, per_token: bool = False):
        """Caller-owned copies of what the last ``tts_encode`` (B rows of T tokens) left in the context (include/ovc.h:
        ovc_tts_encode_state): (stats [B,T,2*inter] f32, cum [B,T] int32, g [B,gin] f32) on the device.  A later
        ``tts_encode`` does not touch them.  ``per_token``: the encode took per-token vectors, and g is [B,gin,T]
        (ovc_tts_encode_state_tokens).  Asynchronous on `stream`."""
        import torch
        stats = torch.empty(B, T, 2 * self.hp.inter_channels, device=device, dtype=torch.float32)
        cum = torch.empty(B, T, device=device, dtype=torch.int32)
        g = torch.empty(B, self.hp.gin_channels, *((T,) if per_token else ()), device=device, dtype=torch.float32)
        st = stream if stream is not None else torch.cuda.current_stream(device)
        fn = self.lib.ovc_tts_encode_state_tokens if per_token else self.lib.ovc_tts_encode_state
        rc = fn(self.handle, C.c_void_p(stats.data_ptr()), C.c_void_p(cum.data_ptr()), C.c_void_p(g.data_ptr()),
                C.c_void_p(st.cuda_stream))
        _check(self.lib, rc, "ovc_tts_encode_state")
        return stats, cum, g

    def tts_state_rows(self, dst_row, stats, cum, g, y_lengths, src=None, stream=None):
        """Write encoded rows into rows ``dst_row`` (host ints) of a state pool (include/ovc.h: ovc_tts_encode_state_rows,
        ovc_tts_state_rows): stats [N,Tp,2*inter] f32, cum [N,Tp] int32, g [N,gin] f32, y_lengths [N] int64 on the device,
        written in place.  ``src``: None for the rows of the last ``tts_encode``, or caller-owned state (stats, cum, g,
        y_lengths) of B rows.  Tokens past the source's pitch get the library's padding.  A per-token pool has g
        [N,gin,Tp] (its source g is [B,gin,T]; ovc_tts_encode_state_rows_tokens / ovc_tts_state_rows_tokens).
        Asynchronous on `stream`."""
        import torch
        N, Tp = cum.shape
        dev = cum.device
        per_token = g.dim() == 3
        for t, dt, shape in ((stats, torch.float32, (N, Tp, 2 * self.hp.inter_channels)), (cum, torch.int32, (N, Tp)),
                             (g, torch.float32, (N, self.hp.gin_channels) + ((Tp,) if per_token else ())),
                             (y_lengths, torch.int64, (N,))):
            assert t.is_cuda and t.dtype == dt and t.is_contiguous() and tuple(t.shape) == shape, (t.dtype, t.shape)
        st = stream if stream is not None else torch.cuda.current_stream(dev)
        # the row table goes up through a pinned buffer, reused once its previous upload has left it: no host sync
        dst_row = [int(r) for r in dst_row]
        cache = self.__dict__.setdefault("_rows_bufs", {})
        if cache.get("ev") is not None:
            cache["ev"].synchronize()
        n = max(1, len(dst_row))
        if cache.get("pin") is None or cache["pin"].numel() < n or cache["dev"].device != dev:
            cache["pin"] = torch.empty(int(n * 1.25) + 64, dtype=torch.int64).pin_memory()
            cache["dev"] = torch.empty(cache["pin"].numel(), dtype=torch.int64, device=dev)
        cache["pin"][:len(dst_row)].copy_(torch.tensor(dst_row, dtype=torch.int64))
        rows = cache["dev"][:n]
        with torch.cuda.stream(st):
            rows.copy_(cache["pin"][:n], non_blocking=True)
            cache["ev"] = torch.cuda.Event()
            cache["ev"].record(st)
        p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
        if src is None:
            fn = self.lib.ovc_tts_encode_state_rows_tokens if per_token else self.lib.ovc_tts_encode_state_rows
            rc = fn(self.handle, p(rows), N, Tp, p(stats), p(cum), p(g), p(y_lengths),
                                                    C.c_void_p(st.cuda_stream))
        else:
            s_stats, s_cum, s_g, s_len = src
            B, T = s_cum.shape
            if len(dst_row) != B:
                raise ValueError(f"tts_state_rows: {len(dst_row)} destination rows for {B} source rows")
            for t, dt, shape in ((s_stats, torch.float32, (B, T, 2 * self.hp.inter_channels)),
                                 (s_cum, torch.int32, (B, T)),
                                 (s_g, torch.float32, (B, self.hp.gin_channels) + ((T,) if per_token else ())),
                                 (s_len, torch.int64, (B,))):
                assert t.is_cuda and t.dtype == dt and t.is_contiguous() and tuple(t.shape) == shape, (t.dtype, t.shape)
            fn = self.lib.ovc_tts_state_rows_tokens if per_token else self.lib.ovc_tts_state_rows
            rc = fn(self.handle, p(s_stats), p(s_cum), p(s_g), p(s_len), B, T, p(rows), N, Tp, p(stats), p(cum), p(g),
                    p(y_lengths), C.c_void_p(st.cuda_stream))
        _check(self.lib, rc, "ovc_tts_state_rows")
        return stats, cum, g, y_lengths

    def tts_decode_windows(self, stats, cum, g, y_lengths, row, frame0, length, seed, streams, noise_scale, w_max: int,
                           latents: bool = False, slot: int = 0, stream=None):
        """Decode W windows of caller-owned encode state (``tts_encode_state`` + the encode's y_lengths; include/ovc.h:
        ovc_tts_decode_windows).  ``row``, ``frame0``, ``length``, ``seed`` (decode keys in [0, 2^64)), ``streams`` and
        ``noise_scale`` are host sequences of W values.  They are staged through slot ``slot``'s pinned and device
        buffers, and ``o`` is written into the slot's device buffer: with every address stable, a repeated (W, w_max)
        call is replayed from a CUDA graph with the new values.  Returns (o [W, hop * w_max], z_p [W, inter, w_max] or
        None); ``o`` is overwritten by the next call on the slot.  A per-token ``g`` [N, gin, T]
        (``tts_encode_state(per_token=True)``) decodes through ovc_tts_decode_windows_tokens.  Asynchronous on `stream`."""
        import numpy as np
        import torch
        W = len(row)
        vals = [row, frame0, length, seed, streams, noise_scale]
        if W < 1 or any(len(v) != W for v in vals):
            raise ValueError(f"tts_decode_windows: every per-window sequence needs the same length >= 1, got "
                             f"{[len(v) for v in vals]}")
        N, T = cum.shape
        dev = cum.device
        per_token = g.dim() == 3
        for t, dt, shape in ((stats, torch.float32, (N, T, 2 * self.hp.inter_channels)), (cum, torch.int32, (N, T)),
                             (g, torch.float32, (N, self.hp.gin_channels) + ((T,) if per_token else ())),
                             (y_lengths, torch.int64, (N,))):
            assert t.is_cuda and t.dtype == dt and t.is_contiguous() and tuple(t.shape) == shape, (t.dtype, t.shape)
        cache = self.__dict__.setdefault("_win_bufs", {})
        ev = cache.get(("ev", slot))
        if ev is not None:
            ev.synchronize()                  # the slot's previous upload has left the pinned buffers
        ints = np.empty((5, W), dtype=np.int64)
        ints[0], ints[1], ints[2], ints[4] = row, frame0, length, streams
        ints[3] = np.asarray([int(s) & (2 ** 64 - 1) for s in seed], dtype=np.uint64).view(np.int64)

        def buf(name, numel, dtype, pinned=False):
            b = cache.get((name, slot))
            if b is None or b.numel() < numel:
                b = torch.empty(int(numel * 1.25) + 64, dtype=dtype, device="cpu" if pinned else dev)
                b = b.pin_memory() if pinned else b
                cache[(name, slot)] = b
            return b[:numel]
        pin_i, pin_f = buf("pin_i", 5 * W, torch.int64, True), buf("pin_f", W, torch.float32, True)
        pin_i.copy_(torch.from_numpy(ints.reshape(-1)))
        pin_f.copy_(torch.tensor([float(v) for v in noise_scale], dtype=torch.float32))
        d_i, d_f = buf("d_i", 5 * W, torch.int64), buf("d_f", W, torch.float32)
        st = stream if stream is not None else torch.cuda.current_stream(dev)
        with torch.cuda.stream(st):
            d_i.copy_(pin_i, non_blocking=True)
            d_f.copy_(pin_f, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(st)
        cache[("ev", slot)] = ev
        hop = self.hp.hop_length
        o = buf("o", W * hop * int(w_max), torch.float32).view(W, hop * int(w_max))
        zp = torch.empty(W, self.hp.inter_channels, int(w_max), device=dev, dtype=torch.float32) if latents else None
        p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
        fn = self.lib.ovc_tts_decode_windows_tokens if per_token else self.lib.ovc_tts_decode_windows
        rc = fn(
            self.handle, p(stats), p(cum), p(g), p(y_lengths), N, T, p(d_i[0:W]), p(d_i[W:2 * W]), p(d_i[2 * W:3 * W]), W,
            int(w_max), p(d_i[3 * W:4 * W]), p(d_i[4 * W:]), p(d_f), p(o), p(zp) if zp is not None else None,
            C.c_void_p(st.cuda_stream))
        _check(self.lib, rc, "ovc_tts_decode_windows")
        return o, zp

    @property
    def last_launch_count(self) -> int:
        return int(self.lib.ovc_last_launch_count(self.handle))

    @property
    def graph_replays(self) -> int:
        """calls served from a captured CUDA graph so far (include/ovc.h: ovc_graph_replays)"""
        return int(self.lib.ovc_graph_replays(self.handle))

    # ---- instrumentation -------------------------------------------------------------------
    def profile_enable(self, on: bool):
        _check(self.lib, self.lib.ovc_profile_enable(self.handle, 1 if on else 0), "ovc_profile_enable")

    def profile_read(self):
        ms, n, fl, by = C.c_double(), C.c_int64(), C.c_double(), C.c_double()
        _check(self.lib, self.lib.ovc_profile_read(self.handle, C.byref(ms), C.byref(n), C.byref(fl), C.byref(by)),
               "ovc_profile_read")
        return dict(ms=ms.value, launches=n.value, flops=fl.value, bytes=by.value)

    def profile_detail(self, max_entries: int = 4096):
        """Per-launch (name, ms, flops, bytes, family) of the conv kernels since the last reset."""
        names = C.create_string_buffer(16 * max_entries)
        ms = (C.c_double * max_entries)()
        fl = (C.c_double * max_entries)()
        by = (C.c_double * max_entries)()
        fam = (C.c_int * max_entries)()
        n = self.lib.ovc_profile_detail(self.handle, max_entries, names, ms, fl, by, fam)
        _check(self.lib, n, "ovc_profile_detail")
        raw = names.raw
        return [(raw[16 * i: 16 * i + 16].split(b"\0")[0].decode(), ms[i], fl[i], by[i], fam[i]) for i in range(n)]

    def debug_enable(self, on: bool):
        _check(self.lib, self.lib.ovc_debug_enable(self.handle, 1 if on else 0), "ovc_debug_enable")

    def debug_fetch(self, name: str):
        """Returns a numpy array [B, C, T] of the named tap of the last call."""
        import numpy as np
        shape = (C.c_int64 * 4)()
        _check(self.lib, self.lib.ovc_debug_fetch(self.handle, name.encode(), None, 0, shape), "ovc_debug_fetch")
        B, Cc, T, pitch = [int(v) for v in shape]
        buf = np.empty((B, Cc, pitch), dtype=np.float32)
        _check(self.lib, self.lib.ovc_debug_fetch(self.handle, name.encode(), buf.ctypes.data_as(C.c_void_p),
                                                  buf.size, shape), "ovc_debug_fetch")
        return buf[:, :, :T]
