"""Drop-in for the tone-colour-converter half of the reference's ``openvoice/api.py``.

Same classes, method names, arguments and return types as ``OpenVoiceBaseClass`` /
``ToneColorConverter`` (openvoice/api.py:14-39, :101-201); ``self.model`` is a
``NativeSynthesizer`` whose ``voice_conversion`` (the seam at openvoice/api.py:154) runs in
libovc_b200.so.  Supersets of the reference: ``convert`` also accepts a NumPy waveform,
``convert_batch`` converts a list of utterances in one launch sequence, ``clone_batch`` /
``clone_stream_batch`` take text to cloned voice with the TTS audio joined on the device,
``enable_watermark=False`` works (it raises TypeError in the reference, SURVEY.md section 3.2).
CUDA only: there is no CPU path.
"""
from __future__ import annotations

import math
import os
from typing import Iterator, List, NamedTuple, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import utils
from ._native import NativeConverter, resample_span
from .ref_enc import ReferenceEncoder
from .schema import hot_path_keys, ref_enc_keys, tts_keys

AudioLike = Union[str, np.ndarray]


class ToneTrack:
    """A tone colour that changes over time: keyframes ``(frame, embedding)`` at non-decreasing spectrogram frames
    (256 samples at the model's rate each).  At frame t the embedding is the first key's before the first key, the last
    key's from the last key on, and between keys f_k <= t < f_{k+1} the fp32 interpolation
    ``se_k + ((t - f_k) / (f_{k+1} - f_k)) * (se_{k+1} - se_k)``; two keys at the same frame switch hard to the later one
    there.  A track means exactly the per-frame embedding ``dense`` returns, and the conversion paths evaluate it on the
    device (include/ovc.h: ovc_tone_track_expand) with the same arithmetic."""

    def __init__(self, keys):
        ks = list(keys)
        if not ks:
            raise ValueError("a ToneTrack needs at least one keyframe")
        frames, ses = [], []
        for f, se in ks:
            if int(f) != f or f < 0:
                raise ValueError(f"keyframe frame {f!r} is not a non-negative integer")
            frames.append(int(f))
            ses.append(torch.as_tensor(se, dtype=torch.float32).detach().reshape(-1).cpu())
        if any(b < a for a, b in zip(frames, frames[1:])):
            raise ValueError(f"keyframe frames must not decrease: {frames}")
        if any(s_.numel() != ses[0].numel() for s_ in ses):
            raise ValueError("keyframe embeddings differ in size")
        self.frames = np.asarray(frames, dtype=np.int64)
        self.se = torch.stack(ses).contiguous()          # [K, gin]

    def dense(self, T: int, frame0: int = 0) -> torch.Tensor:
        """[1, gin, T] float32 (host): the embedding at frames frame0 .. frame0 + T - 1."""
        kf, kse = self.frames, self.se.numpy()
        t = np.arange(frame0, frame0 + T, dtype=np.int64)
        hi = np.searchsorted(kf, t, side="right")                  # first key with frame > t
        lo = np.clip(hi - 1, 0, len(kf) - 1)
        nx = np.clip(hi, 0, len(kf) - 1)
        inner = (hi > 0) & (hi < len(kf))
        span = np.where(inner, kf[nx] - kf[lo], 1).astype(np.float32)
        u = np.where(inner, (t - kf[lo]).astype(np.float32) / span, np.float32(0)).astype(np.float32)
        a, b = kse[lo], kse[nx]                                     # [T, gin]
        out = np.where(inner[:, None], a + u[:, None] * (b - a), a).astype(np.float32)
        return torch.from_numpy(np.ascontiguousarray(out.T))[None]


def _take(side, idx):
    """Items ``idx`` of a ``ToneColorConverter._se_items`` result (tensor rows or list entries)."""
    return [side[i] for i in idx] if isinstance(side, list) else side[idx]


def is_per_frame_se(se, gin: Optional[int] = None) -> bool:
    """Whether ``se`` (an embedding or a per-item sequence of them) varies over time: a ToneTrack or a [n, gin, T]
    tensor with T > 1.  Without ``gin`` any [n, C, T] with C > 1 and T > 1 counts, so a [1, 1, gin] row vector stays
    one embedding per item, as it always was."""
    if isinstance(se, (list, tuple)):
        return any(is_per_frame_se(x, gin) for x in se)
    if isinstance(se, ToneTrack):
        return True
    if not torch.is_tensor(se) or se.dim() != 3 or se.shape[-1] <= 1:
        return False
    return se.shape[-2] == gin if gin is not None else se.shape[-2] > 1


def pack_tone_keys(entries, frame0: Sequence[int], frames: Sequence[int], what: str = "embedding",
                   clip: Optional[int] = None):
    """Keyframes for ``ovc_tone_track_expand`` of items whose embeddings are ``entries``: a [gin] tensor (one
    embedding), a [gin, T] tensor (per frame over the item's whole clip, T == ``clip``, default frames[b]) or a
    ``ToneTrack``; item b is read at frames frame0[b] .. frame0[b] + frames[b] - 1.  Returns (key_frame [K] int64,
    key_se [K, gin] float32, key0 [B], nkeys [B]), all on the host.

    Only the keys a window can read are packed: a per-frame tensor gives one key per frame of the window (a key at
    every integer frame reproduces the values exactly), a track its keys from the last one at or before the window's
    first frame to the first one after its last frame.  Items that read the same keys share them.  So K is at most the
    windows' frames plus a few keys per track, whatever the clip's length or the track's history."""
    key_frame, key_se, key0, nkeys, seen = [], [], [], [], {}
    for b, e in enumerate(entries):
        f0, n = int(frame0[b]), int(frames[b])
        if isinstance(e, ToneTrack):
            kf = e.frames
            k0 = max(0, int(np.searchsorted(kf, f0, side="right")) - 1)
            k1 = min(len(kf), int(np.searchsorted(kf, f0 + n - 1, side="right")) + 1)
            tag = (id(e), k0, k1)
            if tag not in seen:
                seen[tag] = (len(key_frame), k1 - k0)
                key_frame.extend(kf[k0:k1].tolist())
                key_se.append(e.se[k0:k1])
        elif e.dim() == 2:
            want = n if clip is None else clip
            if e.shape[1] != want:
                raise ValueError(f"{what}: item {b} has {want} frames but its per-frame embedding {e.shape[1]}")
            tag = (id(e), f0, n)
            if tag not in seen:
                seen[tag] = (len(key_frame), n)
                key_frame.extend(range(f0, f0 + n))
                key_se.append(e[:, f0:f0 + n].T)
        else:
            tag = (id(e),)
            if tag not in seen:
                seen[tag] = (len(key_frame), 1)
                key_frame.append(0)
                key_se.append(e.reshape(1, -1))
        key0.append(seen[tag][0])
        nkeys.append(seen[tag][1])
    ks = torch.cat([k.detach().to(torch.float32).cpu() for k in key_se], 0).contiguous()
    return np.asarray(key_frame, dtype=np.int64), ks, key0, nkeys


def expand_tone_keys(native, entries, frame0, frames, Tmax: int, out=None, what: str = "embedding",
                     clip: Optional[int] = None):
    """The per-frame [B, gin, Tmax] embedding of ``entries`` (``pack_tone_keys``), expanded on the device by the
    tone-track kernel into ``out`` when given (zeros past each item's frames)."""
    dev = torch.device("cuda", native.device_index)
    kf, ks, key0, nkeys = pack_tone_keys(entries, frame0, frames, what, clip)
    i64 = lambda v: torch.as_tensor(np.asarray(v, dtype=np.int64)).to(dev)  # noqa: E731
    return native.tone_track_expand(i64(kf), ks.to(dev), i64(key0), i64(nkeys), i64(list(frame0)), i64(list(frames)),
                                    Tmax, out=out)


def check_seeds(seeds, n: int, what: str = "seeds") -> Optional[List[int]]:
    """Per-item Philox keys: None, or ``n`` integers in [0, 2^64).  ValueError otherwise (before any launch)."""
    if seeds is None:
        return None
    seeds = list(seeds)
    if len(seeds) != n:
        raise ValueError(f"{len(seeds)} {what} for {n} items")
    for i, s in enumerate(seeds):
        if isinstance(s, (bool, np.bool_)) or not isinstance(s, (int, np.integer)) or not 0 <= int(s) < 2 ** 64:
            raise ValueError(f"{what}[{i}] = {s!r} is not an integer in [0, 2^64)")
    return [int(s) for s in seeds]


def check_per_item(value, n: int, what: str, positive: bool = False) -> Tuple[float, Optional[List[float]]]:
    """A sampling parameter given as one float for all items or one per item: returns (scalar, None) or
    (first value, per-item list).  A per-item sequence of the wrong length, or a non-finite value (non-positive with
    ``positive``), raises ValueError (before any launch)."""
    if np.ndim(value) == 0:
        return float(value), None
    vals = [float(v) for v in value]
    if len(vals) != n:
        raise ValueError(f"{len(vals)} values of {what} for {n} items")
    for i, v in enumerate(vals):
        if not math.isfinite(v) or (positive and not v > 0):
            raise ValueError(f"{what}[{i}] = {v!r} is not {'a positive' if positive else 'a finite'} number")
    return (vals[0] if vals else 0.0), vals


def seed_array(seeds: Sequence[int]) -> np.ndarray:
    """int64 array holding the uint64 bit patterns of ``seeds`` (the device arrays of ovc_item_params.seed)."""
    return np.asarray([int(s) & (2 ** 64 - 1) for s in seeds], dtype=np.uint64).view(np.int64)


def _load_audio(src: AudioLike, sr: int) -> np.ndarray:
    """Stand-in for ``librosa.load(path, sr=sr)`` (openvoice/api.py:144): mono float32 at ``sr``.
    Uses librosa when it is installed; otherwise .npy (already at ``sr``) and PCM/float .wav via
    scipy, with polyphase resampling (not bit-identical to librosa's resampler -- third-party
    arithmetic the reference does not pin, SURVEY.md section 8c)."""
    if isinstance(src, np.ndarray):
        return np.ascontiguousarray(src, dtype=np.float32).reshape(-1)
    if src.endswith(".npy"):
        return np.ascontiguousarray(np.load(src), dtype=np.float32).reshape(-1)
    try:
        import librosa  # type: ignore
        return librosa.load(src, sr=sr)[0].astype(np.float32)
    except ImportError:
        pass
    from scipy.io import wavfile
    from scipy.signal import resample_poly
    file_sr, data = wavfile.read(src)
    if data.dtype.kind == "i":
        data = data.astype(np.float32) / float(np.iinfo(data.dtype).max + 1)
    elif data.dtype.kind == "u":
        data = (data.astype(np.float32) - 128.0) / 128.0
    data = data.astype(np.float32)
    if data.ndim == 2:
        data = data.mean(axis=1)
    if sr is not None and file_sr != sr:   # sr=None keeps the file's rate (librosa.load(sr=None))
        from math import gcd
        g = gcd(int(file_sr), int(sr))
        data = resample_poly(data, sr // g, file_sr // g).astype(np.float32)
    return np.ascontiguousarray(data)


def _write_audio(path: str, audio: np.ndarray, sr: int) -> None:
    """Stand-in for ``soundfile.write`` (openvoice/api.py:160)."""
    if path.endswith(".npy"):
        np.save(path, audio)
        return
    try:
        import soundfile  # type: ignore
        soundfile.write(path, audio, sr)
    except ImportError:
        from scipy.io import wavfile
        wavfile.write(path, sr, audio.astype(np.float32))


# Padded-frame budget of one batched reference-encoder pass in extract_se / extract_se_batch.  The encoder's device
# workspace (ovc_reference_encoder) is two copies of its largest activation -- conv layer 1: 32 channels x ceil(T/2)
# rows x 257 columns, ~4.1 k floats per padded input frame -- plus the GRU inputs (384 floats per 64 frames):
# 32 768 padded frames (~6 min of audio at 22.05 kHz, hop 256) take 2 * 4112 * 32768 * 4 B ~= 1.1 GB, which the
# context keeps for reuse.  A pass of that size already gives its first conv ~1.3e8 output threads.
SE_CHUNK_FRAMES = 32768


def plan_se_chunks(frames: Sequence[int], budget: int = SE_CHUNK_FRAMES) -> List[List[int]]:
    """Group clips of ``frames[i]`` spectrogram frames into batches of one reference-encoder pass each.  Clips are
    taken longest first; a chunk is closed when one more clip would take (clips x longest) over ``budget`` padded
    frames, so a clip longer than the budget runs alone.  Returns lists of clip indices covering every clip once."""
    order = sorted(range(len(frames)), key=lambda i: -int(frames[i]))
    chunks: List[List[int]] = []
    for i in order:
        if chunks and (len(chunks[-1]) + 1) * int(frames[chunks[-1][0]]) <= budget:
            chunks[-1].append(i)
        else:
            chunks.append([i])
    return chunks


# Receptive field of the TTS decode in frames, per direction.  After the expansion, which is pointwise in time, it runs
# the flow in reverse and the generator.  Flow: 4 couplings x a WaveNet of 4 layers with k = 5, dilation 1, i.e. +-2 per
# layer, +-8 per coupling, +-32 in all.  Generator: +-13.3 frames (conv_pre k = 7, the transposed convs, ResBlocks up to
# k = 11 d = 5; ToneColorConverter.HALO_FRAMES).  That is +-45.3 frames; 64 leaves margin.  There is no enc_q and no
# forward flow here, so this is about half of HALO_FRAMES.
TTS_HALO_FRAMES = 64

# Range of the length scale a duration fit may choose (include/ovc.h: ovc_tts_fit): speed 4x down to 0.25x.
FIT_SCALE_RANGE = (0.25, 4.0)


def plan_tts_windows(frames: int, first_window: int, window: int, halo: int) -> List[Tuple[int, int, int, int]]:
    """Windows of one sentence of ``frames`` decoded frames: (lo, hi, e0, e1) with decoded span [lo, hi) and interior
    [e0, e1).  The first interior has ``first_window`` frames and the others ``window`` (the last may be shorter); the
    interiors cover [0, frames) once and in order; lo = max(0, e0 - halo) and hi = min(frames, e1 + halo)."""
    frames, first_window, window, halo = int(frames), int(first_window), int(window), int(halo)
    if frames < 1 or first_window < 1 or window < 1 or halo < 0:
        raise ValueError(f"plan_tts_windows needs frames, first_window, window >= 1 and halo >= 0 (got {frames}, "
                         f"{first_window}, {window}, {halo})")
    out, e0 = [], 0
    while e0 < frames:
        e1 = min(frames, e0 + (first_window if e0 == 0 else window))
        out.append((max(0, e0 - halo), min(frames, e1 + halo), e0, e1))
        e0 = e1
    return out


def plan_clone(frames: Sequence[int], owner: Sequence[int], speeds: Sequence[float], hop: int,
               sr: int) -> Tuple[List[List[Tuple[int, int, int]]], List[int]]:
    """Layout of each request's utterance as ``BaseSpeakerTTS.tts_batch`` joins it (``audio_numpy_concat``): sentence
    i (a row of the TTS decode, owned by request ``owner[i]``) contributes its ``hop * frames[i]`` samples, then
    ``int(sr * 0.05 / speed)`` zeros.  Returns per request the runs (src_row, src_off, count) in order (src_row -1: zeros)
    and its length in samples."""
    runs: List[List[Tuple[int, int, int]]] = [[] for _ in speeds]
    for i, r in enumerate(owner):
        runs[r] += [(i, 0, int(hop) * int(frames[i])), (-1, 0, int((sr * 0.05) / speeds[r]))]
    return runs, [sum(n for _, _, n in rr) for rr in runs]


def splice_table(runs: Sequence[Sequence[Tuple[int, int, int]]], pitch: int) -> np.ndarray:
    """``ovc_splice`` segments [S, 5] that write item b's runs back to back into row b of a [len(runs), pitch] buffer,
    and zeros from its end to the row's end."""
    segs = []
    for b, rr in enumerate(runs):
        at = 0
        for row, off, n in rr:
            if n:
                segs.append((row, off, n, b, at))
                at += n
        if at < pitch:
            segs.append((-1, 0, pitch - at, b, at))
    return np.asarray(segs, dtype=np.int64).reshape(-1, 5)


class TtsState(NamedTuple):
    """Encode state of ``NativeSynthesizer.tts_encode``, owned by the caller: device tensors stats [N,T,2*inter],
    cum [N,T] int32, g [N,gin] ([N,gin,T] after a per-token encode) and y_lengths [N], each row's decoded frames (host), and the decode key, stream and
    noise scale ``infer`` would draw each row's prior noise with."""
    stats: torch.Tensor
    cum: torch.Tensor
    g: torch.Tensor
    y_lengths: torch.Tensor
    frames: List[int]
    dec_keys: List[int]
    dec_streams: List[int]
    dec_noise_scale: List[float]
    length_scale: Optional[List[float]] = None     # each row's length scale, after an encode with fit groups


def fit_groups(fit, B: int, device) -> Optional[tuple]:
    """The ``fit`` argument of ``NativeSynthesizer.tts_encode`` / ``infer_ragged`` as ``_native`` takes it: groups
    ``[(row0, row1, target_frames), ...]`` of rows [row0, row1) in increasing order that do not overlap, each with a
    target of at least 1 frame.  None or [] -> None (an encode without fit groups).  ValueError for anything else."""
    if not fit:
        return None
    fit = [tuple(int(v) for v in f) for f in fit]
    end = 0
    for i, f in enumerate(fit):
        if len(f) != 3:
            raise ValueError(f"fit group {i}: expected (row0, row1, target_frames), got {f}")
        r0, r1, target = f
        if not end <= r0 < r1 <= B:
            raise ValueError(f"fit group {i}: rows [{r0}, {r1}) must be non-empty, inside [0, {B}) and after the "
                             f"previous group's rows")
        if target < 1:
            raise ValueError(f"fit group {i}: target of {target} frames (at least 1)")
        end = r1
    cols = [torch.tensor(c, dtype=torch.int64, device=device) for c in zip(*fit)]
    return (*cols, *FIT_SCALE_RANGE)


class TtsPool:
    """Encode state shared by the sentences of many live requests: device tensors stats [N,Tp,2*inter], cum [N,Tp] int32,
    g [N,gin] and y_lengths [N], grown on demand and never shrunk.  ``NativeSynthesizer.tts_encode(..., pool=, rows=)``
    writes an encode's rows into any rows of it (include/ovc.h: ovc_tts_encode_state_rows); a larger token pitch
    re-pitches the rows already there once, with the library's padding.  The owner tracks which rows are live.

    Once a per-token encode is written into it, the pool holds g per token, [N,gin,Tp], for good (``to_per_token``):
    the rows already there keep their vector in every token column, later rows with one vector get it in every column,
    and its windows decode through ovc_tts_decode_windows_tokens (bit-identical for a constant row)."""

    def __init__(self, native, device):
        self.native, self.device = native, torch.device(device)
        self.N = self.Tp = 0
        self.stats = self.cum = self.g = self.y_lengths = None
        self.per_token = False

    def to_per_token(self) -> None:
        """Hold g per token from now on; each row's vector fills its token columns."""
        if self.per_token:
            return
        self.per_token = True
        if self.N:
            self.g = self.g[:, :, None].expand(-1, -1, self.Tp).contiguous()

    def fit(self, N: int, T: int) -> None:
        """At least ``N`` rows at a pitch of at least ``T`` tokens; the rows already held keep their contents."""
        if N <= self.N and T <= self.Tp:
            return
        N2 = max(int(N), self.N + self.N // 2) if N > self.N else self.N
        Tp2 = -(-max(int(T), self.Tp) // 16) * 16
        hp, dev = self.native.hp, self.device
        stats = torch.zeros(N2, Tp2, 2 * hp.inter_channels, device=dev)
        cum = torch.zeros(N2, Tp2, dtype=torch.int32, device=dev)
        g = torch.zeros(N2, hp.gin_channels, *((Tp2,) if self.per_token else ()), device=dev)
        y_lengths = torch.zeros(N2, dtype=torch.int64, device=dev)
        if self.N:
            self.native.tts_state_rows(range(self.N), stats, cum, g, y_lengths,
                                       src=(self.stats, self.cum, self.g, self.y_lengths))
        self.stats, self.cum, self.g, self.y_lengths, self.N, self.Tp = stats, cum, g, y_lengths, N2, Tp2


_POOL = None


def _pool():
    """Host-side staging threads: copying the utterances into / out of the pinned buffers is plain memcpy work (numpy
    releases the GIL for it) that sits inside every end-to-end call."""
    global _POOL
    if _POOL is None:
        from concurrent.futures import ThreadPoolExecutor
        try:
            n = len(os.sched_getaffinity(0))
        except Exception:
            n = os.cpu_count() or 1
        _POOL = ThreadPoolExecutor(max_workers=max(1, min(8, n)), thread_name_prefix="ovc-stage")
    return _POOL


def _parallel(fn, n, min_items=4):
    if n < min_items:
        return [fn(i) for i in range(n)]
    return list(_pool().map(fn, range(n)))


def watermark_device(audio, payload_bits, model, chunk: int = 16000, stride: int = 32000):
    """On-device chunking of openvoice/api.py:162-184.  ``audio``: 1-D float32 tensor (any device), modified in place;
    ``payload_bits``: flat 0/1 array, 32 per chunk.  Chunk n = samples [n * stride, n * stride + chunk); as in the
    reference the walk stops at the first chunk that does not fit ("Audio too short").  All full chunks are gathered
    by a strided view (no copy), encoded by ONE batched ``model.encode([m, chunk], [m, 32])`` call and scattered back."""
    n_repeat = len(payload_bits) // 32
    L = int(audio.shape[0])
    m = 0
    while m < n_repeat and m * stride + chunk <= L:
        m += 1
    if m < n_repeat:
        print("Audio too short, fail to add watermark")
    if m == 0:
        return audio
    with torch.no_grad():
        view = torch.as_strided(audio, (m, chunk), (stride, 1))
        bits = torch.as_tensor(np.asarray(payload_bits[: 32 * m], dtype=np.float32).reshape(m, 32), device=audio.device)
        enc = model.encode(view.contiguous(), bits).detach().reshape(m, chunk).to(audio.dtype)
        view.copy_(enc)
    return audio


class NativeSynthesizer:
    """Stands where ``SynthesizerTrn`` stands in the reference (``converter.model``) for the
    ``n_speakers == 0`` converter (openvoice/models.py:399-465): ``voice_conversion``,
    ``ref_enc``, ``load_state_dict``, ``eval``, ``zero_g``."""

    def __init__(self, hps, device: str, precision: Optional[str] = None):
        """``precision``: arithmetic of the generator's ResBlock / upsampling convolutions --
        ``"f16x3"`` (default; split-precision fp16 on the tensor cores (wgmma), fp32-grade),
        ``"fp32"`` (CUDA-core FFMA everywhere) or ``"f16"`` (single-pass fp16: the 11-bit operand precision the
        reference itself gets on a GPU through cuDNN's allow_tf32 default; ~1e-2).  Env override: OVC_PRECISION."""
        dev = torch.device(device)
        if dev.type != "cuda":
            raise RuntimeError("openvoice_b200 runs on CUDA (sm_90a) only; there is no CPU path")
        self.device = dev
        self.hps = hps
        self.zero_g = bool(getattr(hps.model, "zero_g", False))
        self.n_speakers = int(getattr(hps.data, "n_speakers", 0))
        index = dev.index if dev.index is not None else torch.cuda.current_device()
        self.native = NativeConverter(hps, index)
        self.precision = precision or os.environ.get("OVC_PRECISION", "f16x3")
        self.native.set_precision(self.precision)
        self.spec_channels = hps.data.filter_length // 2 + 1
        self.ref_enc = ReferenceEncoder(self.native, self.spec_channels, int(getattr(hps.model, "gin_channels", 256)))
        # n_speakers == 0: converter (ReferenceEncoder); > 0: V1 base speaker (enc_p / dp / sdp / emb_g), models.py:451-465
        self._expected = hot_path_keys(hps) + (ref_enc_keys() if self.n_speakers == 0 else tts_keys(hps))

    # nn.Module-ish surface used by callers of the reference
    def eval(self):
        return self

    def to(self, device):
        if torch.device(device) != self.device and torch.device(device).type != "cuda":
            raise RuntimeError("CUDA only")
        return self

    def load_state_dict(self, state_dict, strict: bool = False):
        """Returns (missing_keys, unexpected_keys) like torch with strict=False.  Unlike the
        reference, a checkpoint that lacks hot-path tensors is an error (the reference would
        silently keep random weights)."""
        provided = set(state_dict.keys())
        expected = set(self._expected)
        missing = sorted(expected - provided)
        unexpected = sorted(provided - expected)
        self.native.load_state_dict(state_dict)
        self.native.finalize()          # raises OvcError naming the first missing hot-path key
        self._state_dict = state_dict   # kept (by reference) so that per-stream replicas can be built on demand
        if strict and (missing or unexpected):
            raise RuntimeError(f"missing keys {missing}, unexpected keys {unexpected}")
        return missing, unexpected

    @torch.no_grad()
    def voice_conversion(self, y, y_lengths, sid_src, sid_tgt, tau: float = 1.0, noise=None,
                         ragged: bool = False, seed: Optional[int] = None, latents: bool = True,
                         seeds: Optional[Sequence[int]] = None, taus: Optional[Sequence[float]] = None,
                         frame0: Optional[Sequence[int]] = None, streams: Optional[Sequence[int]] = None):
        """(o_hat, y_mask, (z, z_p, z_hat)) = SynthesizerTrn.voice_conversion
        (openvoice/models.py:492-499).  ``noise`` ([B,192,T]) replaces the reference's
        ``randn_like``; when None, Philox normals are drawn in-kernel from ``seed`` (default: a
        draw from torch's global CPU generator, so ``torch.manual_seed`` makes runs repeatable).
        ``ragged=True`` converts every item at its exact length (what ``convert`` does).  ``sid_src`` / ``sid_tgt`` may
        each be per item ([B or 1, gin(, 1)]) or per frame ([B or 1, gin, T]), as in the reference.

        Per-item sampling (include/ovc.h: ovc_item_params): ``seeds`` gives item b its own Philox key, drawn at stream
        ``streams[b]`` (default 0 for every item: a request's own noise, independent of its batch index) and frame
        ``frame0[b] + t`` (default 0: ``frame0`` places a window of a longer clip at its absolute frames); ``taus``
        one tau per item.  Without ``seeds`` the call's seed keys every item at stream b, as before.  A seed with
        ``noise``, a length that is not B, a non-finite tau, a seed outside [0, 2^64) or a frame counter past 2^32
        raises ValueError."""
        B, _, T = y.shape
        seeds = check_seeds(seeds, B)
        taus = check_per_item(taus, B, "taus")[1] if taus is not None else None
        if noise is not None and seeds is not None:
            raise ValueError("pass either noise or seeds, not both")
        f0 = None if frame0 is None else [int(v) for v in frame0]
        if f0 is not None and (len(f0) != B or any(v < 0 or v + T > 2 ** 32 for v in f0)):
            raise ValueError(f"frame0 needs {B} values with 0 <= frame0 and frame0 + {T} <= 2^32")
        st_ = None if streams is None else [int(v) for v in streams]
        if st_ is not None and (len(st_) != B or any(not 0 <= v < 2 ** 32 for v in st_)):
            raise ValueError(f"streams needs {B} values in [0, 2^32)")
        y = y.to(self.device, torch.float32).contiguous()
        y_lengths = y_lengths.to(self.device, torch.int64).contiguous()
        sid_src = self._expand_se(sid_src, B, T)
        sid_tgt = self._expand_se(sid_tgt, B, T)
        if noise is None and seed is None:
            seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        if noise is not None:
            noise = noise.to(self.device, torch.float32)
        items = None
        if seeds is not None or taus is not None or f0 is not None or st_ is not None:
            dev = self.device
            if seeds is not None and st_ is None:
                st_ = [0] * B
            items = {
                "seed": None if seeds is None else torch.from_numpy(seed_array(seeds)).to(dev),
                "stream": None if st_ is None else torch.tensor(st_, dtype=torch.int64, device=dev),
                "frame0": None if f0 is None else torch.tensor(f0, dtype=torch.int64, device=dev),
                "tau": None if taus is None else torch.tensor(taus, dtype=torch.float32, device=dev),
            }
        o, lat = self.native.voice_conversion(y, y_lengths, sid_src, sid_tgt, noise=noise, tau=float(tau),
                                              seed=seed or 0, ragged=ragged, latents=latents, items=items)
        y_mask = (torch.arange(T, device=self.device)[None, :] < y_lengths[:, None]).unsqueeze(1).to(torch.float32)
        return o, y_mask, lat

    @torch.no_grad()
    def infer(self, x, x_lengths, sid=None, noise_scale=1, length_scale=1, noise_scale_w=1.0, sdp_ratio=0.2,
              max_len=None, noise_w=None, noise=None, ragged: bool = False, seed: Optional[int] = None,
              latents: bool = True, seeds: Optional[Sequence[int]] = None, streams: Optional[Sequence[int]] = None,
              g=None):
        """(o, attn, y_mask, (z, z_p, None, None)) = SynthesizerTrn.infer (openvoice/models.py:467-490) for a V1
        base-speaker checkpoint.  ``x`` [B,T] token ids, ``x_lengths`` [B], ``sid`` [B] speaker ids.
        ``noise_w`` ([B,2,T]) / ``noise`` ([B,192,>=Ty]) replace the two random draws (models.py:173, 487); when None,
        Philox normals are drawn in-kernel from ``seed``.  The expanded m_p / logs_p of the reference's return
        tuple are not materialised (they only feed z_p).  One host sync, where the reference has one too
        (y_lengths sizes every later tensor, models.py:476-478).

        Per-item sampling (include/ovc.h: ovc_item_params): ``noise_scale``, ``length_scale``, ``noise_scale_w`` and
        ``sdp_ratio`` each take one value per item as well as a scalar; ``seeds`` gives item b its own key (the
        duration noise draws from ``seeds[b]``, the prior noise from ``seeds[b] + 1``, as a scalar ``seed`` does) at
        stream ``streams[b]`` (default: b).  Sentence j of a call with ``seed=s`` is reproduced in any batch by
        ``seeds[i] = s, streams[i] = j`` and the same parameters.

        ``g`` replaces ``sid`` with speaker vectors (include/ovc.h: ovc_tts_encode_g): [B or 1, gin(, 1)] one per row
        (e.g. a blend of ``BaseSpeakerTTS.style`` rows), or [B or 1, gin, T] one per token.  Per token, the duration
        predictors read token t's vector and the flow and generator read, at frame y, the vector of the token that
        covers y (0 past the row's frames), as m_p is expanded."""
        a = self._tts_args(x, x_lengths, sid, noise_scale, length_scale, noise_scale_w, sdp_ratio, seed, seeds, streams, g)
        x, x_lengths, sid, seed, B = a["x"], a["x_lengths"], a["sid"], a["seed"], a["B"]
        noise_scale, enc_items, dec_items = a["noise_scale"], a["enc_items"], a["dec_items"]
        if noise_w is not None:
            noise_w = noise_w.to(self.device, torch.float32)
        y_lengths, w_ceil, _ = self.native.tts_encode(x, x_lengths, sid, noise_w=noise_w, seed=seed, items=enc_items,
                                                      g=a["g"], **a["enc_scalars"])
        Ty = int(y_lengths.max().item())                       # the sync
        if noise is not None:
            noise = noise.to(self.device, torch.float32)[:, :, :Ty].contiguous()
        o, lat = self.native.tts_decode(B, Ty, self.device, noise=noise, seed=seed + 1, noise_scale=float(noise_scale),
                                        ragged=ragged, latents=latents, max_len=max_len, items=dec_items)
        ar = torch.arange(Ty, device=self.device)
        y_mask = (ar[None, :] < y_lengths[:, None]).unsqueeze(1).to(torch.float32)
        cum = torch.cumsum(w_ceil, 1)                          # commons.generate_path (commons.py:128-142)
        path = (ar[None, :, None] < cum[:, None, :]) & (ar[None, :, None] >= (cum - w_ceil)[:, None, :])
        attn = (path.to(torch.float32) * y_mask.transpose(1, 2)).unsqueeze(1)      # [B,1,Ty,T]
        z, z_p = lat if lat else (None, None)
        return o, attn, y_mask, (z, z_p, None, None)

    @torch.no_grad()
    def infer_ragged(self, x, x_lengths, sid=None, noise_scale=1, length_scale=1, noise_scale_w=1.0, sdp_ratio=0.2,
                     seed: Optional[int] = None, seeds: Optional[Sequence[int]] = None,
                     streams: Optional[Sequence[int]] = None, g=None, fit=None) -> Tuple[torch.Tensor, List[int]]:
        """The audio of ``infer(..., ragged=True, latents=False)`` (same arguments and draws) left on the device, with
        each row's decoded frames on the host: (o [B, hop * max(frames)], frames).  Row b's samples are
        o[b, : hop * frames[b]], zeros after.  One host sync (y_lengths), as in ``infer``.  ``fit`` as in
        ``tts_encode``."""
        a = self._tts_args(x, x_lengths, sid, noise_scale, length_scale, noise_scale_w, sdp_ratio, seed, seeds, streams, g)
        y_lengths = self.native.tts_encode(a["x"], a["x_lengths"], a["sid"], seed=a["seed"], items=a["enc_items"],
                                           g=a["g"], fit=fit_groups(fit, a["B"], self.device), **a["enc_scalars"])[0]
        frames = [int(v) for v in y_lengths.cpu()]             # the sync
        o, _ = self.native.tts_decode(a["B"], max(frames), self.device, seed=a["seed"] + 1,
                                      noise_scale=float(a["noise_scale"]), ragged=True, latents=False,
                                      items=a["dec_items"])
        return o[:, 0], frames

    def check_tts_input(self, x, sid, need_sid: bool = True):
        """The token and speaker checks of ``infer`` / ``tts_encode``, before anything is launched: RuntimeError for a
        checkpoint without the TTS half, ValueError for a token id outside [0, n_vocab), a missing ``sid`` or a speaker id
        outside [0, n_speakers).  ``x``: int64 token ids (any shape, at least one); returns ``sid`` as a flat int64
        tensor, or None without ``need_sid`` (speaker vectors given instead)."""
        info = self.native.tts_info()
        if not info["has_tts"]:
            raise RuntimeError("this checkpoint has no enc_p / dp / sdp / emb_g: infer() needs a V1 base speaker")
        if int(x.min()) < 0 or int(x.max()) >= info["n_vocab"]:
            raise ValueError(f"token ids must lie in [0, {info['n_vocab']})")
        if not need_sid:
            return None
        if sid is None:
            raise ValueError("sid is required (n_speakers > 0)")
        sid = sid.to(torch.int64).reshape(-1)
        if int(sid.min()) < 0 or int(sid.max()) >= info["n_speakers"]:
            raise ValueError(f"speaker ids must lie in [0, {info['n_speakers']})")
        return sid

    def check_tts_g(self, g, B: int, T: int) -> torch.Tensor:
        """Speaker vectors for ``infer(g=...)`` as the library takes them: [B, gin] (one per row) or [B, gin, T] (one per
        token; only a 3-D tensor with more than one column is per token).  A batch of 1 serves every row.  ValueError
        for any other shape, before anything is launched."""
        gin = self.native.hp.gin_channels
        g = torch.as_tensor(g).to(self.device, torch.float32)
        per_token = g.dim() == 3 and g.shape[-1] > 1
        if per_token and (g.shape[1] != gin or g.shape[2] != T):
            raise ValueError(f"per-token speaker vectors must be [B, {gin}, {T}] (gin, tokens), got {tuple(g.shape)}")
        if not per_token:
            if g.dim() not in (2, 3) or g.shape[1] != gin or g.numel() != g.shape[0] * gin:
                raise ValueError(f"speaker vectors must be [B, {gin}] or [B, {gin}, 1], got {tuple(g.shape)}")
            g = g.reshape(g.shape[0], gin)
        if g.shape[0] == 1 and B > 1:
            g = g.expand(B, *g.shape[1:])
        if g.shape[0] != B:
            raise ValueError(f"speaker vectors for {g.shape[0]} rows, the batch has {B}")
        return g.contiguous()

    def _tts_args(self, x, x_lengths, sid, noise_scale, length_scale, noise_scale_w, sdp_ratio, seed, seeds, streams,
                  g=None):
        """The checks and device inputs ``infer`` and ``tts_encode`` share: validated tokens, lengths and speakers (ids,
        or vectors ``g``) on the device, the call's key, the per-item parameter arrays of both halves, and each row's
        decode key, stream and noise scale as host lists (what the whole decode draws row b with)."""
        x = x.to(torch.int64)
        if g is None:
            sid = self.check_tts_input(x, sid)
        else:
            sid = self.check_tts_input(x, None, need_sid=False)
            g = self.check_tts_g(g, x.shape[0], x.shape[1])
        x = x.to(self.device).contiguous()
        B, T = x.shape
        x_lengths = x_lengths.to(self.device, torch.int64).contiguous()
        sid = sid.to(self.device).contiguous() if sid is not None else None
        seeds = check_seeds(seeds, B)
        if streams is not None:
            streams = [int(v) for v in streams]
            if len(streams) != B or any(not 0 <= v < 2 ** 32 for v in streams):
                raise ValueError(f"streams needs {B} values in [0, 2^32)")
        noise_scale, ns_b = check_per_item(noise_scale, B, "noise_scale")
        length_scale, ls_b = check_per_item(length_scale, B, "length_scale", positive=True)
        noise_scale_w, nsw_b = check_per_item(noise_scale_w, B, "noise_scale_w")
        sdp_ratio, sr_b = check_per_item(sdp_ratio, B, "sdp_ratio")
        if seed is None:
            seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        dev = self.device
        f32 = lambda v: None if v is None else torch.tensor(v, dtype=torch.float32, device=dev)  # noqa: E731
        key = None if seeds is None else torch.from_numpy(seed_array(seeds)).to(dev)
        key1 = None if seeds is None else torch.from_numpy(seed_array([s + 1 for s in seeds])).to(dev)
        stream_d = None if streams is None else torch.tensor(streams, dtype=torch.int64, device=dev)
        enc_items = dec_items = None
        if any(v is not None for v in (seeds, streams, nsw_b, ls_b, sr_b, ns_b)):
            enc_items = {"seed": key, "stream": stream_d, "noise_scale_w": f32(nsw_b), "length_scale": f32(ls_b),
                         "sdp_ratio": f32(sr_b)}
            dec_items = {"seed": key1, "stream": stream_d, "noise_scale": f32(ns_b)}
        return dict(x=x, x_lengths=x_lengths, sid=sid, g=g, seed=seed, B=B, noise_scale=noise_scale, enc_items=enc_items,
                    dec_items=dec_items,
                    enc_scalars=dict(noise_scale_w=float(noise_scale_w), length_scale=float(length_scale),
                                     sdp_ratio=float(sdp_ratio)),
                    dec_keys=[(seed if seeds is None else seeds[b]) + 1 for b in range(B)],
                    dec_streams=list(range(B)) if streams is None else streams,
                    dec_noise_scale=[noise_scale] * B if ns_b is None else ns_b)

    @torch.no_grad()
    def tts_encode(self, x, x_lengths, sid=None, noise_scale=1, length_scale=1, noise_scale_w=1.0, sdp_ratio=0.2,
                   seed: Optional[int] = None, seeds: Optional[Sequence[int]] = None,
                   streams: Optional[Sequence[int]] = None, pool: Optional["TtsPool"] = None,
                   rows: Optional[Sequence[int]] = None, g=None, fit=None) -> "TtsState":
        """The encode half of ``infer`` (same arguments and draws), returning state the caller owns: a later
        ``tts_encode`` or ``infer`` does not change it.  ``tts_decode_windows`` decodes any frames of its rows, each
        row with the decode key, stream and noise scale ``infer`` would give it.  One host sync (y_lengths), as in
        ``infer``.

        ``pool`` / ``rows``: encoded row b is written into row ``rows[b]`` of ``pool`` instead (one
        ``ovc_tts_encode_state_rows``; the pool grows to fit first).  The returned state then holds the pool's tensors,
        and its host lists (frames, decode keys, streams, noise scales) describe the encoded rows in order.

        ``g`` as in ``infer``.  With per-token vectors the state's g is [B, gin, T] (include/ovc.h:
        ovc_tts_encode_state_tokens), and a pool turns per-token (``TtsPool.to_per_token``).  Into a per-token pool,
        rows with one vector (or a speaker id) are encoded with it in every token column, which gives the same
        values.

        ``fit``: ``[(row0, row1, target_frames), ...]``, runs of rows whose frames are fitted to a target (include/ovc.h:
        ovc_tts_encode_fit): every row of a group is encoded at the smallest length scale s in ``FIT_SCALE_RANGE``
        whose group frames sum_r max(1, sum_t ceil(exp(logw_r[t]) * s)) reach the target (the range's top when none
        does), exactly as an encode given s as the row's ``length_scale``.  Rows outside every group keep their
        ``length_scale``.  The state's ``length_scale`` then lists each row's scale."""
        a = self._tts_args(x, x_lengths, sid, noise_scale, length_scale, noise_scale_w, sdp_ratio, seed, seeds, streams, g)
        x = a["x"]
        B, T = x.shape
        per_token = a["g"] is not None and a["g"].dim() == 3
        if pool is not None and (per_token or pool.per_token):
            if not per_token:
                vec = a["g"]
                if vec is None:
                    vec = self._state_dict["emb_g.weight"].to(self.device, torch.float32)[a["sid"]]
                a["g"] = vec[:, :, None].expand(-1, -1, T).contiguous()
                per_token = True
            pool.to_per_token()
        if pool is not None:
            rows = [int(r) for r in rows]
            if len(rows) != B or min(rows) < 0:
                raise ValueError(f"tts_encode: {len(rows)} pool rows for {B} encoded rows (each >= 0)")
            pool.fit(max(rows) + 1, T)
        groups = fit_groups(fit, B, self.device)
        enc = self.native.tts_encode(x, a["x_lengths"], a["sid"], seed=a["seed"], items=a["enc_items"], g=a["g"],
                                     fit=groups, **a["enc_scalars"])
        y_lengths = enc[0]
        if pool is None:
            stats, cum, g = self.native.tts_encode_state(B, T, self.device, per_token=per_token)
        else:
            stats, cum, g, _ = self.native.tts_state_rows(rows, pool.stats, pool.cum, pool.g, pool.y_lengths)
        frames = [int(v) for v in y_lengths.cpu()]             # the sync
        scales = enc[3].cpu().tolist() if groups is not None else None
        return TtsState(stats, cum, g, y_lengths if pool is None else pool.y_lengths, frames, a["dec_keys"],
                        a["dec_streams"], a["dec_noise_scale"], scales)

    @torch.no_grad()
    def tts_decode_windows(self, state: "TtsState", windows: Sequence[Tuple[int, int, int]], w_max: Optional[int] = None,
                           latents: bool = False, slot: int = 0):
        """Decode ``windows`` = [(row, frame0, length)] of ``state`` in ONE call (include/ovc.h: ovc_tts_decode_windows):
        window i holds frames [frame0, frame0 + length) of its row.  Returns (o [W, hop * w_max] on the device, z_p
        [W, inter, w_max] or None); window i's samples are o[i, : hop * length], and ``o`` lives in slot ``slot``'s buffer
        until the next call on that slot.  ``w_max`` defaults to the longest window.  A row outside the state, a negative
        offset, a length < 1, a window past its row's end, or a w_max shorter than a window raises ValueError before
        anything is launched."""
        windows = [tuple(int(v) for v in w) for w in windows]
        if not windows:
            raise ValueError("tts_decode_windows needs at least one window")
        n = len(state.frames)
        for i, (r, f0, ln) in enumerate(windows):
            if not 0 <= r < n:
                raise ValueError(f"window {i}: row {r} outside [0, {n})")
            if f0 < 0 or ln < 1 or f0 + ln > state.frames[r]:
                raise ValueError(f"window {i}: frames [{f0}, {f0 + ln}) are not inside row {r}'s {state.frames[r]} frames")
        w_max = max(ln for _, _, ln in windows) if w_max is None else int(w_max)
        if w_max < max(ln for _, _, ln in windows):
            raise ValueError(f"w_max {w_max} is shorter than the longest window")
        rows = [r for r, _, _ in windows]
        return self.native.tts_decode_windows(
            state.stats, state.cum, state.g, state.y_lengths, rows, [f0 for _, f0, _ in windows],
            [ln for _, _, ln in windows], [state.dec_keys[r] for r in rows], [state.dec_streams[r] for r in rows],
            [state.dec_noise_scale[r] for r in rows], w_max, latents=latents, slot=slot)

    def _expand_se(self, se, B, T=1):
        """[B, gin] (per item) or [B, gin, T] (per frame) on the device; a batch of 1 serves every item."""
        se = se.to(self.device, torch.float32)
        per_frame = is_per_frame_se(se, self.native.hp.gin_channels)
        if per_frame and se.shape[-1] != T:
            raise ValueError(f"per-frame speaker embedding has {se.shape[-1]} frames, the batch {T}")
        se = se if per_frame else se.reshape(se.shape[0], -1)
        if se.shape[0] == 1 and B > 1:
            se = se.expand(B, *se.shape[1:])
        if se.shape[0] != B:
            raise ValueError(f"speaker embedding batch {se.shape[0]} does not match batch {B}")
        return se.contiguous()


class OpenVoiceBaseClass(object):
    """openvoice/api.py:14-39."""

    def __init__(self, config_path, device="cuda:0", precision=None):
        if "cuda" in device:
            assert torch.cuda.is_available()
        hps = utils.get_hparams_from_file(config_path)
        self.model = NativeSynthesizer(hps, device, precision=precision).eval()
        self.hps = hps
        self.device = device

    def load_ckpt(self, ckpt_path):
        checkpoint_dict = torch.load(ckpt_path, map_location=torch.device("cpu"))
        a, b = self.model.load_state_dict(checkpoint_dict["model"], strict=False)
        print("Loaded checkpoint '{}'".format(ckpt_path))
        print("missing/unexpected keys:", a, b)


class BaseSpeakerTTS(OpenVoiceBaseClass):
    """openvoice/api.py:42-98: the V1 base speaker.  The acoustic model (``SynthesizerTrn.infer``) runs on the
    CUDA library; the text front end (sentence splitting, cleaners, G2P: openvoice/text/*, utils.split_sentence)
    is host-side string processing outside this build's scope (SURVEY.md section 8), so it is pluggable:
    ``text_frontend(text, language_mark) -> list of token-id lists`` (one per sentence, blanks already
    interspersed).  When the reference package is importable its own front end is used."""

    language_marks = {"english": "EN", "chinese": "ZH"}

    def __init__(self, *args, text_frontend=None, **kwargs):
        super().__init__(*args, **kwargs)
        self.text_frontend = text_frontend

    @staticmethod
    def intersperse(lst, item):
        """commons.intersperse (openvoice/commons.py:22-25): [a, b] -> [item, a, item, b, item]."""
        out = [item] * (len(lst) * 2 + 1)
        out[1::2] = lst
        return out

    @staticmethod
    def audio_numpy_concat(segment_data_list, sr, speed=1.0):
        """openvoice/api.py:56-63: sentences joined with 50 ms / speed of silence after each."""
        gap = np.zeros(int((sr * 0.05) / speed), dtype=np.float32)
        parts = []
        for seg in segment_data_list:
            parts += [np.asarray(seg, dtype=np.float32).reshape(-1), gap]
        return np.concatenate(parts) if parts else np.zeros(0, np.float32)

    def _reference_frontend(self, text, mark):
        try:
            import re
            from openvoice import utils as ref_utils          # type: ignore
            from openvoice.text import text_to_sequence      # type: ignore
        except ImportError as e:
            raise RuntimeError("no text front end: pass text_frontend=... to BaseSpeakerTTS, call tts_from_ids(), or "
                               "install the reference package for its cleaners") from e
        seqs = []
        for t in ref_utils.split_sentence(text, language_str=mark):              # api.py:66-71
            t = re.sub(r"([a-z])([A-Z])", r"\1 \2", t)                           # api.py:81
            ids = text_to_sequence(f"[{mark}]{t}[{mark}]", self.hps.symbols, self.hps.data.text_cleaners)
            if getattr(self.hps.data, "add_blank", False):
                ids = self.intersperse(ids, 0)                                   # api.py:50-52
            seqs.append(ids)
        return seqs

    def _sentences(self, text, language):
        mark = self.language_marks.get(language.lower(), None)
        assert mark is not None, f"language {language} is not supported"
        frontend = self.text_frontend or self._reference_frontend
        return frontend(text, mark)

    def tokenize(self, text, language="English") -> List[List[int]]:
        """The token-id lists (one per sentence, blanks included) that ``tts`` / ``tts_batch`` synthesise for ``text``:
        where a per-token speaker places its keys.  Sentence j's tokens sit at positions [o_j, o_j + len(ids_j)) of the
        request's token stream, o_j the earlier sentences' token count."""
        return [list(q) for q in self._sentences(text, language)]

    def style(self, name_or_id) -> torch.Tensor:
        """The speaker vector [gin] (float32, host) of a style of the checkpoint, by name (``hps.speakers``, e.g.
        "cheerful") or id: the emb_g row ``speaker=name_or_id`` conditions with.  Blends are tensor arithmetic, e.g.
        ``speaker=0.7 * tts.style("cheerful") + 0.3 * tts.style("default")``."""
        return self._emb_g()[self._speaker_id(name_or_id, "style")].clone()

    def _emb_g(self) -> torch.Tensor:
        return self.model._state_dict["emb_g.weight"].detach().to("cpu", torch.float32)

    def _speaker_id(self, spk, who: str) -> int:
        """A style name or id as an emb_g row; ValueError for an unknown name or an id outside the table."""
        if isinstance(spk, str):
            names = self.hps.get("speakers", {})
            if spk not in names:
                raise ValueError(f"{who}: unknown style {spk!r} (the checkpoint has {sorted(names)})")
            return int(names[spk])
        n = int(self.hps.data.n_speakers)
        if not 0 <= int(spk) < n:
            raise ValueError(f"{who}: speaker id {spk!r} is not in [0, {n})")
        return int(spk)

    def _speaker(self, spk, who: str):
        """A request's ``speaker``: (id, None) for a name or an id (an id is range-checked by the encode, as before),
        else (None, entry) with entry a [gin] vector, a ``ToneTrack`` over token positions or a [gin, N] per-token
        tensor (host, float32).  ValueError names ``who``."""
        if isinstance(spk, str):
            return self._speaker_id(spk, who), None
        gin = int(self.hps.model.gin_channels)
        if isinstance(spk, ToneTrack):
            if spk.se.shape[1] != gin:
                raise ValueError(f"{who}: the ToneTrack's embeddings have {spk.se.shape[1]} values, the model's {gin}")
            return None, spk
        if not (torch.is_tensor(spk) or isinstance(spk, np.ndarray)) or np.ndim(spk) == 0:
            return int(spk), None
        e = torch.as_tensor(spk).detach().to("cpu", torch.float32)
        if e.dim() == 3 and e.shape[0] == 1 and e.shape[1] == gin and e.shape[2] > 1:
            return None, e[0].contiguous()
        if e.numel() != gin:
            raise ValueError(f"{who}: speaker embedding of shape {tuple(e.shape)} is not [{gin}], [1, {gin}, 1] or "
                             f"[1, {gin}, N] (N = the request's tokens)")
        return None, e.reshape(gin)

    def _speaker_rows(self, rows, T: int) -> Optional[torch.Tensor]:
        """Speaker vectors for sentences ``rows`` = [(id, entry, offset, tokens)] (``_speaker``; offset = o_j): None
        when every row names an id (the emb_g path), [n, gin] when each has one vector, else [n, gin, T] per token
        (zero past each sentence).  Per token, sentence j reads the ToneTrack at positions o_j + t
        (``ToneTrack.dense``) or columns [o_j, o_j + n_j) of a per-token tensor; an id or a vector fills its row."""
        if all(e is None for _, e, _, _ in rows):
            return None
        table = self._emb_g()
        for i, e, _, _ in rows:
            if e is None and not 0 <= i < table.shape[0]:       # the ids ride as emb_g rows: the encode's own check
                raise ValueError(f"speaker ids must lie in [0, {table.shape[0]})")
        vec = lambda i, e: table[i] if e is None else e  # noqa: E731
        if not any(isinstance(e, ToneTrack) or (e is not None and e.dim() == 2) for _, e, _, _ in rows):
            return torch.stack([vec(i, e) for i, e, _, _ in rows]).contiguous()
        g = torch.zeros(len(rows), table.shape[1], T)
        for b, (i, e, o, n) in enumerate(rows):
            if isinstance(e, ToneTrack):
                g[b, :, :n] = e.dense(n, o)[0]
            elif e is not None and e.dim() == 2:
                g[b, :, :n] = e[:, o:o + n]
            else:
                g[b, :, :n] = vec(i, e)[:, None]
        return g

    @torch.no_grad()
    def tts_batch(self, requests: Sequence[dict]) -> List[np.ndarray]:
        """Many TTS requests in ONE ragged ``infer``, each with its own speaker, speed, seed and noise parameters.
        A request is a dict: ``ids`` (list of token-id lists, one per sentence) or ``text`` (+ ``language``, default
        "English", through the text front end), ``speaker``, and optionally ``speed`` (1.0), ``seed`` (default: one
        drawn from torch's global generator), ``noise_scale`` (0.667), ``noise_scale_w`` (0.6), ``sdp_ratio`` (0.2).
        Sentence j of request r draws at (seed_r, stream j) with request r's parameters, so each returned array equals
        ``audio_numpy_concat(tts_from_ids(ids, speaker, speed=..., seed=seed_r, ...), sr, speed)`` bit for bit: the
        sentences joined with 50 ms / speed gaps, as ``tts`` does.  Returns one array per request.

        ``duration`` (seconds) fits the request to that length: its sentences are one fit group (``fit_target``) whose
        length scale the encode solves on the device, and ``speed`` then only sets the gaps.  The array has at least
        round(duration * sr) samples, and less than one hop more unless two tokens change length at the same scale or
        the scale reaches an end of ``FIT_SCALE_RANGE``."""
        reqs = list(requests)
        seqs, sid, owner, speeds, kw = self._request_sentences(reqs)
        sr = self.hps.data.sampling_rate
        audio = self._infer_sentences(seqs, sid, **kw) if seqs else []
        per: List[List[np.ndarray]] = [[] for _ in reqs]
        for r, a in zip(owner, audio):
            per[r].append(a)
        return [self.audio_numpy_concat(per[r], sr=sr, speed=speeds[r]) for r in range(len(reqs))]

    def _request_sentences(self, reqs):
        """The sentences of ``tts_batch`` requests: (token-id lists, speaker ids, owning request, each request's speed,
        the per-sentence ``infer`` keywords).  Sentence j of request r is keyed (seed_r, stream j) with r's parameters.
        When a request's speaker is an embedding or a track, the keywords carry ``g`` (``_speaker_rows``) for every
        sentence and the speaker ids are placeholders."""
        seqs, sid, seeds, streams, owner, rows = [], [], [], [], [], []
        par = {"noise_scale": [], "noise_scale_w": [], "length_scale": [], "sdp_ratio": []}
        speeds, fit = [], []
        for r, q in enumerate(reqs):
            ids = [list(q_ids) for q_ids in (q["ids"] if "ids" in q else self._sentences(q["text"], q.get("language", "English")))]
            k = self._request_keys(q, f"request {r}")
            self._check_speaker_tokens(k["g"], [len(q_ids) for q_ids in ids], f"request {r}")
            speeds.append(k["speed"])
            if k["duration"] is not None and ids:
                target = self.fit_target(k["duration"], len(ids), k["speed"], True, f"request {r}")
                fit.append((len(seqs), len(seqs) + len(ids), target))
            o = 0
            for j, q_ids in enumerate(ids):
                seqs.append(q_ids)
                sid.append(0 if k["speaker"] is None else k["speaker"])
                rows.append((k["speaker"], k["g"], o, len(q_ids)))
                o += len(q_ids)
                seeds.append(k["seed"])
                streams.append(j)
                owner.append(r)
                self._sentence_params(k, par)
        kw = dict(seeds=seeds, streams=streams, **par)
        if fit:
            kw["fit"] = fit
        g = self._speaker_rows(rows, max((len(q) for q in seqs), default=1))
        if g is not None:
            kw["g"] = g
        return seqs, sid, owner, speeds, kw

    @staticmethod
    def _check_speaker_tokens(entry, lengths: Sequence[int], who: str) -> None:
        """ValueError when a per-token speaker tensor's columns are not the request's token count."""
        if torch.is_tensor(entry) and entry.dim() == 2 and entry.shape[1] != sum(lengths):
            raise ValueError(f"{who}: the per-token speaker tensor has {entry.shape[1]} columns, the request "
                             f"{sum(lengths)} tokens")

    def _request_keys(self, q, who: str) -> dict:
        """The TTS keys of one request (all but its text), validated: speaker (``speaker``: an id or None; ``g``: None
        or the embedding / track, ``_speaker``), speed, seed (drawn from torch's generator when absent) and the noise
        parameters.  ValueError names the request as ``who``."""
        spk, g = self._speaker(q["speaker"], who)
        speed = float(q.get("speed", 1.0))
        if not (math.isfinite(speed) and speed > 0):
            raise ValueError(f"{who}: speed {speed!r} must be a positive number")
        duration = self._check_duration(q.get("duration"), who)
        seed = q.get("seed")
        seed = int(torch.randint(0, 2 ** 62, (1,)).item()) if seed is None else check_seeds([seed], 1, "seed")[0]
        return dict(speaker=spk, g=g, speed=speed, seed=seed, noise_scale=float(q.get("noise_scale", 0.667)),
                    noise_scale_w=float(q.get("noise_scale_w", 0.6)), sdp_ratio=float(q.get("sdp_ratio", 0.2)),
                    duration=duration)

    @staticmethod
    def _check_duration(duration, who: str) -> Optional[float]:
        if duration is None:
            return None
        duration = float(duration)
        if not (math.isfinite(duration) and duration > 0):
            raise ValueError(f"{who}: duration {duration!r} must be a positive number of seconds")
        return duration

    def fit_target(self, duration: float, n: int, speed: float, gaps: bool, who: str) -> int:
        """Frames F* that ``n`` sentences must fill to last ``duration`` seconds: ceil((N* - gaps) / hop), N* =
        round(duration * sr) samples and gaps = n * int(sr * 0.05 / speed), the silences ``audio_numpy_concat`` appends
        (0 without ``gaps``).  ValueError naming ``who`` when that leaves less than one frame per sentence."""
        sr, hop = int(self.hps.data.sampling_rate), int(self.hps.data.hop_length)
        total = int(round(duration * sr))
        silence = n * int((sr * 0.05) / speed) if gaps else 0
        target = -(-(total - silence) // hop)
        if target < n:
            raise ValueError(f"{who}: duration {duration} s is too short for {n} sentence(s): it needs more than "
                             f"{(silence + (n - 1) * hop) / sr:.4f} s (the gaps and one {hop}-sample frame per sentence)")
        return target

    @staticmethod
    def _sentence_params(k: dict, par: dict) -> None:
        """Append one sentence's ``infer`` parameters, for a request with keys ``k`` (``_request_keys``), to ``par``."""
        par["noise_scale"].append(k["noise_scale"])
        par["noise_scale_w"].append(k["noise_scale_w"])
        par["length_scale"].append(1.0 / k["speed"])
        par["sdp_ratio"].append(k["sdp_ratio"])

    @staticmethod
    def _pad_ids(sequences):
        """Token-id lists -> (x [n, T] int64 zero-padded, lengths [n])."""
        T = max(len(q) for q in sequences)
        x = torch.zeros(len(sequences), T, dtype=torch.int64)
        for i, q in enumerate(sequences):
            x[i, :len(q)] = torch.as_tensor(q, dtype=torch.int64)
        return x, torch.tensor([len(q) for q in sequences], dtype=torch.int64)

    def tts_stream_batch(self, requests: Sequence[dict], window_frames: int = 256,
                         first_window_frames: int = 32) -> Iterator[Tuple[int, np.ndarray]]:
        """Streaming ``tts_batch``: yields ``(request_index, chunk)`` as the audio is decoded, so playback can start after
        the first window instead of after the whole utterance.  Requests are the dicts ``tts_batch`` takes; all their
        sentences share ONE encode.  Each step is ONE ``NativeSynthesizer.tts_decode_windows`` call over the next window
        of every unfinished request and yields one chunk per such request, in request order.  A request's sentences are
        decoded in order: the first sentence in windows of ``first_window_frames`` then ``window_frames`` frames, the
        others in windows of ``window_frames``, each decoded with ``TTS_HALO_FRAMES`` frames of context on both sides
        (``plan_tts_windows``); a sentence's last chunk ends with its 50 ms / speed of silence.  A ``duration`` key fits
        the request as in ``tts_batch``.  A request's chunks
        concatenate to ``tts_batch``'s array for it (same length, same gaps) within fp32 reordering (2e-6 of its rms),
        whatever requests it is batched with.  Malformed requests (an empty one, a speed <= 0, a bad seed) or window
        sizes < 1 raise ValueError here, before anything is launched."""
        window_frames, first_window_frames = int(window_frames), int(first_window_frames)
        if window_frames < 1 or first_window_frames < 1:
            raise ValueError(f"window_frames ({window_frames}) and first_window_frames ({first_window_frames}) must be >= 1")
        reqs = list(requests)
        seqs, sid, owner, speeds, kw = self._request_sentences(reqs)
        for r in range(len(reqs)):
            if r not in owner:
                raise ValueError(f"request {r} has no sentences")
        return self._stream(seqs, sid, owner, speeds, kw, window_frames, first_window_frames)

    @torch.no_grad()
    def _stream(self, seqs, sid, owner, speeds, kw, window_frames, first_window_frames):
        if not seqs:
            return
        x, lens = self._pad_ids(seqs)
        state = self.model.tts_encode(x, lens, sid=torch.as_tensor(sid, dtype=torch.int64), **kw)
        sr, hop = self.hps.data.sampling_rate, self.hps.data.hop_length
        # per request: its windows in order, (row, lo, hi, e0, e1, silence after the chunk)
        plans: List[List[Tuple[int, int, int, int, int, int]]] = [[] for _ in speeds]
        for i, r in enumerate(owner):
            first = first_window_frames if not plans[r] else window_frames
            wins = plan_tts_windows(state.frames[i], first, window_frames, TTS_HALO_FRAMES)
            gap = int((sr * 0.05) / speeds[r])
            plans[r] += [(i, lo, hi, e0, e1, gap if k == len(wins) - 1 else 0) for k, (lo, hi, e0, e1) in enumerate(wins)]
        for step in range(max(len(p) for p in plans)):
            live = [(r, p[step]) for r, p in enumerate(plans) if step < len(p)]
            o, _ = self.model.tts_decode_windows(state, [(i, lo, hi - lo) for _, (i, lo, hi, _, _, _) in live])
            host = o.cpu().numpy()
            for k, (r, (_, lo, _, e0, e1, gap)) in enumerate(live):
                chunk = host[k, (e0 - lo) * hop: (e1 - lo) * hop]
                yield r, np.concatenate([chunk, np.zeros(gap, np.float32)]) if gap else chunk.copy()

    def tts_stream(self, text=None, speaker=None, language="English", speed=1.0, seed: Optional[int] = None, ids=None,
                   window_frames: int = 256, first_window_frames: int = 32,
                   duration: Optional[float] = None) -> Iterator[np.ndarray]:
        """``tts`` as a stream of float32 chunks (``tts_stream_batch`` with one request): the first chunk is
        ``first_window_frames`` frames of audio, available once the encode and one small decode have run.  ``ids``
        (token-id lists, one per sentence) replaces ``text``.  The chunks concatenate to ``tts(text, None, speaker,
        language, speed, seed)`` within 2e-6 of its rms, with the same length and the same silences.  Feeding them to
        ``streaming.StreamingConverter.push`` gives cloned-voice streaming.  ``duration`` as in ``tts``."""
        q = dict(speaker=speaker, speed=speed, seed=seed, duration=duration)
        q.update({"ids": ids} if ids is not None else {"text": text, "language": language})
        gen = self.tts_stream_batch([q], window_frames=window_frames, first_window_frames=first_window_frames)
        return (chunk for _, chunk in gen)

    def _infer_sentences(self, sequences, sid, **kw) -> List[np.ndarray]:
        """One ragged infer over token-id lists with per-sentence speaker ids; each sentence's samples."""
        x, lens = self._pad_ids(sequences)
        o, frames = self.model.infer_ragged(x, lens, sid=torch.as_tensor(sid, dtype=torch.int64), **kw)
        o = o.cpu().numpy()
        hop = self.hps.data.hop_length
        return [o[i, : frames[i] * hop].copy() for i in range(len(sequences))]

    @torch.no_grad()
    def tts_from_ids(self, sequences, speaker, speed=1.0, noise_scale=0.667, noise_scale_w=0.6, sdp_ratio=0.2,
                     seed: Optional[int] = None, duration: Optional[float] = None) -> List[np.ndarray]:
        """All sentences in ONE batched infer() (the reference loops over them at batch 1, api.py:79-91); every
        sentence gets what its own batch-1 call would give (ragged decode).  ``seed``: the call's key (sentence j
        draws at stream j); default: one drawn from torch's global generator.  ``speaker``: a style name or id, a
        speaker vector ([gin] or [1, gin, 1], e.g. a blend of ``style`` rows), a ``ToneTrack`` keyed in token positions
        of the whole call (sentence j's tokens at [o_j, o_j + n_j)) or a [1, gin, N] per-token tensor with N the
        call's token count; ValueError for anything else.  ``duration`` (seconds of speech: the sentences are returned
        without gaps) fits all the sentences as one group, as ``tts_batch`` does, and replaces ``speed``."""
        return self._from_ids(sequences, speaker, speed, noise_scale, noise_scale_w, sdp_ratio, seed, duration, False)

    def _from_ids(self, sequences, speaker, speed, noise_scale, noise_scale_w, sdp_ratio, seed, duration, gaps):
        """``tts_from_ids``; a ``duration`` counts the gaps ``audio_numpy_concat`` adds when ``gaps`` is set."""
        duration = self._check_duration(duration, "duration")
        sequences = [list(q) for q in sequences]
        speaker_id, entry = self._speaker(speaker, "speaker")
        self._check_speaker_tokens(entry, [len(q) for q in sequences], "speaker")
        n = len(sequences)
        if n == 0:      # the reference's loop over zero sentences yields no audio (api.py:79-91)
            return []
        offs = np.cumsum([0] + [len(q) for q in sequences]).tolist()
        g = self._speaker_rows([(speaker_id, entry, offs[j], len(q)) for j, q in enumerate(sequences)],
                               max(len(q) for q in sequences))
        extra = {} if g is None else {"g": g}
        if duration is not None:
            extra["fit"] = [(0, n, self.fit_target(duration, n, speed, gaps, "duration"))]
        return self._infer_sentences(sequences, [0 if speaker_id is None else speaker_id] * n, noise_scale=noise_scale,
                                     noise_scale_w=noise_scale_w, length_scale=1.0 / speed, sdp_ratio=sdp_ratio, seed=seed,
                                     **extra)

    def tts(self, text, output_path, speaker, language="English", speed=1.0, seed: Optional[int] = None,
            duration: Optional[float] = None):
        """openvoice/api.py:73-98.  ``seed``: the request's key (``tts_from_ids``); same seed, same audio.
        ``duration`` (seconds, gaps included) fits the utterance as ``tts_batch`` does; ``speed`` then sets the gaps."""
        sequences = self._sentences(text, language)
        audio_list = self._from_ids(sequences, speaker, speed, 0.667, 0.6, 0.2, seed, duration, True)
        audio = self.audio_numpy_concat(audio_list, sr=self.hps.data.sampling_rate, speed=speed)
        if output_path is None:
            return audio
        _write_audio(output_path, audio, self.hps.data.sampling_rate)


class ToneColorConverter(OpenVoiceBaseClass):
    """openvoice/api.py:101-201."""

    def __init__(self, *args, **kwargs):
        enable_watermark = kwargs.pop("enable_watermark", True)
        super().__init__(*args, **kwargs)
        self.watermark_model = None
        if enable_watermark:
            # the reference fails hard at `import wavmark` (openvoice/api.py:105-107); silently returning
            # un-watermarked audio to a caller who asked for the watermark is worse than failing
            try:
                import wavmark  # type: ignore
            except ImportError as e:
                raise ImportError("ToneColorConverter(enable_watermark=True) needs the third-party `wavmark` package "
                                  "(openvoice/api.py:105-107); pass enable_watermark=False to convert without it") from e
            self.watermark_model = wavmark.load_model().to(self.device)
        self.version = getattr(self.hps, "_version_", "v1")

    # ------------------------------------------------------------------ speaker embedding
    def extract_se(self, ref_wav_list, se_save_path=None, sr: Optional[int] = None):
        """openvoice/api.py:114-139: mean ReferenceEncoder embedding over the given clips, shape [1, gin, 1].

        Every clip is encoded at its own length, exactly as the reference's per-clip loop does, but the clips share
        batched ("ragged") passes: sorted by length and grouped under ``SE_CHUNK_FRAMES`` padded frames, one upload,
        one ``ovc_spectrogram`` and one ``ovc_reference_encoder_ragged`` per group.  A clip's frames past its own
        length are never read, so its embedding does not depend on which clips it is grouped with: the result is
        bit-identical to encoding the clips one at a time.  The mean is taken over the clips in the caller's order.
        A clip shorter than one hop, or not longer than the STFT reflect padding (384 samples), raises ValueError
        naming it before anything is launched.  ``sr``: rate of NumPy waveform clips when it is not the model's; they
        are resampled on the device (see ``convert_batch``) and the length checks apply to the resampled clips."""
        if isinstance(ref_wav_list, (str, np.ndarray)):
            ref_wav_list = [ref_wav_list]
        rate = self._input_rate(ref_wav_list, sr)
        waves = [_load_audio(f, self.hps.data.sampling_rate) for f in ref_wav_list]
        gs = torch.stack(self._se_rows(waves, rate)).mean(0)
        self._save_se(gs, se_save_path)
        return gs

    def extract_se_batch(self, speakers, se_save_paths=None, sr: Optional[int] = None) -> List[torch.Tensor]:
        """Enrol many voices at once: ``speakers`` is a sequence whose items are each a list of reference clips or a
        single clip (path or waveform).  Returns one [1, gin, 1] embedding per speaker, each bit-identical to
        ``extract_se(speakers[i])``; the clips of all speakers share the same batched passes (see ``extract_se``).
        ``se_save_paths``: one path (or None) per speaker, written like ``extract_se``'s ``se_save_path``; ``sr`` as in
        ``extract_se``."""
        groups = [[s] if isinstance(s, (str, np.ndarray)) else list(s) for s in speakers]
        if se_save_paths is not None and len(se_save_paths) != len(groups):
            raise ValueError(f"{len(se_save_paths)} save paths for {len(groups)} speakers")
        for i, g in enumerate(groups):
            if not g:
                raise ValueError(f"speaker {i} has no reference clips")
        clips = [f for g in groups for f in g]
        rate = self._input_rate(clips, sr)
        rows = self._se_rows([_load_audio(f, self.hps.data.sampling_rate) for f in clips], rate)
        out, k = [], 0
        for i, g in enumerate(groups):
            se = torch.stack(rows[k: k + len(g)]).mean(0)
            k += len(g)
            self._save_se(se, None if se_save_paths is None else se_save_paths[i])
            out.append(se)
        return out

    @staticmethod
    def _save_se(se, path):
        if path is not None:
            if os.path.dirname(path):
                os.makedirs(os.path.dirname(path), exist_ok=True)
            torch.save(se.cpu(), path)

    @torch.no_grad()
    def _se_rows(self, waves, sr: Optional[int] = None) -> List[torch.Tensor]:
        """ReferenceEncoder embedding [1, gin, 1] of every waveform, in order; see ``extract_se``.  ``sr``: the
        waveforms' rate when it is not the model's (``_input_rate``): each group is uploaded raw and resampled on the
        device."""
        hop = self.hps.data.hop_length
        pad = (self.hps.data.filter_length - hop) // 2
        lens = [self._resampled_len(len(w), sr) for w in waves]
        for i, n in enumerate(lens):           # what _enqueue_chunk refuses, checked before any launch
            if n < hop or n <= pad:
                raise ValueError(f"reference clip {i} has {n} samples{'' if sr is None else ' after resampling'}: needs "
                                 f"at least one hop ({hop}) and more than the STFT reflect padding ({pad})")
        dev, nat = self.device, self.model.native
        rows: List[Optional[torch.Tensor]] = [None] * len(waves)
        for idx in plan_se_chunks([n // hop for n in lens], SE_CHUNK_FRAMES):
            k, Lmax = len(idx), max(len(waves[i]) for i in idx)
            ev = self.__dict__.get("_se_h2d_done")
            if ev is not None:
                ev.synchronize()               # the previous chunk's upload has left the staging buffer
            stage = self._pinned("se_in", k * Lmax).view(k, Lmax)
            stage_np = stage.numpy()

            def put(b):
                w = waves[idx[b]]
                stage_np[b, : len(w)] = w
                stage_np[b, len(w):] = 0.0
            _parallel(put, k)
            wav = stage.to(dev, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(dev))
            self._se_h2d_done = ev
            wlen = torch.tensor([len(waves[i]) for i in idx], dtype=torch.int64).to(dev)
            if sr is not None:
                wav = nat.resample(wav, wlen, sr, self.hps.data.sampling_rate, out_pitch=max(lens[i] for i in idx))
                wlen = torch.tensor([lens[i] for i in idx], dtype=torch.int64).to(dev)
            spec, frames = nat.spectrogram(wav, wlen)                     # = spectrogram_torch (api.py:126-128)
            g = nat.reference_encoder(spec, frames)                        # = model.ref_enc per clip (api.py:130)
            for j, i in enumerate(idx):
                rows[i] = g[j: j + 1].unsqueeze(-1)
        return rows  # type: ignore[return-value]

    # ------------------------------------------------------------------ conversion
    def convert(self, audio_src_path, src_se, tgt_se, output_path=None, tau=0.3, message="default",
                noise=None, sr: Optional[int] = None, seed: Optional[int] = None):
        """openvoice/api.py:141-160.  Returns float32 samples (256 * (L // 256) of them) or writes
        ``output_path``.  ``noise`` ([1,192,T]) optionally replaces the random draw (tests).  ``sr``: rate of a NumPy
        waveform that is not at the model's rate (see ``convert_batch``).  ``seed``: the request's own noise key
        (see ``convert_batch``'s ``seeds``): the same seed reproduces the same audio in any batch, stream or window."""
        audio = self.convert_batch([audio_src_path], src_se, tgt_se, tau=tau, messages=[message],
                                   noise=None if noise is None else [noise], sr=sr,
                                   seeds=None if seed is None else [seed])[0]
        if output_path is None:
            return audio
        _write_audio(output_path, audio, self.hps.data.sampling_rate)

    @torch.no_grad()
    def convert_batch(self, audios: Sequence[AudioLike], src_se, tgt_se, tau: Union[float, Sequence[float]] = 0.3,
                      messages: Optional[Sequence[str]] = None, noise: Optional[Sequence] = None,
                      max_batch: int = 64, sr: Optional[int] = None,
                      seeds: Optional[Sequence[int]] = None) -> List[np.ndarray]:
        """Convert a list of utterances (paths or waveforms at the model sampling rate); every item
        gets exactly what ``convert`` would return for it alone.  ``src_se`` / ``tgt_se`` are either
        one [1,gin,1] embedding for all items or a sequence of per-item embeddings.  An embedding may vary over time:
        a ``ToneTrack`` or a [1, gin, T] tensor with T = the item's frames (samples // 256 at the model's rate), as the
        reference's ``voice_conversion`` takes; one [1, gin, T] for the whole call needs every item to have T frames.
        Items with a constant embedding convert exactly as they would alone.

        ``sr``: sampling rate of the NumPy waveform items when it is not the model's.  They are uploaded as they are
        and resampled on the device (``scipy.signal.resample_poly`` arithmetic, within one fp32 ulp of it) into the
        buffer the spectrogram reads; the output stays at the model's rate, as in the reference.  A file path item with
        ``sr`` is refused (files are decoded and resampled on load); so is a rate pair the resampler does not take.

        ``tau``: one value for all items or one per item.  ``seeds``: one Philox key per item, in [0, 2^64).  Item i
        then draws its noise from ``seeds[i]`` alone (include/ovc.h: ovc_item_params, stream 0), so its audio equals
        ``convert(audios[i], seed=seeds[i], tau=tau_i)`` bit for bit wherever it sits: batch order, ``max_batch``,
        ``convert_concurrent``, sharding.  Without ``seeds`` one key drawn from torch's global generator serves the
        call, as in the reference's ``randn_like``.  ``seeds`` with ``noise``, a length that is not ``len(audios)``
        or an invalid value raises ValueError before anything is launched."""
        hps = self.hps
        n = len(audios)
        tau, taus = check_per_item(tau, n, "tau")
        seeds = check_seeds(seeds, n)
        if noise is not None and seeds is not None:
            raise ValueError("pass either noise or seeds, not both")
        rate = self._input_rate(audios, sr)
        waves = [_load_audio(a, hps.data.sampling_rate) for a in audios]
        src = self._se_items(src_se, n, "src_se")
        tgt = self._se_items(tgt_se, n, "tgt_se")
        out: List[Optional[np.ndarray]] = [None] * n
        order = sorted(range(n), key=lambda i: -len(waves[i]))     # similar lengths share a launch
        hop = hps.data.hop_length
        for lo in range(0, n, max_batch):
            idx = order[lo: lo + max_batch]
            res = self._convert_chunk([waves[i] for i in idx], _take(src, idx), _take(tgt, idx),
                                      tau if taus is None else [taus[i] for i in idx],
                                      None if noise is None else [noise[i] for i in idx], rate,
                                      None if seeds is None else [seeds[i] for i in idx])
            for i, a in zip(idx, res):
                msg = messages[i] if messages is not None else "default"
                out[i] = self.add_watermark(a, msg)
        return out  # type: ignore[return-value]

    # ------------------------------------------------------------------ text to cloned voice
    def _clone_requests(self, tts, requests):
        """Validated ``clone_batch`` / ``clone_stream_batch`` requests, before anything is launched: the TTS sentences
        (``BaseSpeakerTTS._request_sentences``) and per request its embeddings (stacked [n, gin]), tau, conversion key
        and watermark message; the embeddings stay on the host.  ValueError for a request without sentences, a missing or mis-sized embedding, a tau
        that is not finite, a bad seed, or models on different devices."""
        reqs = list(requests)
        self._check_same_device(tts)
        seqs, sid, owner, speeds, kw = tts._request_sentences(reqs)
        ses = {"src_se": [], "tgt_se": []}
        taus, seeds, messages = [], [], []
        for r, q in enumerate(reqs):
            if r not in owner:
                raise ValueError(f"request {r} has no sentences")
            k = self._clone_keys(q, f"request {r}")
            for name in ses:
                ses[name].append(k[name])
            taus.append(k["tau"])
            seeds.append(k["convert_seed"])
            messages.append(k["message"])
        stack = {k: torch.cat(v, 0) if v else None for k, v in ses.items()}
        return (seqs, sid, owner, speeds, kw), stack["src_se"], stack["tgt_se"], taus, seeds, messages

    def _check_same_device(self, tts):
        if torch.device(tts.model.device) != torch.device(self.model.device):
            raise ValueError(f"the TTS model is on {tts.model.device} and the converter on {self.model.device}")

    def _clone_keys(self, q, who: str) -> dict:
        """The conversion keys of one clone request, validated: ``src_se`` / ``tgt_se`` ([1, gin] on the host), ``tau``,
        ``convert_seed`` (drawn from torch's generator when absent) and ``message``.  ValueError names it as ``who``."""
        gin = int(getattr(self.hps.model, "gin_channels", 256))
        out = {}
        for name in ("src_se", "tgt_se"):
            if q.get(name) is None:
                raise ValueError(f"{who} has no {name}")
            if isinstance(q[name], ToneTrack):
                raise ValueError(f"{who}: {name} is a ToneTrack; text to cloned voice takes one embedding per request")
            se = torch.as_tensor(q[name], dtype=torch.float32).reshape(1, -1)
            if se.shape[1] != gin:
                raise ValueError(f"{who}: {name} has {se.shape[1]} values, the converter's embeddings have {gin}")
            out[name] = se
        tau = float(q.get("tau", 0.3))
        if not math.isfinite(tau):
            raise ValueError(f"{who}: tau = {tau!r} is not a finite number")
        seed = q.get("convert_seed")
        out["tau"] = tau
        out["convert_seed"] = (int(torch.randint(0, 2 ** 62, (1,)).item()) if seed is None
                               else check_seeds([seed], 1, f"{who}: convert_seed")[0])
        out["message"] = q.get("message", "default")
        return out

    def _check_clone_lengths(self, lengths, rate, names: Optional[Sequence[str]] = None):
        """ValueError for an utterance ``convert`` would refuse: shorter than one hop or not past the STFT padding
        (after resampling from ``rate`` when it is given).  ``names[r]`` names utterance r (default "request r")."""
        hop = self.hps.data.hop_length
        pad = (self.hps.data.filter_length - hop) // 2
        for r, n in enumerate(lengths):
            m = self._resampled_len(n, rate)
            if m < hop or m <= pad:
                who = f"request {r}" if names is None else names[r]
                raise ValueError(f"{who}: its utterance has {m} samples{'' if rate is None else ' after resampling'}: "
                                 f"needs at least one hop ({hop}) and more than the STFT reflect padding ({pad})")

    @torch.no_grad()
    def clone_batch(self, tts: "BaseSpeakerTTS", requests: Sequence[dict], pcm16: bool = False,
                    max_batch: int = 64) -> List[np.ndarray]:
        """Text to cloned voice for many requests, joined on the device: what ``tts.tts(...)`` followed by
        ``convert(...)`` gives, without the audio leaving the GPU in between.  A request is a ``tts.tts_batch`` request
        dict plus ``src_se`` and ``tgt_se`` (required; [1, gin, 1] embeddings), ``tau`` (0.3), ``convert_seed`` (the
        conversion's key; default: drawn from torch's generator, as ``seed`` is) and ``message`` (watermark payload,
        applied on the host as ``convert_batch`` applies it).  A ``duration`` key fits the TTS half as ``tts_batch``
        does; the converted audio keeps ``convert``'s length, hop * floor(L / hop) for an utterance of L samples.

        One ragged TTS encode + decode of every sentence (one host sync, for the frame counts), then per chunk of
        ``max_batch`` requests (sorted by length, as ``convert_batch`` chunks) one ``ovc_splice`` that builds the
        utterances in the converter's input rows -- each sentence followed by int(sr * 0.05 / speed) zeros, as
        ``audio_numpy_concat`` joins them -- one ragged conversion with each request's embeddings, tau and key, and one
        download.  If the TTS model's rate is not the converter's, the joined rows are resampled on the device.

        Request r's array equals ``convert(tts.tts_batch([q])[0], q["src_se"], q["tgt_se"], tau=q["tau"],
        seed=q["convert_seed"], sr=tts_rate)`` bit for bit, whatever else is in the batch.  ``pcm16``: each TTS sample
        first takes the 16-bit PCM round trip of a wav file (include/ovc.h: OVC_SPLICE_PCM16), as when the TTS output is
        written to a 16-bit wav and converted from that file.  Malformed requests raise ValueError before any launch;
        an utterance too short to convert (a very high speed) raises it after the encode, before the conversion."""
        reqs = list(requests)
        (seqs, sid, owner, speeds, kw), src, tgt, taus, seeds, messages = self._clone_requests(tts, reqs)
        if not reqs:
            return []
        rate = self._input_rate([], int(tts.hps.data.sampling_rate))
        x, lens = tts._pad_ids(seqs)
        o, frames = tts.model.infer_ragged(x, lens, sid=torch.as_tensor(sid, dtype=torch.int64), **kw)
        runs, lengths = plan_clone(frames, owner, speeds, tts.hps.data.hop_length, int(tts.hps.data.sampling_rate))
        self._check_clone_lengths(lengths, rate)
        src, tgt = src.to(self.device), tgt.to(self.device)
        out: List[Optional[np.ndarray]] = [None] * len(reqs)
        order = sorted(range(len(reqs)), key=lambda i: -lengths[i])
        for lo in range(0, len(reqs), max_batch):
            idx = order[lo: lo + max_batch]

            def fill(rows, idx=idx):
                table = splice_table([runs[i] for i in idx], rows.shape[1])
                pin = self._pinned_i64("splice", table.size)
                pin.copy_(torch.from_numpy(table.reshape(-1)))
                seg = self._dev("splice", table.size, torch.int64)
                seg.copy_(pin, non_blocking=True)
                self.model.native.splice(o, seg.view(-1, 5), rows, pcm16=pcm16)
            res = self._convert_chunk([lengths[i] for i in idx], src[idx], tgt[idx], [taus[i] for i in idx], None,
                                      sr=rate, seeds=[seeds[i] for i in idx], fill=fill)
            for i, a in zip(idx, res):
                out[i] = self.add_watermark(a, messages[i])
        return out  # type: ignore[return-value]

    def clone_stream_batch(self, tts: "BaseSpeakerTTS", requests: Sequence[dict], window_frames: int = 256,
                           first_window_frames: int = 32) -> Iterator[Tuple[int, np.ndarray]]:
        """Streaming ``clone_batch`` (``pcm16=False``): yields ``(request_index, chunk)`` of cloned audio while the
        requests are still being synthesised.  Requests as in ``clone_batch``; the TTS encode of all their sentences
        runs here, so malformed requests and too-short utterances raise ValueError before the first step.

        Each request is a ``streaming.CloneSessions`` session that says all its sentences at once and ends: its
        ``window_frames``-frame converter windows use the request's embeddings, tau and ``convert_seed``.  A step is
        ``CloneSessions.step``, one batched launch sequence over every unfinished request: ONE ``tts_decode_windows``
        call decodes, per request, the next TTS windows (``plan_tts_windows``: ``first_window_frames`` then
        ``window_frames`` frames) until its converter can emit a window or its text is done; ONE ``ovc_splice`` writes
        the windows' interiors and the sentences' 50 ms / speed gaps into the converter's rings (a ``duration`` key is
        ``CloneSessions.say(duration=)``); then one ring
        spectrogram and ragged conversion of every ready window, and one download.  A request is closed in the step
        that writes its last gap.  Every step yields one non-empty chunk per unfinished request, in
        request order; a request's chunks concatenate to its ``clone_batch`` array (same length; the TTS windows equal
        the whole decode to fp32 reordering).  The models must share a sampling rate (ValueError otherwise)."""
        from .streaming import CloneSessions
        reqs = list(requests)
        cs = CloneSessions(self, tts, window_frames=window_frames, first_window_frames=first_window_frames,
                           label="request")
        (seqs, _, owner, speeds, kw), _, _, taus, seeds, _ = self._clone_requests(tts, reqs)
        if not reqs:
            return iter(())
        targets = {row0: target for row0, _, target in kw.get("fit", [])}
        for r, q in enumerate(reqs):                     # session r is request r, with the keys drawn above
            mine = [i for i, o in enumerate(owner) if o == r]
            keys = {k: q[k] for k in CloneSessions.OPEN_KEYS if k in q}
            keys.update(seed=kw["seeds"][mine[0]], convert_seed=seeds[r], tau=taus[r], speed=speeds[r])
            sid = cs.open(**keys)
            cs._queue(sid, [seqs[i] for i in mine], targets.get(mine[0]))   # checked by the encode below
            cs.end(sid)
        cs.encode_pending()
        return self._clone_stream(cs)

    @staticmethod
    def _clone_stream(cs):
        while cs.sessions:
            out = cs.step()
            for r in sorted(out):
                yield r, out[r]

    # ------------------------------------------------------------------ one utterance per stream
    @torch.no_grad()
    def convert_concurrent(self, audios: Sequence[AudioLike], src_se, tgt_se, tau: Union[float, Sequence[float]] = 0.3,
                           streams: int = 4, messages: Optional[Sequence[str]] = None, sr: Optional[int] = None,
                           seeds: Optional[Sequence[int]] = None) -> List[np.ndarray]:
        """Serve many SMALL independent requests: utterance i runs alone (batch 1, exactly ``convert``) on CUDA
        stream ``i % streams``, each stream with its own converter replica (context + workspace), so the
        latency-bound kernels of different requests overlap on the GPU -- north_star's "one utterance per stream".
        For large batches ``convert_batch`` (one launch sequence for the whole batch) is the faster path.  ``sr``,
        ``tau`` (scalar or per item) and ``seeds`` as in ``convert_batch``."""
        n = len(audios)
        tau, taus = check_per_item(tau, n, "tau")
        seeds = check_seeds(seeds, n)
        rate = self._input_rate(audios, sr)
        src = self._se_items(src_se, n, "src_se")
        tgt = self._se_items(tgt_se, n, "tgt_se")
        reps = self._replicas(max(1, min(streams, n)))
        S, depth = len(reps), 2                       # requests in flight per stream (pinned staging slots)
        out: List[Optional[np.ndarray]] = [None] * n
        for w0 in range(0, n, S * depth):
            wave = list(range(w0, min(n, w0 + S * depth)))
            pending = []
            for j, i in enumerate(wave):
                conv, stream = reps[j % S]
                with torch.cuda.stream(stream):
                    pending.append(conv._enqueue_single(_load_audio(audios[i], self.hps.data.sampling_rate), _take(src, [i]),
                                                        _take(tgt, [i]), tau if taus is None else taus[i], j // S, rate,
                                                        None if seeds is None else seeds[i]))
            for _, stream in reps:
                stream.synchronize()
            for i, (host, n_samples) in zip(wave, pending):
                msg = messages[i] if messages is not None else "default"
                out[i] = self.add_watermark(host[:n_samples].numpy().copy(), msg)
        return out  # type: ignore[return-value]

    def _replicas(self, count):
        """[(converter, stream)]: replica 0 is this object; the others share its hparams and checkpoint."""
        reps = self.__dict__.setdefault("_reps", [(self, torch.cuda.Stream(device=self.device))])
        while len(reps) < count:
            twin = ToneColorConverter.__new__(ToneColorConverter)
            twin.hps, twin.device, twin.watermark_model, twin.version = self.hps, self.device, None, self.version
            twin.model = NativeSynthesizer(self.hps, self.device, precision=self.model.precision)
            twin.model.load_state_dict(self.model._state_dict)
            reps.append((twin, torch.cuda.Stream(device=self.device)))
        return reps[:count]

    def _enqueue_single(self, wave, src, tgt, tau, slot, sr=None, seed=None):
        """Asynchronous batch-1 conversion on the current stream, staging through pinned slot ``slot``;
        returns (pinned host buffer, samples).  The caller synchronises the stream before reading / reusing it.
        ``sr``: the wave's rate when it is not the model's (``_input_rate``): resampled on the device after upload.
        ``seed``: the request's own key (stream 0), else one drawn from torch's global generator."""
        hop = self.hps.data.hop_length
        dev = self.device
        L = self._resampled_len(len(wave), sr)
        if L // hop < 1 or L <= (self.hps.data.filter_length - hop) // 2:
            raise ValueError("audio too short" if sr is None else f"audio too short: {L} samples after resampling")
        stage = self._pinned(f"cin{slot}", len(wave))
        stage.copy_(torch.from_numpy(wave))
        wav = stage.to(dev, non_blocking=True).view(1, len(wave))
        if sr is not None:
            wav = self.model.native.resample(wav, torch.tensor([len(wave)], dtype=torch.int64, device=dev), sr,
                                             self.hps.data.sampling_rate)
        wlen = torch.tensor([L], dtype=torch.int64, device=dev)
        items = None if seed is None else self._item_arrays(f"c{slot}", [seed], None)
        seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        src = self._se_device(src, [L // hop], [0], L // hop, "src_se")
        tgt = self._se_device(tgt, [L // hop], [0], L // hop, "tgt_se")
        o, _ = self.model.native.convert_waveform(wav, wlen, src, tgt, tau=float(tau), seed=seed, items=items)
        host = self._pinned(f"cout{slot}", o.numel())
        host.copy_(o.view(-1), non_blocking=True)
        return host, (L // hop) * hop

    # receptive field of the whole path in spectrogram frames: enc_q +-32 (16 WN layers of k=5), flow forward and
    # reverse +-32 each (4 couplings x 4 layers), generator +-13.3 (conv_pre 3, transposed convs, ResBlocks up to
    # k=11 d=5) -> 110; 128 leaves margin (SURVEY.md section 5 "long-context": measured ~109)
    HALO_FRAMES = 128

    @torch.no_grad()
    def convert_long(self, audio_src_path, src_se, tgt_se, output_path=None, tau=0.3, message="default",
                     window_frames: int = 2048, noise=None, max_batch: int = 32, sr: Optional[int] = None,
                     seed: Optional[int] = None):
        """Row f4 (time-tiled execution): convert a clip of any length with bounded memory.  The spectrogram is
        cut into windows of ``window_frames`` frames plus a halo of the path's receptive field on both sides; the
        windows run as one ragged batch and only their interiors are kept, so the result equals ``convert`` on the
        whole clip (same noise tensor: drawn once for the whole clip, or passed as ``noise`` [192, T]).  ``sr``: rate of
        a NumPy waveform that is not at the model's; it is resampled on the device first (see ``convert_batch``).
        ``seed``: the request's own key; each window then draws the whole clip's noise at its absolute frames in-kernel
        (frame0 = the window's first frame), so the result matches ``convert(seed=seed)`` and no noise tensor is
        built.  ``seed`` with ``noise`` raises ValueError.  ``src_se`` / ``tgt_se`` may vary over time (a ``ToneTrack``
        or [1, gin, T], as in ``convert_batch``): each window reads the whole clip's embedding at its absolute frames."""
        hps = self.hps
        seed = None if seed is None else check_seeds([seed], 1, "seed")[0]
        if seed is not None and noise is not None:
            raise ValueError("pass either noise or seed, not both")
        hop, dev = hps.data.hop_length, self.device
        rate = self._input_rate([audio_src_path], sr)
        wav = torch.from_numpy(_load_audio(audio_src_path, hps.data.sampling_rate)).to(dev)
        if rate is not None:
            wav = self.model.native.resample(wav[None].contiguous(), torch.tensor([wav.numel()], dtype=torch.int64, device=dev),
                                             rate, hps.data.sampling_rate)[0]
        L = wav.numel()
        spec, _ = self.model.native.spectrogram(wav[None].contiguous(), torch.tensor([L], dtype=torch.int64, device=dev))
        T = spec.shape[2]
        C = hps.model.inter_channels
        if seed is None:
            if noise is None:
                gen = torch.Generator(device=dev)
                gen.manual_seed(int(torch.randint(0, 2 ** 62, (1,)).item()))
                noise = torch.randn(C, T, device=dev, generator=gen)
            noise = noise.to(dev, torch.float32).reshape(C, T)
        H = self.HALO_FRAMES
        starts = list(range(0, T, window_frames))
        wins = [(max(0, s - H), min(T, s + window_frames + H), s, min(T, s + window_frames)) for s in starts]
        Wmax = max(hi - lo for lo, hi, _, _ in wins)
        out = torch.empty(T * hop, device=dev, dtype=torch.float32)
        src = self._se_items(src_se, 1, "src_se")
        tgt = self._se_items(tgt_se, 1, "tgt_se")
        for i0 in range(0, len(wins), max_batch):
            chunk = wins[i0: i0 + max_batch]
            B = len(chunk)
            sp = torch.zeros(B, spec.shape[1], Wmax, device=dev)
            nz = None if seed is not None else torch.zeros(B, C, Wmax, device=dev)
            for b, (lo, hi, _, _) in enumerate(chunk):
                sp[b, :, : hi - lo] = spec[0, :, lo:hi]
                if nz is not None:
                    nz[b, :, : hi - lo] = noise[:, lo:hi]
            lens = torch.tensor([hi - lo for lo, hi, _, _ in chunk], dtype=torch.int64, device=dev)
            keyed = {} if seed is None else dict(seeds=[seed] * B, frame0=[lo for lo, _, _, _ in chunk])
            f0s, fr = [lo for lo, _, _, _ in chunk], [hi - lo for lo, hi, _, _ in chunk]
            g_s = src.expand(B, -1) if not isinstance(src, list) else self._se_device(src * B, fr, f0s, Wmax, "src_se", clip=T)
            g_t = tgt.expand(B, -1) if not isinstance(tgt, list) else self._se_device(tgt * B, fr, f0s, Wmax, "tgt_se", clip=T)
            o, _, _ = self.model.voice_conversion(sp, lens, g_s, g_t, tau=tau, noise=nz,
                                                  ragged=True, latents=False, **keyed)
            for b, (lo, hi, s, e) in enumerate(chunk):
                out[s * hop: e * hop] = o[b, 0, (s - lo) * hop: (e - lo) * hop]
        audio = self.add_watermark(out.cpu().numpy(), message)
        if output_path is None:
            return audio
        _write_audio(output_path, audio, hps.data.sampling_rate)

    def _input_rate(self, audios, sr) -> Optional[int]:
        """The rate to resample the NumPy waveforms of ``audios`` from, or None when they are at the model's rate
        (``sr`` None or equal to it: the staging code is then exactly the one without resampling).  A file path is
        decoded and resampled on load, so one combined with ``sr`` raises ValueError, as does a rate pair the device
        resampler refuses -- both before anything is launched."""
        model_sr = int(self.hps.data.sampling_rate)
        if sr is None or int(sr) == model_sr:
            return None
        for i, a in enumerate(audios):
            if isinstance(a, str):
                raise ValueError(f"item {i} is a file path ({a!r}): sr= describes NumPy waveforms; files are decoded and "
                                 f"resampled to {model_sr} Hz on load")
        resample_span(int(sr), model_sr)
        return int(sr)

    def _resampled_len(self, n: int, sr: Optional[int]) -> int:
        """Samples at the model's rate of ``n`` samples at ``sr`` (None: already at the model's rate)."""
        return n if sr is None else resample_span(sr, self.hps.data.sampling_rate, n)[0]

    def _stack_se(self, se, n):
        """[n, gin] per-item embeddings on the device; ValueError for one that varies over time."""
        if is_per_frame_se(se, int(getattr(self.hps.model, "gin_channels", 256))):
            raise ValueError("this path takes one embedding per item ([1, gin] or [1, gin, 1]), not a per-frame one")
        if isinstance(se, (list, tuple)):
            se = torch.cat([s.reshape(1, -1) for s in se], 0)
        se = se.to(self.device, torch.float32).reshape(se.shape[0], -1)
        if se.shape[0] == 1:
            se = se.expand(n, -1)
        assert se.shape[0] == n, "one speaker embedding per utterance (or a single one for all)"
        return se

    def _se_items(self, se, n, what: str):
        """The embeddings of n items: ``_stack_se``'s [n, gin] tensor when none varies over time (the per-item path,
        unchanged), else a list of n entries, each a [gin] tensor (per item), a [gin, T] tensor (per frame, T > 1) or a
        ``ToneTrack``.  ValueError for an embedding of the wrong size or shape."""
        gin = int(getattr(self.hps.model, "gin_channels", 256))
        if not is_per_frame_se(se, gin):
            return self._stack_se(se, n)
        items = list(se) if isinstance(se, (list, tuple)) else [se] * n
        if len(items) != n:
            raise ValueError(f"{what}: {len(items)} embeddings for {n} items")
        out = []
        for i, e in enumerate(items):
            if isinstance(e, ToneTrack):
                if e.se.shape[1] != gin:
                    raise ValueError(f"{what}[{i}]: ToneTrack embeddings have {e.se.shape[1]} values, the model's {gin}")
                out.append(e)
                continue
            e = torch.as_tensor(e, dtype=torch.float32)
            if e.numel() == gin:
                out.append(e.reshape(gin))
            elif e.dim() == 3 and e.shape[0] == 1 and e.shape[1] == gin and e.shape[2] > 1:
                out.append(e[0])
            else:
                raise ValueError(f"{what}[{i}] has shape {tuple(e.shape)}: expected [1, {gin}(, 1)], [1, {gin}, T] or a "
                                 f"ToneTrack")
        return out

    def _se_device(self, side, frames, frame0, Tmax: int, what: str, buf: Optional[str] = None,
                   clip: Optional[int] = None):
        """One side of a launch on the device: a [B, gin] tensor as it is, or a list of ``_se_items`` entries as the
        per-frame [B, gin, Tmax] embedding (item b at frames frame0[b] + t, t < frames[b]; zeros after), expanded by the
        tone-track kernel (``pack_tone_keys``).  A [gin, T] entry must cover the item's whole clip: T == ``clip``
        (default frames[b]).
        ``buf`` names a cached device buffer for the result (a stable address: the launch can be replayed from its CUDA
        graph)."""
        if not isinstance(side, list):
            return side
        gin = int(getattr(self.hps.model, "gin_channels", 256))
        out = None if buf is None else self._dev(buf, len(side) * gin * Tmax, torch.float32).view(len(side), gin, Tmax)
        return expand_tone_keys(self.model.native, side, frame0, frames, Tmax, out, what, clip)

    def _enqueue_chunk(self, waves, src, tgt, tau, noise, slot=0, sr=None, seeds=None, fill=None):
        """Stage, upload and launch one ragged batch on the current stream WITHOUT synchronising the host.
        Returns (o [B, 256 * Tmax] on the device, frames per item).  ``sr``: the waves' rate when it is not the
        model's (``_input_rate``): the raw samples are uploaded and resampled on the device into the slot's buffer.
        ``tau``: a float or one per item; ``seeds``: None or one key per item (validated by the caller).
        ``fill``: the items are already on the device.  ``waves`` then holds each item's sample count, and
        ``fill(rows)`` enqueues the writes of the items' samples, zero padded, into the [B, pitch] device rows the
        upload would have filled."""
        hps = self.hps
        hop = hps.data.hop_length
        B = len(waves)
        lens_in = [len(w) for w in waves] if fill is None else [int(n) for n in waves]
        lens = [self._resampled_len(n, sr) for n in lens_in]
        after = "" if sr is None else " after resampling"
        frames = [n // hop for n in lens]
        if min(frames) < 1:
            raise ValueError("audio shorter than one hop" + after)
        Tmax = max(frames)
        dev = self.device
        if min(lens) <= (hps.data.filter_length - hop) // 2:
            raise ValueError("audio shorter than the STFT reflect padding" + after)   # torch raises here too
        # host -> device: one pinned staging buffer per slot (cached across calls: cudaHostAlloc is slow), one copy;
        # a slot is restaged only after its previous upload has left it
        # the padded length is rounded up to 16 hops: batches of similar length share one launch signature, so the native
        # library replays their CUDA graph; every item still runs at its own exact length (ragged), so nothing changes
        Lmax = -(-max(lens) // (16 * hop)) * (16 * hop)
        Lin = Lmax if sr is None else max(lens_in)       # staged samples per row
        ev = self.__dict__.setdefault("_h2d_done", {}).get(slot)
        if ev is not None:
            ev.synchronize()
        if fill is None:
            stage = self._pinned(f"in{slot}", B * Lin).view(B, Lin)
            stage_np = stage.numpy()

            def put(b):
                w = waves[b]
                stage_np[b, : len(w)] = w
                if len(w) < Lin:
                    stage_np[b, len(w):] = 0.0
            _parallel(put, B)
        # device-side buffers are cached per slot too: with every address stable, a repeated (batch, length) call is
        # replayed from a CUDA graph by the native library (include/ovc.h: OVC_OPT_GRAPH); the resampler writes into
        # the same per-slot buffer the spectrogram reads
        wav = self._dev(f"wav{slot}", B * Lmax, torch.float32).view(B, Lmax)
        if sr is None:
            wav.copy_(stage, non_blocking=True) if fill is None else fill(wav)
        else:
            raw = self._dev(f"raw{slot}", B * Lin, torch.float32).view(B, Lin)
            raw.copy_(stage, non_blocking=True) if fill is None else fill(raw)
            rlen_pin = self._pinned_i64(f"rlen{slot}", B)
            rlen_pin.copy_(torch.tensor(lens_in, dtype=torch.int64))
            rlen = self._dev(f"rlen{slot}", B, torch.int64)
            rlen.copy_(rlen_pin, non_blocking=True)
        lens_pin = self._pinned_i64(f"len{slot}", B)
        lens_pin.copy_(torch.tensor(lens, dtype=torch.int64))
        wlen = self._dev(f"len{slot}", B, torch.int64)
        wlen.copy_(lens_pin, non_blocking=True)
        if isinstance(src, list):
            src_d = self._se_device(src, frames, [0] * B, Lmax // hop, "src_se", f"srcf{slot}")
        else:
            src_d = self._dev(f"src{slot}", src.numel(), torch.float32).view(B, -1)
            src_d.copy_(src.reshape(B, -1), non_blocking=True)
        if isinstance(tgt, list):
            tgt_d = self._se_device(tgt, frames, [0] * B, Lmax // hop, "tgt_se", f"tgtf{slot}")
        else:
            tgt_d = self._dev(f"tgt{slot}", tgt.numel(), torch.float32).view(B, -1)
            tgt_d.copy_(tgt.reshape(B, -1), non_blocking=True)
        taus = None if np.ndim(tau) == 0 else list(tau)
        items = None if seeds is None and taus is None else self._item_arrays(f"b{slot}", seeds, taus)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(dev))
        self._h2d_done[slot] = ev
        if sr is not None:
            self.model.native.resample(raw, rlen, sr, hps.data.sampling_rate, out=wav)
        nz = None
        if noise is not None:
            nz = torch.zeros(B, hps.model.inter_channels, Lmax // hop, device=dev, dtype=torch.float32)
            for b, q in enumerate(noise):
                q = q.reshape(hps.model.inter_channels, -1)
                nz[b, :, : q.shape[1]] = q.to(dev)
        seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        # spectrogram + voice_conversion, every item at its own exact length (api.py:148-154)
        o, _ = self.model.native.convert_waveform(wav, wlen, src_d, tgt_d, noise=nz,
                                                  tau=float(tau) if taus is None else taus[0], seed=seed,
                                                  out=self._dev(f"out{slot}", B * (Lmax // hop) * hop, torch.float32),
                                                  frames_out=self._dev(f"fr{slot}", B, torch.int64), items=items)
        return o.view(B, -1), frames

    def _item_arrays(self, slot, seeds, taus) -> dict:
        """Per-item parameter arrays of one call, staged through pinned buffers into device buffers that stay at the
        slot's addresses (a repeated call is still replayed from its CUDA graph, with the new values).  Seeded items draw
        at stream 0.  The caller restages a slot only after the previous call on it has consumed its upload."""
        B = len(seeds) if seeds is not None else len(taus)
        items = {}
        if seeds is not None:
            pin = self._pinned_i64(f"iseed{slot}", 2 * B)
            pin[:B].copy_(torch.from_numpy(seed_array(seeds)))
            pin[B:].zero_()
            d = self._dev(f"iseed{slot}", 2 * B, torch.int64)
            d.copy_(pin, non_blocking=True)
            items["seed"], items["stream"] = d[:B], d[B:]
        if taus is not None:
            pin = self._pinned(f"itau{slot}", B)
            pin.copy_(torch.tensor(taus, dtype=torch.float32))
            d = self._dev(f"itau{slot}", B, torch.float32)
            d.copy_(pin, non_blocking=True)
            items["tau"] = d
        return items

    def _convert_chunk(self, waves, src, tgt, tau, noise, sr=None, seeds=None, fill=None):
        hop = self.hps.data.hop_length
        o, frames = self._enqueue_chunk(waves, src, tgt, tau, noise, sr=sr, seeds=seeds, fill=fill)
        host = self._pinned("out", o.numel()).view(o.shape)
        host.copy_(o, non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        audio = host.numpy()
        return _parallel(lambda b: audio[b, : frames[b] * hop].copy(), len(waves))

    @torch.no_grad()
    def convert_batch_device(self, audios: Sequence[AudioLike], src_se, tgt_se, tau: Union[float, Sequence[float]] = 0.3,
                             slot: int = 0, sr: Optional[int] = None, seeds: Optional[Sequence[int]] = None):
        """``convert_batch`` up to the device: stages and launches ONE ragged batch asynchronously on the current
        stream and returns (o [n, max samples] float32 on the device, samples per item).  No host synchronisation,
        no device -> host copy: the building block of ``distributed.convert_sharded_async`` (waveforms gathered
        GPU-to-GPU over NCCL) and of pipelined serving.  ``slot`` picks the pinned upload buffer (alternate 0 / 1
        between in-flight calls).  ``sr``, ``tau`` (scalar or per item) and ``seeds`` as in ``convert_batch``."""
        n = len(audios)
        tau, taus = check_per_item(tau, n, "tau")
        seeds = check_seeds(seeds, n)
        rate = self._input_rate(audios, sr)
        waves = [_load_audio(a, self.hps.data.sampling_rate) for a in audios]
        o, frames = self._enqueue_chunk(waves, self._se_items(src_se, n, "src_se"), self._se_items(tgt_se, n, "tgt_se"),
                                        tau if taus is None else taus, None, slot, rate, seeds)
        hop = self.hps.data.hop_length
        return o, [f * hop for f in frames]

    def _dev(self, name, numel, dtype):
        """Grow-only device buffers (per upload slot): the result of slot s is overwritten by the next call on slot s."""
        cache = self.__dict__.setdefault("_dev_cache", {})
        buf = cache.get(name)
        if buf is None or buf.numel() < numel or buf.dtype != dtype:
            buf = torch.empty(int(numel * 1.25) + 64, dtype=dtype, device=self.device)
            cache[name] = buf
        return buf[:numel]

    def _pinned_i64(self, name, numel):
        cache = self.__dict__.setdefault("_pin_cache", {})
        buf = cache.get(name)
        if buf is None or buf.numel() < numel:
            buf = torch.empty(int(numel) + 64, dtype=torch.int64).pin_memory()
            cache[name] = buf
        return buf[:numel]

    def _pinned(self, name, numel):
        """Grow-only pinned host staging buffers."""
        cache = self.__dict__.setdefault("_pin_cache", {})
        buf = cache.get(name)
        if buf is None or buf.numel() < numel:
            buf = torch.empty(int(numel * 1.25) + 1024, dtype=torch.float32).pin_memory()
            cache[name] = buf
        return buf[:numel]

    # ------------------------------------------------------------------ watermark (third-party model)
    _WM_CHUNK = 16000      # samples per watermarked chunk
    _WM_STRIDE = 32000     # chunk n starts at n * 32000 (openvoice/api.py:169-171)

    def _wm_chunks(self, audio, count):
        """Yield (index, slice) of the first ``count`` watermark chunks; a short chunk ends the walk."""
        for n in range(count):
            sl = slice(n * self._WM_STRIDE, n * self._WM_STRIDE + self._WM_CHUNK)
            yield n, sl, len(audio[sl]) == self._WM_CHUNK

    def add_watermark(self, audio, message):
        """Embed ``message`` with the wavmark model, 32 bits per 16000-sample chunk, chunks 32000 samples apart
        (behaviour of openvoice/api.py:162-184, incl. the "Audio too short" early stop).  No model -> no-op.
        The chunks are cut, encoded and written back ON THE DEVICE as one batch (``watermark_device``): one upload and
        one download per utterance instead of two host round trips per chunk."""
        if self.watermark_model is None:
            return audio
        dev_audio = torch.as_tensor(audio, dtype=torch.float32).to(self.device)
        watermark_device(dev_audio, utils.string_to_bits(message).reshape(-1), self.watermark_model)
        audio[...] = dev_audio.cpu().numpy()
        return audio

    def detect_watermark(self, audio, n_repeat):
        """Decode ``n_repeat`` chunks back to text (openvoice/api.py:186-201); "Fail" when the audio is too short."""
        if self.watermark_model is None:
            raise RuntimeError("detect_watermark needs the wavmark model: construct with enable_watermark=True")
        rows = []
        for n, sl, full in self._wm_chunks(audio, n_repeat):
            if not full:
                print("Audio too short, fail to detect watermark")
                return "Fail"
            with torch.no_grad():
                sig = torch.as_tensor(audio[sl], dtype=torch.float32, device=self.device)[None]
                rows.append((self.watermark_model.decode(sig) >= 0.5).int().detach().cpu().numpy().squeeze())
        return utils.bits_to_string(np.stack(rows).reshape(-1, 8))
