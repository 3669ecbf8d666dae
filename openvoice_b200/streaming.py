"""Stateful streaming front of the tone-colour converter (SURVEY.md section 8 row f4).

``ToneColorConverter.convert`` (openvoice/api.py:141-160) needs the whole utterance.  The path is not causal -- the
posterior encoder, both flow passes and the generator together see +-110 spectrogram frames
(``ToneColorConverter.HALO_FRAMES`` = 128 with margin) -- so a stream can emit frame t once the audio of frame
t + 128 has arrived.  ``StreamingConverter`` keeps exactly that much state between calls:

* the spectrogram frames of the last window's right halo plus the left halo of the next one (computed on the device
  from the audio tail, frames whose STFT support is still incomplete are left for the next push),
* the noise columns drawn for those frames (the draw of ``models.py:220`` is per frame: a frame keeps its noise no
  matter which window it is converted in),
* the audio samples not yet covered by a complete STFT frame.

Every ``push`` converts as many ``window_frames``-frame windows as the new audio completes -- window + halo on both
sides as ONE batch-1 ragged call of the same kernels ``convert`` runs -- and returns their interiors; ``flush`` ends
the stream (right reflect padding of ``spectrogram_torch``, mel_processing.py:62-63) and returns the rest.  The
concatenated output equals ``convert`` on the whole clip with the same noise (``tests/test_gpu_parity.py``:
<= 2e-6 * rms, the fp32 reordering between tile geometries), whatever the chunking of the input.
Algorithmic latency: (128 + window_frames) * 256 samples; compute per emitted frame: (window + 256) / window of the
offline cost.

Audio that is not at the model's rate (48 kHz from WebRTC and most sound cards, 16 kHz from telephony) goes through
``StreamingResampler``: ``StreamingConverter(..., input_sr=48000, output_sr=48000)`` resamples the input to the model's
rate and the converted audio back, each on the device, and each bit-identical to resampling the whole signal at once
(no clicks at chunk boundaries).  The two filters add their look-ahead to the latency: 10 max(up, down) / up input
samples each, 0.45 ms for 48 kHz -> 22.05 kHz and 0.45 ms for 22.05 kHz -> 48 kHz, 0.91 ms in all
(``StreamingResampler.lookahead_s`` computes it from the library's span function).

A server with many live callers uses ``StreamingSessions``: each session behaves exactly like its own
``StreamingConverter(request_seed=...)``, but every ``push`` / ``close`` advances all the sessions it names with one
batched launch sequence -- the sessions' audio lives in device rings, ``ovc_spectrogram_ring`` builds every ready
window's spectrogram in one launch, and one ragged voice conversion converts them all.  ``ready_frames`` and
``stream_windows`` are the readiness and window rules both classes follow.
"""
import math
from collections import deque
from typing import Callable, Dict, Iterable, List, Optional, Sequence, Set, Tuple

import numpy as np
import torch

from ._native import STREAM_OPEN, resample_span


def ready_frames(n_in: int, hop: int, nfft: int, final: bool) -> int:
    """Spectrogram frames of a stream of ``n_in`` samples that can be computed: every frame whose STFT support
    [t*hop - pad, t*hop - pad + nfft) has arrived, or all ``n_in // hop`` of them (right reflect padding) once the stream
    has ended."""
    if final:
        return n_in // hop
    pad = (nfft - hop) // 2
    return min(max(0, (n_in + pad - nfft) // hop + 1), n_in // hop)


def stream_windows(emitted: int, have: int, W: int, H: int, final: bool = False) -> List[Tuple[int, int, int, int]]:
    """Windows (lo, hi, e0, e1) a stream converts next: frames [lo, hi) go into the call, the samples of frames [e0, e1)
    come out.  An open stream converts a ``W``-frame window once ``emitted + W + H`` frames exist, over [e0 - H, e1 + H);
    an ended stream (``final``, ``have`` = all its frames) converts the rest, the last windows clipped to its end."""
    wins = []
    while (emitted < have) if final else (emitted + W + H <= have):
        e1 = min(have, emitted + W)
        wins.append((max(0, emitted - H), min(have, e1 + H), emitted, e1))
        emitted = e1
    return wins


def check_stream_length(n_in: int, hop: int, pad: int) -> None:
    """ValueError for a stream that ends shorter than one hop or than the STFT reflect padding, as ``convert`` refuses."""
    if n_in // hop < 1 or n_in <= pad:
        raise ValueError("audio too short")


class Enrollment:
    """How a live stream learns its source embedding from its own audio.  Snapshot k >= 1 is the embedding of the
    stream's first ``k * every_frames * hop`` model-rate samples (``extract_se`` of that prefix, bit for bit), for
    ``k * every_frames <= until_frames``; each one retargets the stream's source over ``ramp_frames`` frames.  The
    defaults are about 2 s and 10 s at 22.05 kHz.  ValueError for ``every_frames < 2``, ``until_frames < every_frames``
    or ``ramp_frames < 0``."""

    def __init__(self, every_frames: int = 172, until_frames: int = 861, ramp_frames: int = 16):
        for name, v in (("every_frames", every_frames), ("until_frames", until_frames), ("ramp_frames", ramp_frames)):
            if isinstance(v, bool) or int(v) != v:
                raise ValueError(f"Enrollment: {name}={v!r} is not an integer")
        self.every_frames, self.until_frames, self.ramp_frames = int(every_frames), int(until_frames), int(ramp_frames)
        if self.every_frames < 2:
            raise ValueError(f"Enrollment: every_frames must be >= 2, got {self.every_frames}")
        if self.until_frames < self.every_frames:
            raise ValueError(f"Enrollment: until_frames {self.until_frames} is below every_frames {self.every_frames}")
        if self.ramp_frames < 0:
            raise ValueError(f"Enrollment: ramp_frames must be >= 0, got {self.ramp_frames}")

    def snapshot(self, n0: int, n1: int, hop: int) -> int:
        """The snapshot a step taking a stream from n0 to n1 model-rate samples produces: the last k whose prefix
        k * every_frames * hop lies in (n0, n1], or 0 for none."""
        k = min(n1 // (self.every_frames * hop), self.until_frames // self.every_frames)
        return k if k >= 1 and k * self.every_frames * hop > n0 else 0

    def __repr__(self):
        return f"Enrollment({self.every_frames}, {self.until_frames}, {self.ramp_frames})"


def enroll_new_frames(n0: int, n1: int, hop: int, nfft: int) -> int:
    """``max_new_frames`` of a ``reference_encoder_stream`` call taking a stream from n0 to n1 samples, rounded up to
    64 so that steady steps reuse one workspace size."""
    f = ready_frames(n1, hop, nfft, False) - ready_frames(n0, hop, nfft, False)
    return max(64, -(-f // 64) * 64)


class StreamingResampler:
    """Stateful ``ovc_resample`` (scipy.signal.resample_poly arithmetic) from ``sr_in`` to ``sr_out``.

    ``push(x)`` returns every output sample whose input support has arrived; ``flush()`` ends the stream and returns
    the rest, up to n_out(total) = ceil(total * sr_out / sr_in).  Only the input tail that future outputs read is kept
    (about 20 max(up, down) / up samples).  Every output is computed by the same fp64 sum as the one-shot call, so for
    any chunking the concatenated output equals ``NativeConverter.resample`` of the whole signal bit for bit.
    ``native``: a ``NativeConverter`` (or anything with a ``.native`` one, such as ``NativeSynthesizer``)."""

    def __init__(self, native, sr_in: int, sr_out: int):
        self.native = getattr(native, "native", native)
        self.sr_in, self.sr_out = int(sr_in), int(sr_out)
        resample_span(self.sr_in, self.sr_out)            # ValueError for a pair the resampler refuses
        self.dev = torch.device("cuda", self.native.device_index)
        self.buf = np.zeros(0, dtype=np.float32)          # input samples [b0, b0 + len(buf))
        self.b0 = 0
        self.n_in = 0
        self.emitted = 0
        self.closed = False

    @property
    def state_samples(self) -> int:
        return int(len(self.buf))

    @property
    def lookahead_s(self) -> float:
        """Seconds of input an output sample waits for past its own time: the filter's half support."""
        m = 10 ** 6
        hi = resample_span(self.sr_in, self.sr_out, 0, m, m + 1)[3]
        return (hi - 1) / self.sr_in - m / self.sr_out

    def _emit(self, m1: int, length: int) -> np.ndarray:
        m0 = self.emitted
        if m1 <= m0:
            return np.zeros(0, dtype=np.float32)
        _, _, lo, hi = resample_span(self.sr_in, self.sr_out, 0, m0, m1)
        lo, hi = max(lo, 0), min(hi, self.n_in)
        seg = self.buf[lo - self.b0: hi - self.b0] if hi > lo else np.zeros(1, dtype=np.float32)
        start = lo if hi > lo else self.n_in              # no sample needed: one that reads as 0
        x = torch.from_numpy(np.ascontiguousarray(seg)).to(self.dev)[None]
        ln = torch.tensor([length], dtype=torch.int64, device=self.dev)
        y = self.native.resample(x, ln, self.sr_in, self.sr_out, out_pitch=m1 - m0, in_start=start, out_start=m0)
        self.emitted = m1
        keep = max(0, resample_span(self.sr_in, self.sr_out, 0, m1, m1 + 1)[2])
        if keep > self.b0:
            self.buf = self.buf[keep - self.b0:]
            self.b0 = keep
        return y[0].cpu().numpy()

    @torch.no_grad()
    def push(self, samples) -> np.ndarray:
        assert not self.closed, "the stream has been flushed"
        x = np.asarray(samples, dtype=np.float32).reshape(-1)
        self.buf = np.concatenate([self.buf, x])
        self.n_in += len(x)
        return self._emit(resample_span(self.sr_in, self.sr_out, self.n_in)[1], STREAM_OPEN)

    @torch.no_grad()
    def flush(self) -> np.ndarray:
        assert not self.closed
        self.closed = True
        return self._emit(resample_span(self.sr_in, self.sr_out, self.n_in)[0], self.n_in)


def retarget_track(track, f: int, new, ramp_frames: int = 0):
    """The ``ToneTrack`` that follows ``track`` on frames < f and then moves to ``new``: hard at f (``ramp_frames`` 0),
    else linearly from ``track``'s value at f to ``new`` at f + ramp_frames.  Frames < f keep ``track``'s values bit for
    bit: the old keys before f stay, and where f falls inside a ramp of ``track`` its frames since the ramp's last key are
    pinned by one key each (a key at every integer frame reproduces the values exactly)."""
    from .api import ToneTrack
    ramp = int(ramp_frames)
    if ramp < 0 or int(f) < 0:
        raise ValueError(f"retarget: frame {f} and ramp_frames {ramp_frames} must be >= 0")
    new = torch.as_tensor(new, dtype=torch.float32).reshape(-1).cpu()
    kf, kse = [int(v) for v in track.frames], track.se
    keys = []
    if f > 0:
        i = sum(1 for v in kf if v < f)                   # old keys before f
        keys = [(kf[k], kse[k]) for k in range(i)]
        p = kf[i - 1] if i else f - 1
        if 0 < i < len(kf):                               # inside a ramp: pin frames (p, f - 1] one by one
            d = track.dense(f - 1 - p, p + 1)[0]
            keys += [(p + 1 + t, d[:, t]) for t in range(f - 1 - p)]
        elif p < f - 1 or not i:                          # holding a value: one key at f - 1 holds it to there
            keys.append((f - 1, track.dense(1, f - 1)[0, :, 0]))
    if ramp:
        keys += [(f, track.dense(1, f)[0, :, 0]), (f + ramp, new)]
    else:
        keys.append((f, new))
    return ToneTrack(keys)


class StreamingConverter:
    def __init__(self, converter, src_se, tgt_se, tau: float = 0.3, window_frames: int = 256,
                 noise_fn: Optional[Callable[[int, int], torch.Tensor]] = None, seed: Optional[int] = None,
                 input_sr: Optional[int] = None, output_sr: Optional[int] = None, request_seed: Optional[int] = None,
                 enroll: Optional[Enrollment] = None):
        """``converter``: a ToneColorConverter.  ``noise_fn(t0, t1) -> [inter_channels, t1 - t0]`` supplies the noise of
        absolute frames [t0, t1) (tests pass slices of one tensor); default: a seeded device generator.
        ``input_sr`` / ``output_sr``: rates of the pushed and of the returned audio when they are not the model's
        (``StreamingResampler`` on each side; None: the model's rate).
        ``request_seed``: the request's own key, as ``ToneColorConverter.convert(seed=...)`` takes it: each window draws
        its noise in-kernel at its absolute frames, so the stream gives ``convert(seed=request_seed)`` and no noise is
        kept.  It excludes ``noise_fn`` and ``seed`` (ValueError).
        ``enroll``: an ``Enrollment``: the stream learns its source embedding from its own audio (see
        ``StreamingSessions.open``), with one reference-encoder state row and a device ring of its own.  ``src_se`` may
        then be None: no window is converted before the first snapshot, which becomes the source from frame 0."""
        from .api import check_seeds
        if request_seed is not None:
            if noise_fn is not None or seed is not None:
                raise ValueError("request_seed replaces noise_fn and seed: pass only one of them")
            request_seed = check_seeds([request_seed], 1, "request_seed")[0]
        self.request_seed = request_seed
        self.conv = converter
        hp = converter.hps
        self.rs_in = self.rs_out = None
        if input_sr is not None and int(input_sr) != int(hp.data.sampling_rate):
            self.rs_in = StreamingResampler(converter.model, input_sr, hp.data.sampling_rate)
        if output_sr is not None and int(output_sr) != int(hp.data.sampling_rate):
            self.rs_out = StreamingResampler(converter.model, hp.data.sampling_rate, output_sr)
        self.hop = hp.data.hop_length
        self.nfft = hp.data.filter_length
        self.pad = (self.nfft - self.hop) // 2            # reflect padding of spectrogram_torch
        self.C = hp.model.inter_channels
        self.S = hp.data.filter_length // 2 + 1
        self.H = converter.HALO_FRAMES
        self.W = int(window_frames)
        assert self.W >= 1
        self.tau = float(tau)
        self.dev = converter.device
        if enroll is not None and not isinstance(enroll, Enrollment):
            raise ValueError(f"enroll must be an Enrollment, got {enroll!r}")
        if src_se is None and enroll is None:
            raise ValueError("src_se is None: a stream without a source embedding needs enroll=Enrollment(...)")
        self.enroll = enroll
        self.src = None if src_se is None else converter._stack_se(src_se, 1)
        self.tgt = converter._stack_se(tgt_se, 1)
        if enroll is not None:
            nat = converter.model.native
            self._est = torch.zeros(1, nat.refenc_state_floats, device=self.dev)
            self._ering = torch.zeros(1, 4 * self.nfft, device=self.dev)
        self.tracks = {"src": None, "tgt": None}          # ToneTrack of a side once it has been retargeted
        if noise_fn is None and request_seed is None:
            gen = torch.Generator(device=self.dev)
            gen.manual_seed(int(seed if seed is not None else torch.randint(0, 2 ** 62, (1,)).item()))
            noise_fn = lambda t0, t1: torch.randn(self.C, t1 - t0, device=self.dev, generator=gen)  # noqa: E731
        self.noise_fn = noise_fn
        # ---- state
        self.audio = np.zeros(0, dtype=np.float32)        # samples from absolute index a0 on
        self.a0 = 0
        self.n_in = 0                                     # samples received so far
        self.spec = torch.zeros(1, self.S, 0, device=self.dev)    # frames [f0, f0 + spec.shape[2])
        self.noise = torch.zeros(self.C, 0, device=self.dev)
        self.f0 = 0
        self.emitted = 0                                  # frames whose samples have been returned
        self.closed = False

    # ------------------------------------------------------------------ state size (tests: bounded)
    @property
    def state_frames(self) -> int:
        return int(self.spec.shape[2])

    @property
    def state_samples(self) -> int:
        return int(len(self.audio))

    # ------------------------------------------------------------------ spectrogram frames as audio arrives
    def _extend_spec(self, final: bool):
        """Append every frame whose STFT support [t*hop - pad, t*hop - pad + nfft) is complete (all of them, with the
        right reflect padding, when the stream ends)."""
        hop, pad = self.hop, self.pad
        have = self.f0 + self.spec.shape[2]               # next frame to compute
        upto = ready_frames(self.n_in, hop, self.nfft, final)
        if upto <= have:
            return
        # segment of audio that gives frames [have, upto) away from its own reflect-padded ends: the native STFT pads
        # the segment it is given, so start 2 frames early (unless at the stream start) and require the support of
        # frame upto-1 inside the segment (unless the stream has ended)
        lead = 2 if have >= 2 else have
        s_lo = (have - lead) * hop
        s_hi = self.n_in
        seg = self.audio[s_lo - self.a0: s_hi - self.a0]
        wav = torch.from_numpy(np.ascontiguousarray(seg)).to(self.dev)[None]
        wlen = torch.tensor([wav.shape[1]], dtype=torch.int64, device=self.dev)
        sp, _ = self.conv.model.native.spectrogram(wav.contiguous(), wlen)
        new = sp[:, :, lead: lead + (upto - have)]
        assert new.shape[2] == upto - have, (new.shape, upto, have, lead)
        self.spec = torch.cat([self.spec, new], 2)
        if self.request_seed is None:
            self.noise = torch.cat([self.noise, self.noise_fn(have, upto).to(self.dev, torch.float32).reshape(self.C, -1)], 1)
        # audio before the support of the next frame (and its 2 lead frames) is no longer needed
        keep_from = max(0, (upto - 2) * hop - pad)
        if keep_from > self.a0:
            self.audio = self.audio[keep_from - self.a0:]
            self.a0 = keep_from

    def _window_se(self, name: str, lo: int, hi: int):
        """A side's embedding for the window's frames [lo, hi): [1, gin] where it is constant over them (the per-item
        launch, as before any retarget), else [1, gin, hi - lo] expanded from its track at the window's absolute frames."""
        tr = self.tracks[name]
        if tr is None:
            return self.src if name == "src" else self.tgt
        if hi - 1 < tr.frames[0]:
            return tr.se[:1].to(self.dev)
        if lo >= tr.frames[-1]:
            return tr.se[-1:].to(self.dev)
        return self.conv._se_device([tr], [hi - lo], [lo], hi - lo, name)

    @torch.no_grad()
    def retarget(self, src_se=None, tgt_se=None, ramp_frames: int = 0) -> int:
        """Change the stream's source and / or target embedding without closing it.  The change starts at frame f, the
        first frame no window has read yet (the frames ready so far), and is hard (``ramp_frames`` 0) or linear over
        ``ramp_frames`` frames (``retarget_track``).  Returns f.  The stream's output then equals ``convert`` on the whole
        clip with ``tone_track(side)`` as that side's embedding, bit for bit.  A window that overlaps no transition runs
        exactly the per-item launch.  ValueError for an embedding that is not one per item, and for ``src_se`` on an
        enrolling stream without a prior that has no source yet (its first snapshot will be the source from frame 0)."""
        assert not self.closed, "the stream has been flushed"
        if src_se is not None and self.src is None:
            raise ValueError("retarget(src_se=...): the stream has no source before its first enrollment snapshot")
        f = self.f0 + int(self.spec.shape[2])
        for name, se in (("src", src_se), ("tgt", tgt_se)):
            if se is not None:
                new = self.conv._stack_se(se, 1)[0].cpu()
                self.tracks[name] = retarget_track(self.tone_track(name), f, new, ramp_frames)
        return f

    def tone_track(self, name: str):
        """The ``ToneTrack`` of side ``"src"`` or ``"tgt"`` over the whole stream so far.  ValueError for ``"src"`` of an
        enrolling stream without a prior before its first snapshot."""
        from .api import ToneTrack
        if name == "src" and self.src is None:
            raise ValueError("the stream has no source embedding before its first enrollment snapshot")
        tr = self.tracks[name]
        return tr if tr is not None else ToneTrack([(0, (self.src if name == "src" else self.tgt)[0].cpu())])

    def _convert_window(self, lo: int, hi: int, e0: int, e1: int) -> np.ndarray:
        """Samples of frames [e0, e1): one ragged batch-1 call over the window's frames [lo, hi)."""
        sp = self.spec[:, :, lo - self.f0: hi - self.f0].contiguous()
        lens = torch.tensor([hi - lo], dtype=torch.int64, device=self.dev)
        src, tgt = self._window_se("src", lo, hi), self._window_se("tgt", lo, hi)
        if self.request_seed is None:
            nz = self.noise[None, :, lo - self.f0: hi - self.f0].contiguous()
            o, _, _ = self.conv.model.voice_conversion(sp, lens, src, tgt, tau=self.tau, noise=nz, ragged=True,
                                                       latents=False)
        else:
            o, _, _ = self.conv.model.voice_conversion(sp, lens, src, tgt, tau=self.tau, ragged=True,
                                                       latents=False, seeds=[self.request_seed], frame0=[lo])
        out = o[0, 0, (e0 - lo) * self.hop: (e1 - lo) * self.hop].cpu().numpy().copy()
        self.emitted = e1
        # frames before the next window's left halo can go
        drop = max(0, e1 - self.H) - self.f0
        if drop > 0:
            self.spec = self.spec[:, :, drop:]
            if self.request_seed is None:
                self.noise = self.noise[:, drop:]
            self.f0 += drop
        return out

    # ------------------------------------------------------------------ public
    @torch.no_grad()
    def push(self, samples) -> np.ndarray:
        """Feed float32 samples (at ``input_sr``, default the model's rate); returns the converted samples that became
        final (at ``output_sr``, default the model's rate)."""
        assert not self.closed, "the stream has been flushed"
        x = np.asarray(samples, dtype=np.float32).reshape(-1)
        if self.rs_in is not None:
            x = self.rs_in.push(x)
        y = self._push(x)
        return y if self.rs_out is None else self.rs_out.push(y)

    @torch.no_grad()
    def flush(self) -> np.ndarray:
        """End of the stream: converts what is left (the last frames use the right reflect padding, exactly like the
        whole-clip spectrogram).  Total output = hop * (samples_in // hop) at the model's rate, as ``convert`` returns
        (then resampled to ``output_sr``)."""
        assert not self.closed
        y = (self._flush() if self.rs_in is None else
             np.concatenate([self._push(self.rs_in.flush(), ending=True), self._flush()]))
        return y if self.rs_out is None else np.concatenate([self.rs_out.push(y), self.rs_out.flush()])

    def _push(self, x: np.ndarray, ending: bool = False) -> np.ndarray:
        """Append model-rate samples and convert the windows they complete.  A snapshot the samples produce retargets
        the source after those windows, unless the stream is ``ending``: then it would take effect after the stream's
        last window (as a session's closing step applies it), and is dropped."""
        n0 = self.n_in
        self.audio = np.concatenate([self.audio, x])
        self.n_in += len(x)
        snap = self._enroll_step(n0) if self.enroll is not None else None
        self._extend_spec(final=False)
        have = self.f0 + self.spec.shape[2]
        wins = stream_windows(self.emitted, have, self.W, self.H) if self.src is not None else []
        outs = [self._convert_window(*w) for w in wins]
        if snap is not None and not ending:
            self.retarget(src_se=snap, ramp_frames=self.enroll.ramp_frames)
        return np.concatenate(outs) if outs else np.zeros(0, dtype=np.float32)

    def _enroll_step(self, n0: int):
        """Advance the stream's reference encoder over the pushed samples.  Returns the snapshot the push produces (to
        retarget to once the push's windows are converted), or None; a stream without a source takes its first
        snapshot as the source from frame 0."""
        hop, pad = self.hop, self.pad
        lo = max(0, ready_frames(n0, hop, self.nfft, False) * hop - pad)     # first sample the encoder still reads
        at = n0
        if self.n_in - lo > self._ering.shape[1]:         # grow: the samples [lo, n0) go to their new places too
            self._ering = torch.zeros(1, 1 << (int((self.n_in - lo) * 1.25) - 1).bit_length(), device=self.dev)
            at = lo
        if self.n_in > at:
            seg = torch.from_numpy(np.ascontiguousarray(self.audio[at - self.a0:])).to(self.dev)
            pos = torch.from_numpy(np.arange(at, self.n_in) % self._ering.shape[1]).to(self.dev)
            self._ering[0].index_copy_(0, pos, seg)
        k = self.enroll.snapshot(n0, self.n_in, hop)
        desc = torch.tensor([[0, 0, self.n_in, k * self.enroll.every_frames * hop]], dtype=torch.int64).to(self.dev)
        out = self.conv.model.native.reference_encoder_stream(self._ering, self._est, desc,
                                                              enroll_new_frames(n0, self.n_in, hop, self.nfft))
        if not k:
            return None
        se = out.cpu()
        if self.src is None:
            self.src = se.to(self.dev)
            return None
        return se

    @torch.no_grad()
    def source_se(self):
        """(embedding [1, gin, 1], n): ``extract_se`` of everything the stream has received (n model-rate samples),
        bit for bit, from its encoder state in one call.  ValueError without ``enroll`` or for a stream still shorter
        than one hop or than the STFT padding."""
        if self.enroll is None:
            raise ValueError("source_se needs a stream opened with enroll=Enrollment(...)")
        n = self.n_in
        if n < self.hop or n <= self.pad:
            raise ValueError(f"source_se: the stream has {n} samples, needs at least {max(self.hop, self.pad + 1)}")
        desc = torch.tensor([[0, 0, n, n]], dtype=torch.int64).to(self.dev)
        se = self.conv.model.native.reference_encoder_stream(self._ering, self._est, desc, 1)
        return se.cpu().reshape(1, -1, 1), n

    def _flush(self) -> np.ndarray:
        if self.src is None:
            raise ValueError("the stream ends before its first enrollment snapshot: it has no source embedding")
        self.closed = True
        check_stream_length(self.n_in, self.hop, self.pad)
        self._extend_spec(final=True)
        T = self.n_in // self.hop
        outs = [self._convert_window(*w) for w in stream_windows(self.emitted, T, self.W, self.H, final=True)]
        return np.concatenate(outs) if outs else np.zeros(0, dtype=np.float32)


# Padded frames (windows x Tmax) of one voice-conversion launch of ``StreamingSessions``: a step whose windows exceed it
# runs several launches.  64 sessions' 256-frame windows with both 128-frame halos (64 x 512) fill one launch, about the
# converter workspace of ``convert_batch``'s 64-item batches of 10 s clips.
SESSION_BATCH_FRAMES = 32768


class _Session:
    __slots__ = ("row", "seed", "tau", "n_in", "emitted", "in_sr", "out_sr", "raw_n", "out_n", "se", "tracks", "enroll",
                 "has_src", "lat")

    def __init__(self, row: int, seed: int, tau: float, in_sr: Optional[int] = None, out_sr: Optional[int] = None):
        self.row, self.seed, self.tau = row, seed, tau
        self.n_in = 0                                     # samples received (at the model's rate)
        self.emitted = 0                                  # frames whose samples have been returned
        self.in_sr, self.out_sr = in_sr, out_sr           # rates of the pushed / returned audio; None: the model's
        self.raw_n = 0                                    # samples received at in_sr
        self.out_n = 0                                    # samples returned at out_sr
        self.se = None                                    # [2, gin] host copy of the embedding table row
        self.tracks = [None, None]                        # ToneTrack of the source / target once retargeted
        self.enroll = None                                # Enrollment of a session that learns its source
        self.has_src = True                               # False until an enrolling session without a prior has one
        self.lat = 0                                      # StagedSessions: frames whose final latents are in its ring


class StreamingSessions:
    """Many live streams through one converter, advanced together.

    ``open`` starts a session and returns its id; ``push({id: samples, ...})`` feeds any number of sessions and returns
    ``{id: float32 samples that became final}``; ``close(ids)`` ends sessions and returns the rest of their audio.  Each
    session's output equals ``StreamingConverter(converter, src_se, tgt_se, tau, window_frames, request_seed=seed)`` fed
    the same chunks, bit for bit, whatever else runs beside it: the windows follow ``stream_windows``, the spectrogram
    frames are those of the whole clip, and each window draws its noise at its own seed and absolute frames.

    Every ``push`` / ``close`` is one step: one packed upload (the pushed samples and every per-window value), one
    ``ovc_splice`` of the samples into the sessions' device audio rings, one ``ovc_spectrogram_ring`` over every ready
    window of every session in the call, one gather of their embeddings from a device table, ragged voice conversions of up to
    ``SESSION_BATCH_FRAMES`` padded frames each (one for a typical step), one gather of the emitted frames, one download
    and one synchronisation.  Buffers are grow-only and the padded window length is rounded up to 16 frames, so a steady
    lockstep step replays its CUDA graph.  A session keeps the audio of its next window and both halos, plus the STFT
    support and its largest push, on the device.

    Sessions may push and receive audio at other rates than the model's: ``rates`` declares them up front (the
    constructor builds each rate's two filter banks, which waits for the device), and ``open(input_sr=, output_sr=)``
    takes any declared rate.  Such a session equals ``StreamingConverter(..., input_sr=, output_sr=)`` bit for bit.  Its
    pushed samples go into a raw ring row (a second ``ovc_splice``), and ONE ``ovc_resample_rings`` over every such
    session of the step writes their new model-rate samples into their ring rows; on the way out, the emitted frames are
    spliced into an output ring row (a third splice) and ONE more ``ovc_resample_rings`` writes every such session's new
    samples at its rate into the buffer the frames are gathered into, so the step still has one download.  A step that
    names a resampling session thus has at most four more launches, however many it names; one that names none runs
    exactly the launches above.  The raw ring keeps the input the next model-rate sample reads plus the largest push,
    the output ring the model-rate samples the next output sample reads.

    Noise is drawn in-kernel from each session's seed (no ``noise_fn``)."""

    def __init__(self, converter, window_frames: int = 256, rates: Iterable[int] = ()):
        """``rates``: the rates other than the model's that ``open`` will accept for ``input_sr`` / ``output_sr``.
        ValueError for a rate that is not a positive integer or that the resampler refuses, before anything is built."""
        W = int(window_frames)
        if W < 1:
            raise ValueError(f"window_frames must be >= 1, got {window_frames!r}")
        hp = converter.hps
        self.native = converter.model.native
        self.sr = int(hp.data.sampling_rate)
        declared = []
        for r in rates:
            if isinstance(r, bool) or int(r) != r or int(r) <= 0:
                raise ValueError(f"rates: {r!r} is not a positive integer rate")
            r = int(r)
            resample_span(r, self.sr)                     # ValueError for a pair the resampler refuses
            resample_span(self.sr, r)
            declared.append(r)
        self.rates = tuple(sorted(set(declared)))
        self.hop = hp.data.hop_length
        self.nfft = hp.data.filter_length
        self.pad = (self.nfft - self.hop) // 2
        self.S = self.nfft // 2 + 1
        self.gin = int(getattr(hp.model, "gin_channels", 256))
        self.H = converter.HALO_FRAMES
        self.W = W
        self.dev = torch.device(converter.device)
        self.cuda = self.dev.type == "cuda"
        self.sessions: Dict[int, _Session] = {}
        self.free_rows: List[int] = []
        self.rows = 0
        self.cap = self.hop * (W + 2 * self.H + 8) + 4096   # samples per ring row; grows for larger pushes
        self.rings = torch.zeros(0, self.cap, device=self.dev)
        self.se = torch.zeros(2, 0, self.gin, device=self.dev)   # [src | tgt, row, gin]
        self.est = None                                   # reference-encoder state rows of enrolling sessions
        self.next_id = 0
        self._bufs: dict = {}
        self._h2d_done = None
        # resampling: plan ids of rate -> model and model -> rate, raw input rings and output rings (row = session row)
        self.plans: Dict[Tuple[int, int], int] = {}
        for r in self.rates:
            if r != self.sr:
                self.plans[(r, self.sr)] = self.native.resample_plan(r, self.sr)
                self.plans[(self.sr, r)] = self.native.resample_plan(self.sr, r)
        self.raw = self.orings = None
        if self.plans:                                    # both grow with the largest push / emitted run
            span1 = max(resample_span(a, b, 0, 0, 1)[3] - resample_span(a, b, 0, 0, 1)[2] for a, b in self.plans)
            extra = -(-(span1 + 8192) // 1024) * 1024
            self.raw = torch.zeros(self.rows, extra, device=self.dev)
            self.orings = torch.zeros(self.rows, self.hop * (W + 8) + extra, device=self.dev)

    # ------------------------------------------------------------------ sessions
    def open(self, src_se, tgt_se, tau: float = 0.3, seed: Optional[int] = None, input_sr: Optional[int] = None,
             output_sr: Optional[int] = None, enroll: Optional[Enrollment] = None) -> int:
        """Start a session converting from ``src_se`` to ``tgt_se`` (tone-colour embeddings of ``gin`` values each) and
        return its id.  ``seed``: the session's Philox key in [0, 2^64) (default: drawn from torch's generator).
        ``input_sr`` / ``output_sr``: rates of the pushed and of the returned audio, the model's or one declared with
        ``rates`` (None: the model's); any other rate is refused.

        ``enroll``: an ``Enrollment``: the session learns its source embedding from its own model-rate audio.  Its
        reference-encoder state row advances in every step that names it, in the step's one
        ``ovc_reference_encoder_stream`` call.  With a prior ``src_se``, snapshot k (``extract_se`` of the first
        ``k * every_frames * hop`` samples) takes effect exactly as ``retarget(sid, src_se=snapshot_k,
        ramp_frames=ramp_frames)`` called right after the step whose push makes that prefix available; a step crossing
        several boundaries applies only the last.  With ``src_se=None`` the session converts no window before its first
        snapshot, which is the source from frame 0."""
        from .api import check_seeds
        sr = {}
        for name, rate in (("input_sr", input_sr), ("output_sr", output_sr)):
            ok = rate is None or (not isinstance(rate, bool) and int(rate) == rate
                                  and (int(rate) == self.sr or int(rate) in self.rates))
            if not ok:
                raise ValueError(f"{name}={rate!r}: StreamingSessions takes and returns audio at the model's rate "
                                 f"({self.sr} Hz) or at a rate declared with rates= (declared: "
                                 f"{', '.join(map(str, self.rates)) or 'none'})")
            sr[name] = None if rate is None or int(rate) == self.sr else int(rate)
        tau = float(tau)
        if not math.isfinite(tau):
            raise ValueError(f"tau = {tau!r} is not a finite number")
        seed = int(torch.randint(0, 2 ** 62, (1,)).item()) if seed is None else check_seeds([seed], 1, "seed")[0]
        if enroll is not None and not isinstance(enroll, Enrollment):
            raise ValueError(f"enroll must be an Enrollment, got {enroll!r}")
        if src_se is None and enroll is None:
            raise ValueError("src_se is None: a session without a source embedding needs enroll=Enrollment(...)")
        if enroll is not None and self.native.refenc_state_floats == 0:
            raise ValueError("enroll: the checkpoint has no reference encoder (ref_enc.* tensors)")
        ses = []
        for name, se in (("src_se", src_se), ("tgt_se", tgt_se)):
            se = torch.zeros(self.gin) if se is None else self._per_item_se(name, se)
            if se.numel() != self.gin:
                raise ValueError(f"{name} has {se.numel()} values, the model's embeddings have {self.gin}")
            ses.append(se)
        if not self.free_rows:
            rows = self.rows + max(1, self.rows // 2)
            self.free_rows += range(self.rows, rows)
            self._grow(rows, self.cap, [])
        row = min(self.free_rows)
        self.free_rows.remove(row)
        self.se[:, row] = torch.stack(ses).to(self.dev)
        sid = self.next_id
        self.next_id += 1
        s = self.sessions[sid] = _Session(row, seed, tau, sr["input_sr"], sr["output_sr"])
        s.se = torch.stack(ses)
        if enroll is not None:
            s.enroll, s.has_src = enroll, src_se is not None
            if self.est is None or self.est.shape[0] < self.rows:
                self._grow_est()
            self.est[row].zero_()
        return sid

    def _grow_est(self):
        est = torch.zeros(self.rows, self.native.refenc_state_floats, device=self.dev)
        if self.est is not None:
            est[: self.est.shape[0]] = self.est
        self.est = est

    @torch.no_grad()
    def source_se(self, sid: int):
        """(embedding [1, gin, 1], n): ``extract_se`` of everything session ``sid`` has received (n model-rate samples),
        bit for bit, from its encoder state with one call and one sync.  ValueError for a session opened without
        ``enroll`` or still shorter than one hop or than the STFT padding."""
        s = self.sessions[self._check_ids([sid])[0]]
        if s.enroll is None:
            raise ValueError(f"session {sid} was opened without enroll")
        n = s.n_in
        if n < self.hop or n <= self.pad:
            raise ValueError(f"session {sid} has {n} samples, source_se needs at least {max(self.hop, self.pad + 1)}")
        desc = torch.tensor([[s.row, s.row, n, n]], dtype=torch.int64).to(self.dev)
        se = self.native.reference_encoder_stream(self.rings, self.est, desc, 1)
        return se.cpu().reshape(1, -1, 1), n

    def retarget(self, sid: int, src_se=None, tgt_se=None, ramp_frames: int = 0) -> int:
        """``StreamingConverter.retarget`` for session ``sid``: the change starts at the session's ready frames (the
        first frame no window of it has read) and the call returns that frame; ``tone_track(sid, side)`` then gives the
        whole-clip schedule, and the session equals ``StreamingConverter`` with the same retargets bit for bit.  A step
        none of whose windows overlaps a transition runs exactly the launches it did before; one that has such windows
        adds one tone-track expansion per varying side (after a small upload of the keys) and the per-frame conditioning
        of that side's launches.  ValueError for an embedding that is not ``gin`` values, and for ``src_se`` on an
        enrolling session without a prior that has no source yet (its first snapshot will be the source from frame 0)."""
        s = self.sessions[self._check_ids([sid])[0]]
        if src_se is not None and not s.has_src:
            raise ValueError(f"retarget(src_se=...): session {sid} has no source before its first enrollment snapshot")
        f = ready_frames(s.n_in, self.hop, self.nfft, False)
        for k, se in enumerate((src_se, tgt_se)):
            if se is None:
                continue
            new = self._per_item_se(("src_se", "tgt_se")[k], se)
            if new.numel() != self.gin:
                raise ValueError(f"{('src_se', 'tgt_se')[k]} has {new.numel()} values, the model's embeddings have {self.gin}")
            s.tracks[k] = retarget_track(self.tone_track(sid, ("src", "tgt")[k]), f, new, ramp_frames)
            s.se[k] = new                                 # windows past the last key read the table as before
            self.se[k, s.row] = new.to(self.dev)
        return f

    @staticmethod
    def _per_item_se(name: str, se) -> torch.Tensor:
        """One embedding as a flat host tensor; a ``ToneTrack`` is refused (a session's schedule changes by
        ``retarget``)."""
        from .api import ToneTrack
        if isinstance(se, ToneTrack):
            raise ValueError(f"{name} is a ToneTrack: a session takes one embedding per side and changes it with retarget")
        return torch.as_tensor(se, dtype=torch.float32).reshape(-1)

    def tone_track(self, sid: int, side: str):
        """The ``ToneTrack`` of session ``sid``'s ``"src"`` or ``"tgt"`` embedding over its whole stream so far.
        ValueError for ``"src"`` of an enrolling session without a prior before its first snapshot."""
        from .api import ToneTrack
        s = self.sessions[sid]
        k = ("src", "tgt").index(side)
        if k == 0 and not s.has_src:
            raise ValueError(f"session {sid} has no source embedding before its first enrollment snapshot")
        return s.tracks[k] if s.tracks[k] is not None else ToneTrack([(0, s.se[k].clone())])

    def _window_tracks(self, ses, wins, b0: int, b1: int, Tmax: int, g, fresh=frozenset(), sides=(0, 1)):
        """Per side, the [b1 - b0, gin, Tmax] per-frame embeddings of launch windows b0 .. b1 - 1 when one of them
        overlaps a transition of that side (a track whose last key lies past the window's first frame), else the
        gathered per-item rows g[side] (the launch is then exactly the per-item one).  ``fresh``: sessions whose source
        is the first enrollment snapshot of this step, which only the device table holds: their constant windows take
        the gathered row g[0] at each of their frames.  ``sides``: the sides to return (default both)."""
        out = []
        for k in sides:
            var = [ses[i][1].tracks[k] is not None and lo < ses[i][1].tracks[k].frames[-1]
                   for i, lo, _, _, _ in wins[b0:b1]]
            if not any(var):
                out.append(g[k][b0:b1])
                continue
            from .api import expand_tone_keys
            entries = [ses[i][1].tracks[k] if v else ses[i][1].se[k] for v, (i, _, _, _, _) in zip(var, wins[b0:b1])]
            buf = self._buf(f"gpf{k}", (b1 - b0) * self.gin * Tmax, torch.float32).view(b1 - b0, self.gin, Tmax)
            out.append(expand_tone_keys(self.native, entries, [lo for _, lo, _, _, _ in wins[b0:b1]],
                                        [hi - lo for _, lo, hi, _, _ in wins[b0:b1]], Tmax, buf, ("src_se", "tgt_se")[k]))
            fix = [j for j, (v, (i, _, _, _, _)) in enumerate(zip(var, wins[b0:b1])) if k == 0 and not v and i in fresh]
            if fix:
                ix = torch.tensor(fix, dtype=torch.int64).to(self.dev)
                n = torch.tensor([wins[b0 + j][2] - wins[b0 + j][1] for j in fix], dtype=torch.int64).to(self.dev)
                keep = (torch.arange(Tmax, device=self.dev)[None, :] < n[:, None])[:, None, :]
                rows = g[k][b0:b1].index_select(0, ix)[:, :, None].expand(-1, -1, Tmax)
                out[-1].index_copy_(0, ix, torch.where(keep, rows, torch.zeros((), device=self.dev)))
        return out

    @property
    def rows_in_use(self) -> int:
        return len(self.sessions)

    def state_samples(self, sid: int) -> int:
        """Samples of session ``sid`` still held in its ring row (the ones its next windows read)."""
        s = self.sessions[sid]
        return s.n_in - self._keep_from(s)

    def raw_state_samples(self, sid: int) -> int:
        """Samples at its input rate that session ``sid`` holds in its raw ring row (0 without ``input_sr``)."""
        s = self.sessions[sid]
        return 0 if s.in_sr is None else s.raw_n - self._raw_keep(s)

    def out_state_samples(self, sid: int) -> int:
        """Model-rate samples that session ``sid`` holds in its output ring row (0 without ``output_sr``)."""
        s = self.sessions[sid]
        return 0 if s.out_sr is None else s.emitted * self.hop - self._out_keep(s)

    def _keep_from(self, s: _Session) -> int:
        """First sample of the session's next window: frame max(0, emitted - H) reads from (that frame) * hop - pad."""
        return max(0, (s.emitted - self.H) * self.hop - self.pad)

    def _raw_keep(self, s: _Session) -> int:
        """First raw sample that the session's next model-rate sample reads."""
        return max(0, resample_span(s.in_sr, self.sr, 0, s.n_in, s.n_in + 1)[2])

    def _out_keep(self, s: _Session) -> int:
        """First model-rate sample that the session's next output sample reads."""
        return max(0, resample_span(self.sr, s.out_sr, 0, s.out_n, s.out_n + 1)[2])

    def _model_len(self, s: _Session, n: int) -> int:
        """Model-rate length of session ``s`` once ``n`` more samples at its input rate end it."""
        return s.n_in + n if s.in_sr is None else resample_span(s.in_sr, self.sr, s.raw_n + n)[0]

    def _check_ids(self, ids) -> List[int]:
        ids = list(ids)
        for sid in ids:
            if sid not in self.sessions:
                raise ValueError(f"unknown or closed session {sid!r}")
        if len(set(ids)) != len(ids):
            raise ValueError("a session is named twice")
        return ids

    # ------------------------------------------------------------------ public steps
    @torch.no_grad()
    def push(self, chunks: Dict[int, object]) -> Dict[int, np.ndarray]:
        """Append ``chunks[id]`` (float32 samples at the session's input rate) to each named session; returns, per named
        session, the converted samples that became final (possibly none), at its output rate."""
        ids = self._check_ids(chunks.keys())
        xs = {sid: np.asarray(chunks[sid], dtype=np.float32).reshape(-1) for sid in ids}
        return self._step(xs, final=set())

    @torch.no_grad()
    def push_device(self, runs: Dict[int, Sequence[Tuple[int, int, int]]], src: torch.Tensor,
                    close: Iterable[int] = ()) -> Dict[int, np.ndarray]:
        """``push`` of audio already on the device: appends to each named session, in order, the runs
        ``(src_row, src_off, count)`` of ``src`` ([rows, pitch] float32 on the converter's device, at the session's
        input rate): samples
        src[src_row, src_off : src_off + count], or ``count`` zeros when src_row < 0.  The runs of every session go into
        the rings in ONE ``ovc_splice``; nothing is uploaded but the step's small tables.  The sessions named in
        ``close`` (each also in ``runs``) then end as ``close`` ends them, in the same step.  Returns what ``push`` and
        ``close`` return.  A run outside ``src`` or a session too short to end raises ValueError before any launch."""
        ids = self._check_ids(runs.keys())
        close = set(close)
        if not close <= set(ids):
            raise ValueError("close names a session that has no runs in this call")
        assert src.device.type == self.dev.type and src.dtype == torch.float32 and src.is_contiguous() and src.dim() == 2
        rows, pitch = src.shape
        xs = {}
        for sid in ids:
            xs[sid] = [tuple(int(v) for v in r) for r in runs[sid]]
            for r, o, n in xs[sid]:
                if n < 0 or (r >= 0 and (r >= rows or o < 0 or o + n > pitch)):
                    raise ValueError(f"session {sid}: run {(r, o, n)} is not inside src {tuple(src.shape)}")
        for sid in close:
            check_stream_length(self._model_len(self.sessions[sid], sum(n for _, _, n in xs[sid])), self.hop, self.pad)
            self._check_has_src(sid, self._model_len(self.sessions[sid], sum(n for _, _, n in xs[sid])))
        out = self._step(xs, final=close, src=src)
        for sid in close:
            self.free_rows.append(self.sessions.pop(sid).row)
        return out

    @torch.no_grad()
    def close(self, ids: Iterable[int]) -> Dict[int, np.ndarray]:
        """End the named sessions: converts what is left of each (right reflect padding at its end, like the whole-clip
        spectrogram) and frees their rows.  A session shorter than one hop or than the STFT padding raises ValueError,
        like ``StreamingConverter.flush``; nothing is changed then."""
        ids = self._check_ids(ids)
        for sid in ids:
            check_stream_length(self._model_len(self.sessions[sid], 0), self.hop, self.pad)
            self._check_has_src(sid, self._model_len(self.sessions[sid], 0))
        out = self._step({sid: np.zeros(0, dtype=np.float32) for sid in ids}, final=set(ids))
        for sid in ids:
            self.free_rows.append(self.sessions.pop(sid).row)
        return out

    def _check_has_src(self, sid: int, n: int) -> None:
        """ValueError for a session without a prior that would end (at n model-rate samples) before its first
        snapshot, so it would have no source embedding to convert with."""
        s = self.sessions[sid]
        if not s.has_src and not s.enroll.snapshot(s.n_in, n, self.hop):
            raise ValueError(f"session {sid} ends before its first enrollment snapshot: it has no source embedding "
                             f"(discard it instead)")

    def discard(self, ids: Iterable[int]) -> None:
        """Drop the named sessions without converting what is left of them (a caller that has gone away) and free their
        rows for the next ``open``.  Nothing is launched."""
        for sid in self._check_ids(ids):
            self.free_rows.append(self.sessions.pop(sid).row)

    # ------------------------------------------------------------------ device buffers
    def _buf(self, name: str, numel: int, dtype, pinned: bool = False):
        """Grow-only buffers: stable addresses, so repeated step shapes replay their CUDA graphs."""
        b = self._bufs.get(name)
        if b is None or b.numel() < numel:
            b = torch.empty(int(numel * 1.25) + 64, dtype=dtype, device="cpu" if pinned else self.dev)
            b = b.pin_memory() if pinned and self.cuda else b
            self._bufs[name] = b
        return b[:numel]

    def _moved(self, old: torch.Tensor, rows: int, cap: int, live: List[Tuple[int, int, int]]) -> torch.Tensor:
        """``old`` reallocated as [rows, cap]: each live session's samples [a, b) of row r (``live``: (r, a, b)) moved to
        their places under the new capacity, or, without ``live``, the old rows copied as they are."""
        new = torch.zeros(rows, cap, device=self.dev)
        if live:
            oc = old.shape[1]
            src = np.concatenate([r * oc + np.arange(a, b) % oc for r, a, b in live])
            dst = np.concatenate([r * cap + np.arange(a, b) % cap for r, a, b in live])
            new.view(-1)[torch.from_numpy(dst).to(self.dev)] = old.reshape(-1)[torch.from_numpy(src).to(self.dev)]
        else:
            new[: old.shape[0]] = old
        return new

    def _grow(self, rows: int, cap: int, live: List[Tuple[int, int, int]]):
        """Reallocate the rings as [rows, cap] (and the embedding table as [2, rows, gin], the raw and output rings as
        [rows, their capacity]), moving each live session's samples [a, b) of row r (``live``: (r, a, b)) to their
        places under the new capacity."""
        rings = self._moved(self.rings, rows, cap, live)
        se = torch.zeros(2, rows, self.gin, device=self.dev)
        se[:, : self.rows] = self.se
        if self.raw is not None and rows != self.rows:
            self.raw = self._moved(self.raw, rows, self.raw.shape[1], [])
            self.orings = self._moved(self.orings, rows, self.orings.shape[1], [])
        self.rings, self.se, self.rows, self.cap = rings, se, rows, cap
        if self.est is not None and self.est.shape[0] < rows:
            self._grow_est()

    def _splice(self, source: torch.Tensor, seg: torch.Tensor, segs: Optional[List[Tuple[int, int, int, int, int]]],
                dst: torch.Tensor, src_wrap: bool = False):
        """``ovc_splice`` of ``segs`` (on the device as ``seg``; None: only there) from ``source`` into the ring array
        ``dst``; ``src_wrap``: the source rows are rings too (``SPLICE_SRC_WRAP``)."""
        if self.cuda:
            self.native.splice(source, seg, dst, src_wrap=src_wrap)
        else:   # only the CPU stand-in converters of the host tests get here: the same writes as one index_copy_
            segs = seg.tolist() if segs is None else segs
            cap, pitch = dst.shape[1], source.shape[1]
            at = np.concatenate([r * cap + np.arange(a, a + n) % cap for _, _, n, r, a in segs])
            val = torch.cat([torch.zeros(n) if row < 0 else source[row, (off + torch.arange(n)) % pitch] if src_wrap
                             else source[row, off:off + n] for row, off, n, _, _ in segs])
            dst.view(-1).index_copy_(0, torch.from_numpy(at), val)

    # ------------------------------------------------------------------ one step
    def _step(self, xs: Dict[int, object], final: Set[int], src: Optional[torch.Tensor] = None) -> Dict[int, np.ndarray]:
        """One step over the sessions of ``xs``: xs[sid] is the session's new host samples, or with ``src`` its runs
        (src_row, src_off, count) of that device array, at the session's input rate; the sessions in ``final`` end after
        them."""
        hop, sr = self.hop, self.sr
        ses = [(sid, self.sessions[sid], xs[sid]) for sid in xs]
        if src is None:                                   # host samples: the upload's sample block is the one source row
            counts = [len(x) for _, _, x in ses]
            starts = np.cumsum([0] + counts)
            runs = [[(0, int(a), n)] for a, n in zip(starts, counts)]
        else:
            runs = [x for _, _, x in ses]
            counts = [sum(n for _, _, n in r) for r in runs]
        # model-rate samples each session gains: its pushed samples, or the outputs of its input resampler that become
        # ready (all of them once it ends); rin: (plan, row, in_len, m0, count, row, m0) of the ring resampling
        gains, rin = [], []
        for (sid, s, _), n in zip(ses, counts):
            if s.in_sr is None:
                gains.append(n)
                continue
            n_out, n_ready = resample_span(s.in_sr, sr, s.raw_n + n)[:2]
            m1 = n_out if sid in final else n_ready
            gains.append(m1 - s.n_in)
            if m1 > s.n_in:
                rin.append((self.plans[(s.in_sr, sr)], s.row, s.raw_n + n if sid in final else STREAM_OPEN, s.n_in,
                            m1 - s.n_in, s.row, s.n_in))
        need = max([s.n_in + n - self._keep_from(s) for (_, s, _), n in zip(ses, gains)], default=0)
        if need > self.cap:
            cap = -(-int(need * 1.25) // hop) * hop
            self._grow(self.rows, cap, [(s.row, self._keep_from(s), s.n_in) for s in self.sessions.values()])
        need = max([s.raw_n + n - self._raw_keep(s) for (_, s, _), n in zip(ses, counts) if s.in_sr], default=0)
        if self.raw is not None and need > self.raw.shape[1]:
            live = [(s.row, self._raw_keep(s), s.raw_n) for s in self.sessions.values() if s.in_sr]
            self.raw = self._moved(self.raw, self.rows, -(-int(need * 1.25) // 1024) * 1024, live)
        # enrolling sessions: (session index, snapshot k of the step or 0); first: the items (in enr) of sessions whose
        # first snapshot becomes their source in this step
        enr = [(i, s.enroll.snapshot(s.n_in, s.n_in + n, hop)) for i, ((_, s, _), n) in enumerate(zip(ses, gains))
               if s.enroll is not None]
        first = [b for b, (i, k) in enumerate(enr) if k and not ses[i][1].has_src]
        no_src = {i for i, k in enr if not k and not ses[i][1].has_src}
        nE, nF, gin = len(enr), len(first), self.gin
        # the windows whose frames the step emits, (session index, lo, hi, e0, e1), and how they are converted
        wins, plan = self._plan(ses, gains, final, no_src)
        # splice segments: each run to the ring row (raw ring row when the session resamples its input) of its session,
        # at the session's next sample positions
        segs, rsegs = [], []
        for (_, s, _), r in zip(ses, runs):
            at, dst = (s.n_in, segs) if s.in_sr is None else (s.raw_n, rsegs)
            for row, off, n in r:
                if n:
                    dst.append((row, off, n, s.row, at))
                    at += n
        B, nS, nR, Ns = len(wins), len(segs), len(rsegs), (sum(counts) if src is None else 0)
        Nf = sum(e1 - e0 for _, _, _, e0, e1 in wins)
        # output side: the emitted frames of output-resampling sessions go to their output ring rows (osegs: splice
        # from the gathered frames) and their new output-rate samples are packed after the frames (rout, qn)
        emitted = [max([e1 for j, _, _, _, e1 in wins if j == i], default=s.emitted) for i, (_, s, _) in enumerate(ses)]
        osegs, at = [], 0
        for i, _, _, e0, e1 in wins:
            if ses[i][1].out_sr is not None:
                osegs.append((0, at * hop, (e1 - e0) * hop, ses[i][1].row, e0 * hop))
            at += e1 - e0
        rout, qn, No = [], [0] * len(ses), 0
        for i, (sid, s, _) in enumerate(ses):
            if s.out_sr is None:
                continue
            M = emitted[i] * hop
            n_out, n_ready = resample_span(sr, s.out_sr, M)[:2]
            qn[i] = (n_out if sid in final else n_ready) - s.out_n
            if qn[i] > 0:
                rout.append((self.plans[(sr, s.out_sr)], s.row, M if sid in final else STREAM_OPEN, s.out_n, qn[i], 0,
                             Nf * hop + No))
                No += qn[i]
        if self.orings is not None:
            need = max([emitted[i] * hop - self._out_keep(s) for i, (_, s, _) in enumerate(ses) if s.out_sr], default=0)
            if need > self.orings.shape[1]:
                live = [(s.row, self._out_keep(s), s.emitted * hop) for s in self.sessions.values() if s.out_sr]
                self.orings = self._moved(self.orings, self.rows, -(-int(need * 1.25) // 1024) * 1024, live)
        nO, nI, nQ = len(osegs), len(rin), len(rout)
        # packed upload (int64 words): the conversion's tables (``_pack``), the splice segments (5 words each), the raw
        # splice segments, the input resampling items (6 words each, then their plans as int32), the output splice
        # segments, the output resampling items, the encoder descriptors (4 words each) with the first snapshots' items
        # and embedding table rows, and the pushed samples (float32)
        o = self._plan_words(plan)
        o_r = o + 5 * nS
        o_i = o_r + 5 * nR
        o_o = o_i + 6 * nI + (nI + 1) // 2
        o_q = o_o + 5 * nO
        o_e = o_q + 6 * nQ + (nQ + 1) // 2
        o_s = o_e + 4 * nE + 2 * nF
        n_words = o_s + (Ns + 1) // 2
        if self._h2d_done is not None:
            self._h2d_done.synchronize()                  # the previous step's upload has left the pinned buffer
        pin = self._buf("pin", n_words, torch.int64, pinned=True)
        w = pin.numpy()
        self._pack(w, plan, ses, gains, final)
        for at, sg in ((o, segs), (o_r, rsegs), (o_o, osegs)):
            if sg:
                w[at:at + 5 * len(sg)] = np.asarray(sg, dtype=np.int64).reshape(-1)
        for at, it in ((o_i, rin), (o_q, rout)):
            if it:
                v = np.asarray(it, dtype=np.int64)
                w[at:at + 6 * len(it)] = v[:, 1:].T.reshape(-1)
                w[at + 6 * len(it):at + 6 * len(it) + (len(it) + 1) // 2].view(np.int32)[:len(it)] = v[:, 0]
        if nE:
            w[o_e:o_e + 4 * nE] = np.asarray([[ses[i][1].row, ses[i][1].row, ses[i][1].n_in + gains[i],
                                               k * ses[i][1].enroll.every_frames * hop] for i, k in enr],
                                             dtype=np.int64).reshape(-1)
            w[o_e + 4 * nE:o_e + 4 * nE + nF] = first
            w[o_e + 4 * nE + nF:o_s] = [ses[enr[b][0]][1].row for b in first]
        if Ns:
            w[o_s:].view(np.float32)[:Ns] = np.concatenate([x for _, _, x in ses])
        d = self._buf("up", n_words, torch.int64)
        d.copy_(pin, non_blocking=True)
        if self.cuda:
            self._h2d_done = torch.cuda.Event()
            self._h2d_done.record(torch.cuda.current_stream(self.dev))
        if nS or nR:
            source = d[o_s:].view(torch.float32)[:Ns].view(1, Ns) if src is None else src
        if nS:
            self._splice(source, d[o:o + 5 * nS].view(nS, 5), segs, self.rings)
        if nR:
            self._splice(source, d[o_r:o_r + 5 * nR].view(nR, 5), rsegs, self.raw)
        if nI:
            self._resample_rings(d, o_i, nI, self.raw, self.rings, max(it[4] for it in rin))
        res = {sid: np.zeros(0, dtype=np.float32) for sid, _, _ in ses}
        snaps = [b for b, (_, k) in enumerate(enr) if k]
        ybuf = self._buf("y", Nf * hop + No + (nE * gin if snaps else 0), torch.float32)
        if nE:                                            # after the splice and the resampling: the samples are in
            eout = ybuf[Nf * hop + No:Nf * hop + No + nE * gin].view(nE, gin) if snaps else \
                self._buf("e", nE * gin, torch.float32).view(nE, gin)
            M = max(enroll_new_frames(ses[i][1].n_in, ses[i][1].n_in + gains[i], hop, self.nfft) for i, _ in enr)
            self.native.reference_encoder_stream(self.rings, self.est, d[o_e:o_e + 4 * nE].view(nE, 4), M, out=eout)
            if nF:                                        # first snapshots are the sources of this step's windows
                self.se[0].index_copy_(0, d[o_e + 4 * nE + nF:o_s], eout.index_select(0, d[o_e + 4 * nE:o_e + 4 * nE + nF]))
        y = self._convert(d, plan, ses, {enr[b][0] for b in first}, ybuf[:Nf * hop].view(Nf, hop))
        if B:
            if nO:
                self._splice(y.view(1, Nf * hop), d[o_o:o_o + 5 * nO].view(nO, 5), osegs, self.orings)
            if nQ:
                self._resample_rings(d, o_q, nQ, self.orings, ybuf.view(1, -1), max(it[4] for it in rout))
        if B or snaps:
            host = self._buf("host", ybuf.numel(), torch.float32, pinned=True)
            host.copy_(ybuf, non_blocking=True)
            if self.cuda:
                torch.cuda.current_stream(self.dev).synchronize()
            y = host.numpy()
            at, per_ses = 0, {}
            for i, _, _, e0, e1 in wins:
                if ses[i][1].out_sr is None:
                    per_ses.setdefault(i, []).append(y[at * hop:(at + e1 - e0) * hop])
                at += e1 - e0
            for i, parts in per_ses.items():
                res[ses[i][0]] = np.concatenate(parts)
            at = Nf * hop
            for i, (sid, s, _) in enumerate(ses):
                if qn[i] > 0:
                    res[sid] = y[at:at + qn[i]].copy()
                    at += qn[i]
        for i, (_, s, _) in enumerate(ses):
            s.n_in += gains[i]
            s.raw_n += counts[i] if s.in_sr is not None else 0
            s.out_n += qn[i]
            s.emitted = emitted[i]
        for b in snaps:                                   # each snapshot takes effect after the step
            sid, s, _ = ses[enr[b][0]]
            se = torch.from_numpy(y[Nf * hop + No + b * gin:Nf * hop + No + (b + 1) * gin].copy())
            if s.has_src:
                self.retarget(sid, src_se=se, ramp_frames=s.enroll.ramp_frames)
            else:
                s.se[0], s.has_src = se, True
        return res

    # ------------------------------------------------------------------ the conversion part of a step
    def _plan(self, ses, gains: List[int], final: Set[int], skip: Set[int]):
        """(windows, plan) of a step whose sessions ``ses`` gain ``gains`` model-rate samples: the windows (session
        index, lo, hi, e0, e1) whose frames [e0, e1) the step emits, and what ``_pack`` and ``_convert`` take -- here the
        same windows, each converted whole with both halos.  Sessions in ``skip`` have nothing to convert with yet."""
        wins = []
        for i, ((sid, s, _), n) in enumerate(zip(ses, gains)):
            if i in skip:
                continue
            have = ready_frames(s.n_in + n, self.hop, self.nfft, sid in final)
            wins += [(i,) + w for w in stream_windows(s.emitted, have, self.W, self.H, sid in final)]
        return wins, wins

    @staticmethod
    def _tmax(wins) -> int:
        """Padded window length of a launch: the longest window rounded up to 16 frames (steady steps repeat it)."""
        return -(-max([hi - lo for _, lo, hi, _, _ in wins], default=1) // 16) * 16

    def _plan_words(self, wins) -> int:
        B = len(wins)
        return 8 * B + (B + 1) // 2 + sum(e1 - e0 for _, _, _, e0, e1 in wins)

    def _pack(self, w: np.ndarray, wins, ses, gains: List[int], final: Set[int]) -> None:
        """The conversion's tables at the front of the step's upload ``w``: row, lo, frames, stream length, seed,
        stream (0), embedding rows (2B), tau (float32), then the emitted frames' rows of the output."""
        B = len(wins)
        if not B:
            return
        nt, Tmax = (B + 1) // 2, self._tmax(wins)
        ii = np.asarray([i for i, _, _, _, _ in wins])
        rows = np.asarray([s.row for _, s, _ in ses], dtype=np.int64)[ii]
        lo = np.asarray([v[1] for v in wins], dtype=np.int64)
        w[0:B], w[B:2 * B], w[2 * B:3 * B] = rows, lo, [hi - l for _, l, hi, _, _ in wins]
        w[3 * B:4 * B] = [ses[i][1].n_in + gains[i] if ses[i][0] in final else STREAM_OPEN for i in ii]
        from .api import seed_array
        w[4 * B:5 * B] = seed_array([ses[i][1].seed for i in ii])
        w[5 * B:6 * B] = 0
        w[6 * B:7 * B], w[7 * B:8 * B] = rows, rows + self.rows
        w[8 * B:8 * B + nt].view(np.float32)[:B] = [ses[i][1].tau for i in ii]
        w[8 * B + nt:self._plan_words(wins)] = np.concatenate([b * Tmax + np.arange(e0 - l, e1 - l)
                                                                for b, (_, l, _, e0, e1) in enumerate(wins)])

    def _convert(self, d: torch.Tensor, wins, ses, fresh: Set[int], y: torch.Tensor) -> Optional[torch.Tensor]:
        """Spectrogram -> voice conversion -> emitted frames of the step's windows, from the tables ``_pack`` put at the
        front of the uploaded ``d``: the emitted frames go into ``y`` [Nf, hop], which is returned (None without
        windows).  ``fresh``: sessions whose source is the first enrollment snapshot of this step."""
        B = len(wins)
        if not B:
            return None
        hop, nt, Tmax, Nf = self.hop, (B + 1) // 2, self._tmax(wins), y.shape[0]
        spec = self._buf("spec", B * self.S * Tmax, torch.float32).view(B, self.S, Tmax)
        self.native.spectrogram_ring(self.rings, d[0:B], d[B:2 * B], d[2 * B:3 * B], d[3 * B:4 * B], Tmax, out=spec)
        g = torch.index_select(self.se.view(-1, self.gin), 0, d[6 * B:8 * B],
                               out=self._buf("g", 2 * B * self.gin, torch.float32).view(2 * B, self.gin))
        obuf = self._buf("o", B * Tmax * hop, torch.float32)
        per = max(1, SESSION_BATCH_FRAMES // Tmax)
        taus = d[8 * B:8 * B + nt].view(torch.float32)[:B]
        for b0 in range(0, B, per):
            b1 = min(B, b0 + per)
            items = {"seed": d[4 * B + b0:4 * B + b1], "stream": d[5 * B + b0:5 * B + b1],
                     "frame0": d[B + b0:B + b1], "tau": taus[b0:b1]}
            gs, gt = self._window_tracks(ses, wins, b0, b1, Tmax, (g[:B], g[B:]), fresh)
            self.native.voice_conversion(spec[b0:b1], d[2 * B + b0:2 * B + b1], gs, gt,
                                         ragged=True, latents=False, items=items,
                                         out=obuf[b0 * Tmax * hop:b1 * Tmax * hop])
        fo = 8 * B + nt
        return torch.index_select(obuf.view(B * Tmax, hop), 0, d[fo:fo + Nf], out=y)

    def _resample_rings(self, d: torch.Tensor, at: int, n: int, src: torch.Tensor, dst: torch.Tensor, max_count: int):
        """One ``ovc_resample_rings`` over the n items packed at word ``at`` of the step's upload ``d``."""
        v = [d[at + k * n:at + (k + 1) * n] for k in range(6)]
        plan = d[at + 6 * n:at + 6 * n + (n + 1) // 2].view(torch.int32)[:n]
        self.native.resample_rings(plan, src, v[0], v[1], v[2], v[3], dst, v[4], v[5], max_count)


# Halo of each stage of StagedSessions (frames on each side whose context a frame's value depends on).  The latent stack
# (posterior encoder, flow forward, flow reverse) sees +-96: the encoder's WN has 16 layers of kernel 5 at dilation 1
# (16 x 2 = 32), and each flow direction 4 couplings of 4 such layers (4 x 4 x 2 = 32); its other convs are 1x1.  The
# generator sees +-14: conv_pre (k 7: 3 frames), then per upsampling stage the ResBlock dilations (k 3/7/11 at 1, 3, 5)
# and the transposed conv, expressed in frames of the stage's input -- the figure the TTS window decode relies on.
LATENT_HALO_FRAMES = 96
GEN_HALO_FRAMES = 14


class StagedSessions(StreamingSessions):
    """``StreamingSessions`` converting in two stages, so the generator -- about 93 % of the converter's work -- no
    longer recomputes the whole converter's 2 x 128 halo frames.  Each session keeps its final latents (z_hat, the flow
    reverse's output) in a device ring of ``[inter_channels, cap]`` rows:

    * stage A (latent): windows of U = min(window_frames, 16) frames with ``LATENT_HALO_FRAMES`` (96) on each side
      (``stream_windows`` over the ready spectrogram frames); one ``ovc_spectrogram_ring`` over all of them, ragged
      latent-half calls (``NativeConverter.latent``) of up to ``SESSION_BATCH_FRAMES`` padded frames each, and one
      ``ovc_splice`` of their interiors into the latent rings;
    * stage B (generator): windows of ``window_frames`` frames with ``GEN_HALO_FRAMES`` (14) on each side over the final
      latent frames; one source-wrapping ``ovc_splice`` gathers them from the rings into a padded batch, ragged generator
      calls (``NativeConverter.generate``) convert it, and the emitted frames go out as in ``StreamingSessions``.

    Stage A runs before stage B in the same step, so a push that completes both emits in that step.  A window's geometry
    depends on absolute frames only and every item is converted at its own length, so a session's audio depends on its
    own stream alone -- not on its chunking nor on the sessions beside it -- and is within the streaming bound of
    ``convert`` on the whole clip (the tile geometry differs from ``StreamingConverter``'s, so it is not bit-identical to
    it).  The largest look-ahead, at the first frame of a stage-B window starting at e0, is U * ceil((e0 + W + 14) / U) +
    96 - e0 frames: W + 112 for every W that U divides (all W <= 16 and every multiple of 16), against W + 128 for
    ``StreamingSessions``.

    Everything else -- ``open`` (rates, enrollment), ``push``, ``push_device``, ``close``, ``discard``, ``retarget``,
    ``tone_track``, ``source_se``, ``state_samples`` -- is ``StreamingSessions``'.  The audio ring keeps the next stage-A
    window and the STFT support (plus the largest push), the latent ring the next stage-B window and the stage-A unit
    ahead of it; both are grow-only."""

    def __init__(self, converter, window_frames: int = 256, rates: Iterable[int] = ()):
        super().__init__(converter, window_frames, rates)
        self.U = min(self.W, 16)
        self.C = int(converter.hps.model.inter_channels)
        self.cap = self.hop * (self.U + 2 * LATENT_HALO_FRAMES + 8) + 4096
        self.rings = torch.zeros(0, self.cap, device=self.dev)
        self.lcap = self.U + self.W + 2 * GEN_HALO_FRAMES + 16          # latent frames per ring row; grows
        self.lrings = torch.zeros(0, self.lcap, device=self.dev)        # [rows * C, lcap]: session row r at r*C + c
        # channel c's splice segment of a latent window: the window's channel-0 segment plus (c, 0, 0, c, 0)
        coff = torch.zeros(1, self.C, 5, dtype=torch.int64)
        coff[0, :, 0] = coff[0, :, 3] = torch.arange(self.C)
        self._coff = coff.to(self.dev)

    def _keep_from(self, s: _Session) -> int:
        """First sample of the session's next stage-A window."""
        return max(0, (s.lat - LATENT_HALO_FRAMES) * self.hop - self.pad)

    def _grow(self, rows: int, cap: int, live: List[Tuple[int, int, int]]):
        if rows != self.rows:
            self.lrings = self._moved(self.lrings, rows * self.C, self.lcap, [])
        super()._grow(rows, cap, live)

    def _plan(self, ses, gains: List[int], final: Set[int], skip: Set[int]):
        """Stage-A windows over the ready spectrogram frames, then stage-B windows over the latent frames stage A leaves
        final (ended: all of them once the session is closed).  Grows the latent rings when a session's step would write
        past what it still reads: from its next stage-B window's left halo to its new latent end."""
        winsA, winsB, lat = [], [], {}
        for i, ((sid, s, _), n) in enumerate(zip(ses, gains)):
            if i in skip:
                continue
            end = sid in final
            have = ready_frames(s.n_in + n, self.hop, self.nfft, end)
            wa = stream_windows(s.lat, have, self.U, LATENT_HALO_FRAMES, end)
            lat[i] = wa[-1][3] if wa else s.lat
            winsA += [(i,) + w for w in wa]
            winsB += [(i,) + w for w in stream_windows(s.emitted, lat[i], self.W, GEN_HALO_FRAMES, end and lat[i] == have)]
        need = max([v - max(0, ses[i][1].emitted - GEN_HALO_FRAMES) for i, v in lat.items()], default=0)
        if need > self.lcap:
            cap = -(-int(need * 1.25) // 16) * 16
            live = [(s.row * self.C + c, max(0, s.emitted - GEN_HALO_FRAMES), s.lat)
                    for s in self.sessions.values() if s.lat > max(0, s.emitted - GEN_HALO_FRAMES) for c in range(self.C)]
            self.lrings = (self._moved(self.lrings, self.rows * self.C, cap, live) if live
                           else torch.zeros(self.rows * self.C, cap, device=self.dev))
            self.lcap = cap
        return winsB, (winsA, winsB, lat)

    def _plan_words(self, plan) -> int:
        winsA, winsB, _ = plan
        BA, BB = len(winsA), len(winsB)
        return 13 * BA + (BA + 1) // 2 + 7 * BB + sum(e1 - e0 for _, _, _, e0, e1 in winsB)

    def _pack(self, w: np.ndarray, plan, ses, gains: List[int], final: Set[int]) -> None:
        """Stage A: row, lo, frames, stream length, seed, stream (0), embedding rows (2 BA), tau (float32), the channel-0
        scatter segments of the interiors (5 words each).  Stage B: the channel-0 gather segments (5 words each), frames,
        target embedding rows, the emitted frames' rows of the output."""
        from .api import seed_array
        winsA, winsB, _ = plan
        BA, BB, C = len(winsA), len(winsB), self.C
        if BA:
            ii = [i for i, _, _, _, _ in winsA]
            rows = np.asarray([ses[i][1].row for i in ii], dtype=np.int64)
            w[0:BA], w[BA:2 * BA] = rows, [lo for _, lo, _, _, _ in winsA]
            w[2 * BA:3 * BA] = [hi - lo for _, lo, hi, _, _ in winsA]
            w[3 * BA:4 * BA] = [ses[i][1].n_in + gains[i] if ses[i][0] in final else STREAM_OPEN for i in ii]
            w[4 * BA:5 * BA] = seed_array([ses[i][1].seed for i in ii])
            w[5 * BA:6 * BA] = 0
            w[6 * BA:7 * BA], w[7 * BA:8 * BA] = rows, rows + self.rows
            w[8 * BA:8 * BA + (BA + 1) // 2].view(np.float32)[:BA] = [ses[i][1].tau for i in ii]
            o = 8 * BA + (BA + 1) // 2
            w[o:o + 5 * BA] = np.asarray([(a * C, e0 - lo, e1 - e0, ses[i][1].row * C, e0)
                                          for a, (i, lo, _, e0, e1) in enumerate(winsA)], dtype=np.int64).reshape(-1)
        if BB:
            o, Tmax = 13 * BA + (BA + 1) // 2, self._tmax(winsB)
            rows = np.asarray([ses[i][1].row for i, _, _, _, _ in winsB], dtype=np.int64)
            w[o:o + 5 * BB] = np.asarray([(r * C, lo, hi - lo, b * C, 0) for b, (r, (_, lo, hi, _, _))
                                          in enumerate(zip(rows, winsB))], dtype=np.int64).reshape(-1)
            w[o + 5 * BB:o + 6 * BB] = [hi - lo for _, lo, hi, _, _ in winsB]
            w[o + 6 * BB:o + 7 * BB] = rows + self.rows
            w[o + 7 * BB:self._plan_words(plan)] = np.concatenate([b * Tmax + np.arange(e0 - lo, e1 - lo)
                                                                    for b, (_, lo, _, e0, e1) in enumerate(winsB)])

    def _segs(self, base: torch.Tensor, n: int, name: str) -> torch.Tensor:
        """The [n * C, 5] per-channel splice segments of n latent windows from their channel-0 segments ``base``."""
        out = self._buf(name, n * self.C * 5, torch.int64).view(n, self.C, 5)
        torch.add(base.view(n, 1, 5), self._coff, out=out)
        return out.view(n * self.C, 5)

    def _convert(self, d: torch.Tensor, plan, ses, fresh: Set[int], y: torch.Tensor) -> Optional[torch.Tensor]:
        """Stage A, then stage B, from the tables ``_pack`` put at the front of ``d``; advances each session's latent
        end.  Returns ``y`` [Nf, hop] holding the emitted frames, or None when stage B has no window."""
        winsA, winsB, lat = plan
        BA, BB, C, hop, gin = len(winsA), len(winsB), self.C, self.hop, self.gin
        if BA:
            nt, Tmax = (BA + 1) // 2, self._tmax(winsA)
            spec = self._buf("spec", BA * self.S * Tmax, torch.float32).view(BA, self.S, Tmax)
            self.native.spectrogram_ring(self.rings, d[0:BA], d[BA:2 * BA], d[2 * BA:3 * BA], d[3 * BA:4 * BA], Tmax,
                                         out=spec)
            g = torch.index_select(self.se.view(-1, gin), 0, d[6 * BA:8 * BA],
                                   out=self._buf("g", 2 * BA * gin, torch.float32).view(2 * BA, gin))
            z = self._buf("za", BA * C * Tmax, torch.float32).view(BA, C, Tmax)
            per = max(1, SESSION_BATCH_FRAMES // Tmax)
            taus = d[8 * BA:8 * BA + nt].view(torch.float32)[:BA]
            for b0 in range(0, BA, per):
                b1 = min(BA, b0 + per)
                items = {"seed": d[4 * BA + b0:4 * BA + b1], "stream": d[5 * BA + b0:5 * BA + b1],
                         "frame0": d[BA + b0:BA + b1], "tau": taus[b0:b1]}
                gs, gt = self._window_tracks(ses, winsA, b0, b1, Tmax, (g[:BA], g[BA:]), fresh)
                self.native.latent(spec[b0:b1], d[2 * BA + b0:2 * BA + b1], gs, gt, items=items, out=z[b0:b1])
            o = 8 * BA + nt
            self._splice(z.view(BA * C, Tmax), self._segs(d[o:o + 5 * BA], BA, "sega"), None, self.lrings)
        for i, v in lat.items():
            ses[i][1].lat = v
        if not BB:
            return None
        o, Tmax, Nf = 13 * BA + (BA + 1) // 2, self._tmax(winsB), y.shape[0]
        z = self._buf("zb", BB * C * Tmax, torch.float32).view(BB, C, Tmax)
        self._splice(self.lrings, self._segs(d[o:o + 5 * BB], BB, "segb"), None, z.view(BB * C, Tmax), src_wrap=True)
        g = torch.index_select(self.se.view(-1, gin), 0, d[o + 6 * BB:o + 7 * BB],
                               out=self._buf("gb", BB * gin, torch.float32).view(BB, gin))
        obuf = self._buf("o", BB * Tmax * hop, torch.float32)
        per = max(1, SESSION_BATCH_FRAMES // Tmax)
        for b0 in range(0, BB, per):
            b1 = min(BB, b0 + per)
            gt = self._window_tracks(ses, winsB, b0, b1, Tmax, (None, g), fresh, sides=(1,))[0]
            self.native.generate(z[b0:b1], d[o + 5 * BB + b0:o + 5 * BB + b1], gt,
                                 out=obuf[b0 * Tmax * hop:b1 * Tmax * hop])
        fo = o + 7 * BB
        return torch.index_select(obuf.view(BB * Tmax, hop), 0, d[fo:fo + Nf], out=y)


class _CloneSession:
    __slots__ = ("tts_keys", "conv_keys", "said", "unencoded", "plans", "length", "ended", "checked", "ss_id", "out_sr",
                 "tokens", "tokens_encoded")

    def __init__(self, tts_keys: dict, conv_keys: dict, out_sr: Optional[int] = None):
        self.tts_keys, self.conv_keys, self.out_sr = tts_keys, conv_keys, out_sr
        self.said = 0                                     # sentences said so far: the next one is sentence `said`
        self.unencoded = 0                                # said sentences still waiting for the encode
        self.tokens = 0                                   # tokens said so far: the next sentence starts at this position
        self.tokens_encoded = 0                           # tokens of the sentences already encoded
        self.plans: deque = deque()                       # TTS windows to decode: (pool row, lo, hi, e0, e1, gap, last)
        self.length = 0                                   # samples of the encoded sentences and their gaps
        self.ended = False
        self.checked = False                              # ended, fully encoded and long enough to convert
        self.ss_id: Optional[int] = None                  # its StreamingSessions session, from its first audio on


class CloneSessions:
    """Live text-to-cloned-voice sessions: requests open, receive text one sentence at a time and end while the others run,
    and every ``step`` advances all of them with one batched launch sequence.

    ``open`` takes the keys of a ``ToneColorConverter.clone_batch`` request other than its text and returns the session's
    id; ``say(sid, text=... | ids=...)`` queues sentences through the text front end ``tts_batch`` uses; ``end`` marks
    that no more text follows; ``cancel`` drops a session at once.  Sentence j of a session (counted across ``say``
    calls) draws at (seed, stream j) with the session's parameters, as sentence j of the one-shot request does, so a
    session's chunks concatenate to those of ``clone_stream_batch(tts, [request])`` for the request holding the same
    sentences and keys, bit for bit, whenever its text arrives and whatever runs beside it.

    A ``step`` is at most:
      1. ONE ragged ``tts_encode`` of every sentence said since the last step (one host sync, for the frame counts),
         written by ONE ``ovc_tts_encode_state_rows`` into free rows of a ``TtsPool`` shared by all sessions.  The pool
         is grow-only (a larger token pitch re-pitches it once, one more copy) and a sentence's row is freed once its
         last window is decoded.
      2. ONE ``tts_decode_windows`` over the pool: per session, the next TTS windows (``plan_tts_windows``;
         ``first_window_frames`` for its first sentence only) until its converter can emit a window or its encoded text
         runs out.
      3. ONE ``StreamingSessions.push_device`` of every session's window interiors and 50 ms / speed gaps, closing the
         sessions that have ended and whose last gap is written (``close`` alone when a session ended after that).
    A session waiting for text costs nothing; a step in which nothing can advance returns {} and launches nothing.

    Bad input is refused where its session can be named: keys in ``open``, token and speaker ids in ``say`` (the session
    keeps what it had said), so the shared encode of a step only sees checked text.  An encode that still fails takes no
    pool rows and keeps the text for the next step.  A session whose whole utterance turns out too short to convert
    raises ValueError naming it in the step where its length becomes known, before that step's decode; it is cancelled
    and the others continue on the next ``step``.  Both
    models must be on one device and at one sampling rate (ValueError here)."""

    OPEN_KEYS = ("speaker", "src_se", "tgt_se", "tau", "seed", "convert_seed", "speed", "noise_scale", "noise_scale_w",
                 "sdp_ratio")

    def __init__(self, converter, tts, window_frames: int = 256, first_window_frames: int = 32, label: str = "session",
                 output_rates: Iterable[int] = ()):
        """``label``: how errors name a session ("session 3"); ``clone_stream_batch`` passes "request".
        ``output_rates``: the rates other than the model's that ``open(output_sr=)`` accepts (``StreamingSessions``
        ``rates``: the converter side is made here, with their filter banks, rather than with the first audio)."""
        W, W1 = int(window_frames), int(first_window_frames)
        if W < 1 or W1 < 1:
            raise ValueError(f"window_frames ({W}) and first_window_frames ({W1}) must be >= 1")
        sr = int(converter.hps.data.sampling_rate)
        if int(tts.hps.data.sampling_rate) != sr:
            raise ValueError(f"the TTS model runs at {tts.hps.data.sampling_rate} Hz and the converter at {sr} Hz: "
                             f"streaming text to cloned voice needs one rate (clone_batch resamples)")
        converter._check_same_device(tts)
        self.conv, self.tts, self.W, self.W1, self.sr, self.label = converter, tts, W, W1, sr, label
        self.output_rates = tuple(output_rates)
        self.hop, self.nfft = converter.hps.data.hop_length, converter.hps.data.filter_length
        self.H = converter.HALO_FRAMES
        self.sessions: Dict[int, _CloneSession] = {}
        self.next_id = 0
        self.pending: List[Tuple[int, List[int]]] = []   # (session, token ids) said since the last encode, in order
        # beside each pending sentence: None, or (say number, target frames), shared by the sentences of one
        # say(duration=), which the encode fits as one group
        self.pending_fit: List[Optional[Tuple[int, int]]] = []
        self.says = 0
        self.ss: Optional[StreamingSessions] = None       # the converter side, made with the first audio
        if self.output_rates:                             # ... or here, where its filter banks may wait for the device
            self.ss = StreamingSessions(converter, window_frames=W, rates=self.output_rates)
        self.pool = None                                  # api.TtsPool, made with the first encode
        self.free_rows: List[int] = []
        self.rows = 0                                     # pool rows handed out so far
        # host side of each pool row: decoded frames, decode key, stream and noise scale of its sentence
        self.row_frames: List[int] = []
        self.row_keys: List[int] = []
        self.row_streams: List[int] = []
        self.row_noise: List[float] = []
        self._fresh: List[Tuple[object, List[Tuple[int, int]]]] = []   # (encode state, [(its row i, pool row)]) whose
                                                                          # decode keys are not in the row lists yet

    # ------------------------------------------------------------------ sessions
    def open(self, speaker, src_se=None, tgt_se=None, tau: float = 0.3, seed: Optional[int] = None,
             convert_seed: Optional[int] = None, speed: float = 1.0, noise_scale: float = 0.667,
             noise_scale_w: float = 0.6, sdp_ratio: float = 0.2, output_sr: Optional[int] = None) -> int:
        """Start a session and return its id.  The keys are those of a ``clone_batch`` request, validated as it
        validates them, and the noise parameters as the encode checks them (ValueError naming the session); ``seed`` /
        ``convert_seed`` default to draws from torch's generator.  The speaker id is checked against the checkpoint
        with the session's first ``say``.  ``output_sr``: the rate of the returned audio, the model's or one of
        ``output_rates`` (None: the model's)."""
        from .api import check_per_item
        q = dict(speaker=speaker, src_se=src_se, tgt_se=tgt_se, tau=tau, seed=seed, convert_seed=convert_seed,
                 speed=speed, noise_scale=noise_scale, noise_scale_w=noise_scale_w, sdp_ratio=sdp_ratio)
        who = f"{self.label} {self.next_id}"
        declared = self.ss.rates if self.ss is not None else ()
        if output_sr is not None and (isinstance(output_sr, bool) or int(output_sr) != output_sr
                                      or int(output_sr) not in (self.sr,) + declared):
            raise ValueError(f"{who}: output_sr={output_sr!r}: sessions return audio at the model's rate ({self.sr} Hz) "
                             f"or at a rate declared with output_rates= (declared: "
                             f"{', '.join(map(str, declared)) or 'none'})")
        tts_keys = self.tts._request_keys(q, who)
        for name in ("noise_scale", "noise_scale_w", "sdp_ratio"):
            check_per_item([tts_keys[name]], 1, f"{who}: {name}")
        conv_keys = self.conv._clone_keys(q, who)
        sid = self.next_id
        self.next_id += 1
        self.sessions[sid] = _CloneSession(tts_keys, conv_keys, None if output_sr is None else int(output_sr))
        return sid

    def _session(self, sid) -> _CloneSession:
        s = self.sessions.get(sid)
        if s is None:
            raise ValueError(f"unknown or closed {self.label} {sid!r}")
        return s

    def say(self, sid: int, text: Optional[str] = None, ids: Optional[Sequence[Sequence[int]]] = None,
            language: str = "English", duration: Optional[float] = None) -> None:
        """Queue sentences for session ``sid``: ``ids`` (token-id lists, one per sentence) or ``text`` through the TTS
        model's front end.  They are encoded in the next ``step``.  ValueError for an unknown or ended session, no
        sentences, a token id outside the vocabulary or a session speaker outside the checkpoint's speakers
        (``NativeSynthesizer.check_tts_input``, the encode's own check); the session keeps what it had said before.

        ``duration`` (seconds) fits these sentences and their 50 ms / speed gaps to that length, as a ``tts_batch``
        request with ``duration`` is fitted (``BaseSpeakerTTS.fit_target``): they form one fit group of the step's
        encode, which fits the groups of every session at once.  ValueError for a duration that is not positive and
        finite or too short for the gaps and one frame per sentence."""
        ids = self._sentences(sid, text, ids, language)
        target = None
        if duration is not None:
            who = f"{self.label} {sid}"
            target = self.tts.fit_target(self.tts._check_duration(duration, who), len(ids),
                                         self.sessions[sid].tts_keys["speed"], True, who)
        flat = [t for q in ids for t in q]
        keys = self.sessions[sid].tts_keys
        try:
            if keys["speaker"] is None:
                self.tts.model.check_tts_input(torch.as_tensor(flat or [0], dtype=torch.int64), None, need_sid=False)
            else:
                self.tts.model.check_tts_input(torch.as_tensor(flat or [0], dtype=torch.int64),
                                               torch.as_tensor([keys["speaker"]], dtype=torch.int64))
        except ValueError as e:
            raise ValueError(f"{self.label} {sid}: {e}") from None
        e, n = keys["g"], self.sessions[sid].tokens + len(flat)
        if torch.is_tensor(e) and e.dim() == 2 and n > e.shape[1]:
            raise ValueError(f"{self.label} {sid}: its per-token speaker tensor has {e.shape[1]} columns, the session "
                             f"would reach {n} tokens")
        self._queue(sid, ids, target)

    def _sentences(self, sid, text, ids, language) -> List[List[int]]:
        s = self._session(sid)
        if s.ended:
            raise ValueError(f"{self.label} {sid} has ended: it takes no more text")
        if ids is None:
            if text is None:
                raise ValueError("say needs text or ids")
            ids = self.tts._sentences(text, language)
        ids = [list(q) for q in ids]
        if not ids:
            raise ValueError(f"{self.label} {sid}: no sentences to say")
        return ids

    def _queue(self, sid: int, ids: List[List[int]], target: Optional[int] = None) -> None:
        """``say`` after its checks (``target``: the frames to fit the sentences to, or None).  ``clone_stream_batch``
        queues here: its eager encode checks every sentence of the call before the generator is returned, so a bad
        request fails the whole call and no step ever runs."""
        s = self.sessions[sid]
        fit = None if target is None else (self.says, int(target))
        self.says += 1
        self.pending += [(sid, q) for q in ids]
        self.pending_fit += [fit] * len(ids)
        s.said += len(ids)
        s.unencoded += len(ids)
        s.tokens += sum(len(q) for q in ids)

    def end(self, sid: int) -> None:
        """No more text for session ``sid``: it closes once its audio is out."""
        s = self._session(sid)
        if s.ended:
            raise ValueError(f"{self.label} {sid} has already ended")
        s.ended = True

    def cancel(self, sid: int) -> None:
        """Drop session ``sid`` now: its queued text, pool rows and converter row are freed; it returns nothing more."""
        s = self._session(sid)
        keep = [i for i, (o, _) in enumerate(self.pending) if o != sid]
        self.pending, self.pending_fit = [self.pending[i] for i in keep], [self.pending_fit[i] for i in keep]
        self.free_rows += sorted({p[0] for p in s.plans})
        if s.ss_id is not None:
            self.ss.discard([s.ss_id])
        del self.sessions[sid]

    @property
    def pool_rows_in_use(self) -> int:
        return self.rows - len(self.free_rows)

    # ------------------------------------------------------------------ one step
    def encode_pending(self) -> None:
        """The encode half of ``step``: one ragged encode of every sentence said since the last step into free pool rows,
        then the length check of every session whose utterance is now complete (ValueError naming the first one too
        short, after cancelling each such session)."""
        if self.pending:
            self._encode()
        bad = []
        for sid, s in self.sessions.items():
            if s.ended and not s.unencoded and not s.checked:
                try:
                    self.conv._check_clone_lengths([s.length], None, names=[f"{self.label} {sid}"])
                    s.checked = True
                except ValueError as e:
                    bad.append((sid, e))
        for sid, _ in bad:
            self.cancel(sid)
        if bad:
            raise bad[0][1]

    def _encode(self) -> None:
        from .api import TTS_HALO_FRAMES, TtsPool, plan_tts_windows
        tts = self.tts
        seqs, spk, spk_rows = [q for _, q in self.pending], [], []
        kw = {"seeds": [], "streams": [], "noise_scale": [], "noise_scale_w": [], "length_scale": [], "sdp_ratio": []}
        nth: Dict[int, int] = {}
        at: Dict[int, int] = {}                           # next token position of each session in this encode
        fit: List[List[int]] = []                         # [row0, row1, target] of each say(duration=) in the encode
        for i, f in enumerate(self.pending_fit):
            if f is not None:
                if fit and fit[-1][1] == i and self.pending_fit[i - 1] == f:
                    fit[-1][1] = i + 1
                else:
                    fit.append([i, i + 1, f[1]])
        if fit:
            kw["fit"] = fit
        for sid, q in self.pending:
            s = self.sessions[sid]
            j = s.said - s.unencoded + nth.get(sid, 0)    # the sentence's number in its session
            nth[sid] = nth.get(sid, 0) + 1
            o = at.get(sid, s.tokens_encoded)             # o_j: its first token's position in the session's stream
            at[sid] = o + len(q)
            spk.append(0 if s.tts_keys["speaker"] is None else s.tts_keys["speaker"])
            spk_rows.append((s.tts_keys["speaker"], s.tts_keys["g"], o, len(q)))
            kw["seeds"].append(s.tts_keys["seed"])
            kw["streams"].append(j)
            tts._sentence_params(s.tts_keys, kw)
        # free rows first, then new ones; they are taken only once the encode has gone through
        take = self.free_rows[:len(seqs)]
        new = list(range(self.rows, self.rows + len(seqs) - len(take)))
        rows = take + new
        if self.pool is None:
            self.pool = TtsPool(tts.model.native, tts.model.device)
        x, lens = tts._pad_ids(seqs)
        g = tts._speaker_rows(spk_rows, x.shape[1])
        if g is not None:
            kw["g"] = g
        state = tts.model.tts_encode(x, lens, sid=torch.as_tensor(spk, dtype=torch.int64), pool=self.pool, rows=rows, **kw)
        del self.free_rows[:len(take)]
        self.rows += len(new)
        for lst, v in ((self.row_frames, 0), (self.row_keys, 0), (self.row_streams, 0), (self.row_noise, 0.0)):
            lst += [v] * len(new)
        self._fresh.append((state, list(enumerate(rows))))
        for i, ((sid, _), row) in enumerate(zip(self.pending, rows)):
            s = self.sessions[sid]
            frames = state.frames[i]
            self.row_frames[row] = frames
            wins = plan_tts_windows(frames, self.W1 if kw["streams"][i] == 0 else self.W, self.W, TTS_HALO_FRAMES)
            gap = int((self.sr * 0.05) / s.tts_keys["speed"])
            s.plans += [(row, lo, hi, e0, e1, gap if k == len(wins) - 1 else 0, k == len(wins) - 1)
                        for k, (lo, hi, e0, e1) in enumerate(wins)]
            s.length += self.hop * frames + gap
            s.unencoded -= 1
            s.tokens_encoded += len(seqs[i])
        self.pending, self.pending_fit = [], []

    @torch.no_grad()
    def step(self) -> Dict[int, np.ndarray]:
        """Advance every session that can advance; returns {sid: float32 chunk} for each session that produced audio.
        Sessions that have ended and whose audio is all out are closed (and forgotten) here."""
        from .api import TtsState
        self.encode_pending()
        hop, ss = self.hop, self.ss
        wins, runs, closing, done_rows = [], {}, [], []
        for sid, s in self.sessions.items():
            if s.plans:
                st = None if s.ss_id is None else ss.sessions[s.ss_id]
                n_in, emitted = (0, 0) if st is None else (st.n_in, st.emitted)
                r = runs[sid] = []
                while s.plans:
                    row, lo, hi, e0, e1, gap, last = s.plans.popleft()
                    r += [(len(wins), (e0 - lo) * hop, (e1 - e0) * hop)] + ([(-1, 0, gap)] if gap else [])
                    wins.append((row, lo, hi - lo))
                    if last:
                        done_rows.append(row)
                    n_in += (e1 - e0) * hop + gap
                    if ready_frames(n_in, hop, self.nfft, False) >= emitted + self.W + self.H:
                        break
            if s.checked and not s.plans:
                closing.append(sid)
                runs.setdefault(sid, [])
        if not runs:
            return {}
        if self.ss is None:
            self.ss = ss = StreamingSessions(self.conv, window_frames=self.W)
        for sid in runs:
            s = self.sessions[sid]
            if s.ss_id is None:
                c = s.conv_keys
                s.ss_id = ss.open(c["src_se"], c["tgt_se"], tau=c["tau"], seed=c["convert_seed"], output_sr=s.out_sr)
        sids = {sid: self.sessions[sid].ss_id for sid in runs}
        if wins:
            for enc, pairs in self._fresh:               # each row's decode key, stream and noise scale, as encoded
                for i, row in pairs:
                    self.row_keys[row], self.row_streams[row] = enc.dec_keys[i], enc.dec_streams[i]
                    self.row_noise[row] = enc.dec_noise_scale[i]
            self._fresh = []
            state = TtsState(self.pool.stats, self.pool.cum, self.pool.g, self.pool.y_lengths, self.row_frames,
                             self.row_keys, self.row_streams, self.row_noise)
            o, _ = self.tts.model.tts_decode_windows(state, wins)
            out = ss.push_device({sids[sid]: r for sid, r in runs.items()}, o, close=[sids[sid] for sid in closing])
        else:
            out = ss.close([sids[sid] for sid in closing])
        self.free_rows += done_rows                       # reused by a later encode, which the stream orders after
        for sid in closing:
            del self.sessions[sid]
        return {sid: out[sids[sid]] for sid in runs if len(out[sids[sid]])}
