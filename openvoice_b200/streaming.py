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
"""
from typing import Callable, Optional

import numpy as np
import torch

from ._native import STREAM_OPEN, resample_span


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


class StreamingConverter:
    def __init__(self, converter, src_se, tgt_se, tau: float = 0.3, window_frames: int = 256,
                 noise_fn: Optional[Callable[[int, int], torch.Tensor]] = None, seed: Optional[int] = None,
                 input_sr: Optional[int] = None, output_sr: Optional[int] = None, request_seed: Optional[int] = None):
        """``converter``: a ToneColorConverter.  ``noise_fn(t0, t1) -> [inter_channels, t1 - t0]`` supplies the noise of
        absolute frames [t0, t1) (tests pass slices of one tensor); default: a seeded device generator.
        ``input_sr`` / ``output_sr``: rates of the pushed and of the returned audio when they are not the model's
        (``StreamingResampler`` on each side; None: the model's rate).
        ``request_seed``: the request's own key, as ``ToneColorConverter.convert(seed=...)`` takes it: each window draws
        its noise in-kernel at its absolute frames, so the stream gives ``convert(seed=request_seed)`` and no noise is
        kept.  It excludes ``noise_fn`` and ``seed`` (ValueError)."""
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
        self.src = converter._stack_se(src_se, 1)
        self.tgt = converter._stack_se(tgt_se, 1)
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
        if final:
            upto = self.n_in // hop
        else:
            upto = max(0, (self.n_in + pad - self.nfft) // hop + 1)
            upto = min(upto, self.n_in // hop)
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

    def _convert_window(self, e0: int, e1: int, t_end: Optional[int]) -> np.ndarray:
        """Samples of frames [e0, e1): one ragged batch-1 call over [e0 - H, e1 + H) clipped to the stream."""
        lo = max(0, e0 - self.H)
        hi = e1 + self.H if t_end is None else min(t_end, e1 + self.H)
        sp = self.spec[:, :, lo - self.f0: hi - self.f0].contiguous()
        lens = torch.tensor([hi - lo], dtype=torch.int64, device=self.dev)
        if self.request_seed is None:
            nz = self.noise[None, :, lo - self.f0: hi - self.f0].contiguous()
            o, _, _ = self.conv.model.voice_conversion(sp, lens, self.src, self.tgt, tau=self.tau, noise=nz, ragged=True,
                                                       latents=False)
        else:
            o, _, _ = self.conv.model.voice_conversion(sp, lens, self.src, self.tgt, tau=self.tau, ragged=True,
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
        y = self._flush() if self.rs_in is None else np.concatenate([self._push(self.rs_in.flush()), self._flush()])
        return y if self.rs_out is None else np.concatenate([self.rs_out.push(y), self.rs_out.flush()])

    def _push(self, x: np.ndarray) -> np.ndarray:
        self.audio = np.concatenate([self.audio, x])
        self.n_in += len(x)
        self._extend_spec(final=False)
        outs = []
        have = self.f0 + self.spec.shape[2]
        while self.emitted + self.W + self.H <= have:
            outs.append(self._convert_window(self.emitted, self.emitted + self.W, None))
        return np.concatenate(outs) if outs else np.zeros(0, dtype=np.float32)

    def _flush(self) -> np.ndarray:
        self.closed = True
        T = self.n_in // self.hop
        if T < 1 or self.n_in <= self.pad:
            raise ValueError("audio too short")       # shorter than one hop / the STFT reflect padding, like convert
        self._extend_spec(final=True)
        outs = []
        while self.emitted < T:
            e1 = min(T, self.emitted + self.W)
            outs.append(self._convert_window(self.emitted, e1, T))
        return np.concatenate(outs) if outs else np.zeros(0, dtype=np.float32)
