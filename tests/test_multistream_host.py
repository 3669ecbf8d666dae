"""Host logic of StreamingSessions on the CPU, with a stand-in converter: ring bookkeeping and reflect rules against the
oracle STFT, window scheduling against StreamingConverter, the number of native calls per step, and the refusals."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import vc_oracle as O

HOP, NFFT, PAD, GIN, SR = 256, 1024, 384, 8, 22050
KERN = torch.linspace(0.2, 1.0, 201, dtype=torch.float64)[None, None]


def fake_vc(spec, length, seed, frame0, tau):
    """Stand-in voice conversion of one item: frame t of the output depends on frames t-100 .. t+100 of its own length
    (zero padding past it) and on a per-(seed, absolute frame) noise value, so a wrong frame, offset, halo or seed shows."""
    t = torch.arange(frame0, frame0 + length, dtype=torch.float64)
    f = spec[:8, :length].double().mean(0) + tau * torch.sin((seed % 1009) * 0.1 + 0.7 * t)
    g = F.conv1d(f[None, None], KERN, padding=100)[0, 0]
    return (g[:, None] * torch.linspace(1.0, 2.0, HOP, dtype=torch.float64)[None]).reshape(-1).float()


def ring_frames(rings, row, lo, frames, slen):
    """The rule of ovc_spectrogram_ring, spelled out: the padded-signal segment of frames [lo, lo + frames) read from the
    ring with reflection at the start, and at the end once the stream is closed, through the oracle's STFT."""
    from openvoice_b200._native import STREAM_OPEN
    cap = rings.shape[1]
    idx = np.arange(lo * HOP - PAD, (lo + frames - 1) * HOP - PAD + NFFT)
    idx = np.abs(idx)
    if slen != STREAM_OPEN:
        idx = np.where(idx >= slen, 2 * (slen - 1) - idx, idx)
    seg = rings[row, torch.from_numpy(idx % cap)]
    s = torch.stft(seg[None], NFFT, hop_length=HOP, win_length=NFFT, window=torch.hann_window(NFFT), center=False,
                   onesided=True, return_complex=True)
    return torch.sqrt(torch.view_as_real(s).pow(2).sum(-1) + 1e-6)[0]


class FakeNative:
    def __init__(self):
        self.calls = {"spectrogram_ring": 0, "voice_conversion": 0, "spectrogram": 0}

    def spectrogram(self, wav, wlen):
        self.calls["spectrogram"] += 1
        T = wav.shape[1] // HOP
        return O.spectrogram(wav)[:, :, :T], torch.tensor([T])

    def spectrogram_ring(self, rings, row, lo, frames, slen, Tmax, out=None):
        self.calls["spectrogram_ring"] += 1
        out.zero_()
        for b in range(row.numel()):
            n = int(frames[b])
            out[b, :, :n] = ring_frames(rings, int(row[b]), int(lo[b]), n, int(slen[b]))
        return out

    def voice_conversion(self, spec, lens, gs, gt, ragged=True, latents=False, items=None, out=None):
        self.calls["voice_conversion"] += 1
        B, _, T = spec.shape
        o = out.view(B, HOP * T)
        o.zero_()
        seeds = items["seed"].numpy().view(np.uint64)
        for b in range(B):
            n = int(lens[b])
            o[b, :HOP * n] = fake_vc(spec[b], n, int(seeds[b]), int(items["frame0"][b]), float(items["tau"][b]))
        return o.view(B, 1, -1), None


class FakeModel:
    def __init__(self):
        self.native = FakeNative()

    def voice_conversion(self, sp, lens, src, tgt, tau=0.3, ragged=True, latents=False, seeds=None, frame0=None):
        o = fake_vc(sp[0], int(lens[0]), seeds[0], frame0[0], tau)
        return o[None, None], None, None


class FakeConverter:
    class hps:
        class data:
            hop_length, filter_length, sampling_rate = HOP, NFFT, SR

        class model:
            inter_channels, gin_channels = 4, GIN
    HALO_FRAMES = 128
    device = "cpu"

    def __init__(self):
        self.model = FakeModel()

    def _stack_se(self, se, n):
        return se.reshape(1, -1)


def wave(n, seed):
    return np.random.default_rng(seed).standard_normal(n).astype(np.float32)


def se(seed):
    return torch.randn(1, GIN, 1, generator=torch.Generator().manual_seed(seed))


def converter_stream(wav, sizes, W, seed, tau):
    from openvoice_b200.streaming import StreamingConverter
    sc = StreamingConverter(FakeConverter(), se(0), se(1), tau=tau, window_frames=W, request_seed=seed)
    outs, pos, i = [], 0, 0
    while pos < len(wav):
        n = min(sizes[i % len(sizes)], len(wav) - pos)
        outs.append(sc.push(wav[pos:pos + n]))
        pos, i = pos + n, i + 1
    return np.concatenate(outs + [sc.flush()])


def test_ring_frames_follow_the_whole_clip_stft():
    """The ring rule (modular addressing, reflect at the start, reflect at the end only once closed) gives the oracle
    STFT frames of the whole clip, in a ring much shorter than the clip."""
    from openvoice_b200._native import STREAM_OPEN
    L, cap = 22050 * 3 + 77, 8192
    x = torch.from_numpy(wave(L, 3))
    whole = O.spectrogram(x[None])[0, :, : L // HOP]
    T = L // HOP
    for lo, n, upto, closed in ((0, 20, 30 * HOP, False), (120, 24, 150 * HOP, False), (T - 15, 15, L, True)):
        a = max(0, lo * HOP - PAD)
        rings = torch.full((2, cap), float("nan"))
        rings[1, torch.from_numpy(np.arange(a, upto) % cap)] = x[a:upto]
        got = ring_frames(rings, 1, lo, n, L if closed else STREAM_OPEN)
        assert torch.allclose(got, whole[:, lo:lo + n], rtol=1e-5, atol=1e-5), (lo, n)


@pytest.mark.parametrize("W", [32, 64])
def test_sessions_equal_their_own_streaming_converters(W):
    """Six staggered sessions with different lengths, chunkings, embeddings, taus and seeds (rows reused after a close):
    each session's output equals StreamingConverter(request_seed=...) fed the same chunks.  Rows in use and the audio
    each session keeps stay bounded."""
    from openvoice_b200.streaming import StreamingSessions
    H = 128
    specs = [  # (samples, chunk sizes, seed, tau, step of open)
        (22050 * 1 + 5, [441], 11, 0.3, 0),
        (256 * (W + H + 30), [441, 1000, 37], 12, 0.0, 0),
        (22050 * 4 + 131, [441], 13, 0.5, 2),
        (22050 * 2 + 99, [10 ** 9], 14, 0.3, 3),
        (22050 * 2 + 7, [5000, 17, 8191], 2 ** 64 - 1, 1.0, 40),
        (22050 * 3 + 1, [441], 16, 0.3, 260),
    ]
    ss = StreamingSessions(FakeConverter(), window_frames=W)
    waves = [wave(L, 20 + k) for k, (L, *_rest) in enumerate(specs)]
    ids, pos, step, outs, turn = {}, [0] * len(specs), 0, {k: [] for k in range(len(specs))}, [0] * len(specs)
    max_rows, max_keep, biggest = 0, 0, [0] * len(specs)
    done = set()
    while len(done) < len(specs):
        for k, (L, sizes, seed, tau, start) in enumerate(specs):
            if step == start:
                ids[k] = ss.open(se(0), se(1), tau=tau, seed=seed)
        chunks, owner = {}, {}
        for k, sid in ids.items():
            if k in done or pos[k] >= len(waves[k]):
                continue
            n = min(specs[k][1][turn[k] % len(specs[k][1])], len(waves[k]) - pos[k])
            chunks[sid], owner[sid] = waves[k][pos[k]:pos[k] + n], k
            pos[k], turn[k] = pos[k] + n, turn[k] + 1
        for sid, y in ss.push(chunks).items():
            outs[owner[sid]].append(y)
        for sid, c in chunks.items():
            biggest[owner[sid]] = max(biggest[owner[sid]], len(c))
        for k, sid in ids.items():
            if k not in done:                            # beyond the two halos, one window and the STFT lead
                max_keep = max(max_keep, ss.state_samples(sid) - biggest[k])
        ending = [k for k, sid in ids.items() if k not in done and pos[k] >= len(waves[k])]
        if ending:
            for sid, y in ss.close([ids[k] for k in ending]).items():
                outs[[k for k in ending if ids[k] == sid][0]].append(y)
            done.update(ending)
        max_rows = max(max_rows, ss.rows_in_use)
        step += 1
    assert ss.rows < len(specs)                          # a later session reused a closed session's row
    for k, (L, sizes, seed, tau, _) in enumerate(specs):
        got = np.concatenate(outs[k])
        ref = converter_stream(waves[k], sizes, W, seed, tau)
        assert got.shape == ref.shape == (HOP * (L // HOP),), k
        assert np.allclose(got, ref, rtol=1e-5, atol=1e-5), (k, float(np.abs(got - ref).max()))
    assert max_rows <= len(specs)
    assert max_keep <= HOP * (W + 2 * H + 8), max_keep


def count_step(n_sessions, W, monkeypatch, budget=None):
    from openvoice_b200 import streaming as S
    if budget is not None:
        monkeypatch.setattr(S, "SESSION_BATCH_FRAMES", budget)
    conv = FakeConverter()
    ss = S.StreamingSessions(conv, window_frames=W)
    sids = [ss.open(se(k), se(k + 1), tau=0.3, seed=k) for k in range(n_sessions)]
    x = wave(256 * (W + 128 + 4), 1)
    calls = conv.model.native.calls
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU]) as prof:
        out = ss.push({sid: x for sid in sids})
    appends = sum(e.count for e in prof.key_averages() if e.key == "aten::index_copy_")
    return dict(calls), appends, out


def test_native_calls_per_step_do_not_grow_with_sessions(monkeypatch):
    """One ring append, one ring spectrogram and one conversion per step, for 1 session as for 64; a step whose windows
    exceed the padded-frame budget is split into ceil(windows / windows per launch) conversions, still one spectrogram."""
    W = 32
    one, app1, out1 = count_step(1, W, monkeypatch)
    many, app64, out64 = count_step(64, W, monkeypatch)
    assert all(len(v) == HOP * W for v in list(out1.values()) + list(out64.values()))
    for calls, app in ((one, app1), (many, app64)):
        assert calls == {"spectrogram_ring": 1, "voice_conversion": 1, "spectrogram": 0}, calls
        assert app == 1
    Tmax = -(-(W + 128) // 16) * 16
    split, _, _ = count_step(64, W, monkeypatch, budget=10 * Tmax)
    assert split == {"spectrogram_ring": 1, "voice_conversion": math.ceil(64 / 10), "spectrogram": 0}, split


def test_refusals_launch_nothing_and_change_nothing():
    from openvoice_b200.streaming import StreamingSessions
    conv = FakeConverter()
    calls = conv.model.native.calls
    with pytest.raises(ValueError, match="window_frames"):
        StreamingSessions(conv, window_frames=0)
    ss = StreamingSessions(conv, window_frames=32)
    for bad in (2 ** 64, -1, 1.5, True):
        with pytest.raises(ValueError, match="seed"):
            ss.open(se(0), se(1), seed=bad)
    with pytest.raises(ValueError, match="src_se"):
        ss.open(torch.zeros(GIN + 1), se(1))
    with pytest.raises(ValueError, match="tgt_se"):
        ss.open(se(0), torch.zeros(1, GIN - 1, 1))
    with pytest.raises(ValueError, match="input_sr"):
        ss.open(se(0), se(1), input_sr=48000)
    with pytest.raises(ValueError, match="output_sr"):
        ss.open(se(0), se(1), output_sr=16000)
    assert ss.rows_in_use == 0
    a = ss.open(se(0), se(1), seed=1)
    b = ss.open(se(2), se(3), seed=2)
    ss.push({a: wave(300, 1), b: wave(5000, 2)})
    before = {sid: (s.n_in, s.emitted, s.row) for sid, s in ss.sessions.items()}
    calls0 = dict(calls)
    with pytest.raises(ValueError, match="unknown or closed"):
        ss.push({a: wave(441, 3), 12345: wave(441, 3)})
    with pytest.raises(ValueError, match="unknown or closed"):
        ss.close([b, 777])
    with pytest.raises(ValueError, match="audio too short"):
        ss.close([b, a])                                   # a: 300 samples, not past the STFT padding
    assert calls == calls0
    assert {sid: (s.n_in, s.emitted, s.row) for sid, s in ss.sessions.items()} == before
    ss.close([b])
    with pytest.raises(ValueError, match="unknown or closed"):
        ss.push({b: wave(441, 4)})
    with pytest.raises(ValueError, match="unknown or closed"):
        ss.close([b])
    assert calls["spectrogram_ring"] == calls0["spectrogram_ring"] + 1
