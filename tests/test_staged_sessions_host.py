"""Host logic of StagedSessions on the CPU, with a stand-in converter whose latent stack sees exactly +-96 frames and whose
generator sees exactly +-14: coverage of both halos, the window geometry under any chunking, the exact look-ahead, and
the refusals."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import vc_oracle as O

from test_multistream_host import GIN, HOP, FakeConverter, FakeNative, se, wave

LAT_K = torch.linspace(0.3, 1.0, 2 * 96 + 1, dtype=torch.float64)[None, None]
GEN_K = torch.linspace(1.0, 0.2, 2 * 14 + 1, dtype=torch.float64)[None, None]
CH = FakeConverter.hps.model.inter_channels


def fake_latent(spec, n, seed, frame0, tau):
    """[CH, n]: frame t depends on spectrogram frames t-96 .. t+96 of the item (zeros past its ends) and on a per-(seed,
    absolute frame) noise value."""
    t = torch.arange(frame0, frame0 + n, dtype=torch.float64)
    f = spec[:8, :n].double().mean(0) + tau * torch.sin((seed % 1009) * 0.1 + 0.7 * t)
    g = F.conv1d(f[None, None], LAT_K, padding=96)[0, 0]
    return g[None] * torch.arange(1, CH + 1, dtype=torch.float64)[:, None]


def fake_generate(z, n):
    """[hop * n]: frame t depends on latent frames t-14 .. t+14 of the item."""
    f = z[:, :n].double().sum(0)
    g = F.conv1d(f[None, None], GEN_K, padding=14)[0, 0]
    return (g[:, None] * torch.linspace(1.0, 2.0, HOP, dtype=torch.float64)[None]).reshape(-1)


class StagedNative(FakeNative):
    refenc_state_floats = 0

    def __init__(self):
        super().__init__()
        self.calls.update(latent=0, generate=0)

    def latent(self, spec, lens, gs, gt, items=None, out=None):
        self.calls["latent"] += 1
        B, _, T = spec.shape
        z = out.view(B, CH, T)
        z.zero_()
        seeds = items["seed"].numpy().view(np.uint64)
        for b in range(B):
            n = int(lens[b])
            z[b, :, :n] = fake_latent(spec[b], n, int(seeds[b]), int(items["frame0"][b]), float(items["tau"][b])).float()
        return z

    def generate(self, z, lens, gt, out=None):
        self.calls["generate"] += 1
        B, _, T = z.shape
        o = out.view(B, HOP * T)
        o.zero_()
        for b in range(B):
            n = int(lens[b])
            o[b, :HOP * n] = fake_generate(z[b], n).float()
        return o.view(B, 1, -1)


class StagedConverter(FakeConverter):
    def __init__(self):
        super().__init__()
        self.model.native = StagedNative()


def whole_clip(x, seed, tau):
    """The stand-in's conversion of the whole clip (one window, frame0 0)."""
    T = len(x) // HOP
    spec = O.spectrogram(torch.from_numpy(x)[None])[0, :, :T]
    return fake_generate(fake_latent(spec, T, seed, 0, tau), T).float().numpy()


class Recorder:
    """Runs one session of StagedSessions over a chunking, recording each step's stage-A and stage-B windows and the
    frames ready after it."""

    def __init__(self, W):
        from openvoice_b200.streaming import StagedSessions
        self.ss = StagedSessions(StagedConverter(), window_frames=W)
        self.A, self.B, self.steps = [], [], []
        plan = self.ss._plan

        def recording(ses, gains, final, skip):
            wins, p = plan(ses, gains, final, skip)
            self.A += [w[1:] for w in p[0]]
            self.B += [w[1:] for w in p[1]]
            self.steps.append([w[1:] for w in p[1]])
            return wins, p
        self.ss._plan = recording

    def run(self, x, sizes, seed=7, tau=0.3):
        from openvoice_b200.streaming import ready_frames
        sid = self.ss.open(se(0), se(1), tau=tau, seed=seed)
        outs, pos, k, self.ready = [], 0, 0, []
        while pos < len(x):
            n = min(sizes[k % len(sizes)], len(x) - pos)
            outs.append(self.ss.push({sid: x[pos:pos + n]})[sid])
            pos, k = pos + n, k + 1
            self.ready.append(ready_frames(pos, HOP, 1024, False))
        outs.append(self.ss.close([sid])[sid])
        return np.concatenate(outs)


def chunkings(L):
    rng = np.random.default_rng(L)
    return {"441": [441], "random": [int(v) for v in rng.integers(1, 6000, 40)], "whole": [L]}


@pytest.mark.parametrize("W", [8, 16, 32, 256])
def test_halos_cover_every_frame_and_each_frame_is_emitted_once(W):
    """Each stage-B window holds GEN_HALO_FRAMES final latent frames on both sides of its interior and each stage-A
    window LATENT_HALO_FRAMES spectrogram frames, clipped only at the stream's ends; the interiors tile the stream once
    (close emits the rest); and the output equals the whole-clip conversion of halo-exact stand-in stages."""
    from openvoice_b200.streaming import GEN_HALO_FRAMES, LATENT_HALO_FRAMES
    L = HOP * (3 * W + 250) + 77
    T = L // HOP
    x = wave(L, W)
    for name, sizes in chunkings(L).items():
        r = Recorder(W)
        got = r.run(x, sizes)
        for wins, H, unit in ((r.A, LATENT_HALO_FRAMES, min(W, 16)), (r.B, GEN_HALO_FRAMES, W)):
            assert [e0 for _, _, e0, _ in wins] == list(range(0, T, unit)), name
            assert [e1 for _, _, _, e1 in wins] == [min(T, e) for e in range(unit, T + unit, unit)], name
            for lo, hi, e0, e1 in wins:
                assert lo == max(0, e0 - H) and hi == min(T, e1 + H), (name, lo, hi, e0, e1)
        assert got.shape == (HOP * T,), name
        ref = whole_clip(x, 7, 0.3)
        assert np.allclose(got, ref, rtol=1e-5, atol=1e-5), (name, float(np.abs(got - ref).max()))


@pytest.mark.parametrize("W", [8, 32])
def test_geometry_does_not_depend_on_chunking(W):
    L = HOP * (2 * W + 300) + 5
    x = wave(L, 3)
    seen = []
    for sizes in chunkings(L).values():
        r = Recorder(W)
        out = r.run(x, sizes)
        seen.append((sorted(r.A), sorted(r.B), out))
    for A, B, out in seen[1:]:
        assert A == seen[0][0] and B == seen[0][1]
        assert np.array_equal(out, seen[0][2])


@pytest.mark.parametrize("W", [8, 16, 24, 32, 256])
def test_look_ahead_is_exact(W):
    """Pushing one hop at a time, a window's frames come out in the step where the ready frames first reach its
    threshold; the largest (ready frames - frame) over all emitted frames is U * ceil((e0 + W + 14) / U) + 96 - e0
    maximised over window starts e0, which is W + U * ceil(14 / U) + 96 = W + 112 whenever U = min(W, 16) divides W."""
    U = min(W, 16)
    T = 6 * W + 200
    x = wave(HOP * T + 100, 1)
    r = Recorder(W)
    r.run(x, [HOP])
    worst = 0
    for wins, ready in zip(r.steps, r.ready):             # the closing step's windows are past the last push
        for _, _, e0, e1 in wins:
            worst = max(worst, ready - e0)
    starts = range(0, T - W - 14 - 96 - U, W)             # windows an open stream emits
    exact = max(U * -(-(e0 + W + 14) // U) + 96 - e0 for e0 in starts)
    assert worst == exact, (worst, exact)
    if W % U == 0:
        assert exact == W + U * -(-14 // U) + 96 == W + 112


def test_refusals_match_streaming_sessions():
    from openvoice_b200.streaming import Enrollment, StagedSessions
    conv = StagedConverter()
    for bad in (0, -3):
        with pytest.raises(ValueError, match="window_frames"):
            StagedSessions(conv, window_frames=bad)
    for bad in (0, -48000, 1.5, True):
        with pytest.raises(ValueError, match="rates"):
            StagedSessions(conv, window_frames=32, rates=[bad])
    ss = StagedSessions(conv, window_frames=32)
    for bad in (2 ** 64, -1, 1.5, True):
        with pytest.raises(ValueError, match="seed"):
            ss.open(se(0), se(1), seed=bad)
    with pytest.raises(ValueError, match="src_se"):
        ss.open(torch.zeros(GIN + 1), se(1))
    with pytest.raises(ValueError, match="tgt_se"):
        ss.open(se(0), torch.zeros(1, GIN - 1, 1))
    with pytest.raises(ValueError, match="input_sr"):
        ss.open(se(0), se(1), input_sr=48000)
    with pytest.raises(ValueError, match="reference encoder"):
        ss.open(se(0), se(1), enroll=Enrollment())
    with pytest.raises(ValueError, match="src_se is None"):
        ss.open(None, se(1))
    assert ss.rows_in_use == 0
    a = ss.open(se(0), se(1), seed=1)
    ss.push({a: wave(300, 1)})
    with pytest.raises(ValueError, match="audio too short"):
        ss.close([a])
    with pytest.raises(ValueError, match="unknown or closed"):
        ss.push({a: wave(441, 3), 12345: wave(441, 3)})
    assert conv.model.native.calls["latent"] == conv.model.native.calls["generate"] == 0
