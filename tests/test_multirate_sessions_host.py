"""Host logic of StreamingSessions with sessions at other rates than the model's, on the CPU: a stand-in converter and
a stand-in resampler (the geometry of ovc_resample_span, a made-up filter) drive both StreamingSessions and the
reference StreamingConverter(input_sr=, output_sr=).  Per push, the model-rate counts, window schedule and output
lengths match the reference; raw and output rings stay within their keep rules; a step adds at most two splices and two
ring resamples however many sessions it names, and none when it names no resampling session; refusals launch nothing."""
import math

import numpy as np
import pytest
import torch

import test_multistream_host as M
from openvoice_b200._native import STREAM_OPEN, resample_span

SR = M.SR


def plan(a, b):
    g = math.gcd(a, b)
    up, down = b // g, a // g
    half = 0 if up == down else 10 * max(up, down)
    taps = 2 * half + 1
    pre_pad = down - half % down
    return up, down, taps, pre_pad, (half + pre_pad) // down, -(-taps // up) + 1


def support(p, m):
    """Input samples [jlo, jhi] output m reads (ovc_resample.h: output_at)."""
    up, down, taps, pre_pad, pre_remove, _ = p
    t = (m + pre_remove) * down - pre_pad
    return -((taps - 1 - t) // up), t // up


def n_out(p, L):
    return STREAM_OPEN if L == STREAM_OPEN else -(-L * p[0] // p[1])


def fake_outputs(a, b, ms, sample):
    """Stand-in resampler: y[m] = sum over m's support of x[j] * w(j - jlo, m) in fp64, x[j] = sample(j) (0 outside
    what the caller holds); deterministic, so any two callers that hold the same samples agree bit for bit."""
    p = plan(a, b)
    ms = np.asarray(ms, dtype=np.int64)
    if ms.size == 0:
        return np.zeros(0, dtype=np.float32)
    jlo, jhi = support(p, ms)
    k = np.arange(p[5])
    J = jlo[:, None] + k[None]
    x = np.where(J <= jhi[:, None], sample(J), 0.0)
    wgt = np.cos(0.37 * k[None] + 1e-3 * ms[:, None]) / p[5] * 2
    return (x * wgt).sum(1).astype(np.float32)


class FakeNative(M.FakeNative):
    device_index = 0

    def __init__(self):
        super().__init__()
        self.calls.update(resample=0, resample_plan=0, resample_rings=0)
        self.plan_rates = []

    def resample(self, x, ln, sr_in, sr_out, out_pitch=None, in_start=0, out_start=0):
        self.calls["resample"] += 1
        xs, L = x[0].double().numpy(), int(ln[0])

        def sample(J):
            k = J - in_start
            ok = (J >= 0) & (J < L) & (k >= 0) & (k < len(xs))
            return np.where(ok, xs[np.clip(k, 0, len(xs) - 1)], 0.0)
        ms = np.arange(out_start, out_start + out_pitch)
        y = fake_outputs(sr_in, sr_out, ms, sample)
        y[ms >= n_out(plan(sr_in, sr_out), L)] = 0
        return torch.from_numpy(y)[None]

    def resample_plan(self, a, b):
        self.calls["resample_plan"] += 1
        if (a, b) not in self.plan_rates:
            self.plan_rates.append((a, b))
        return self.plan_rates.index((a, b))

    def resample_rings(self, plan_ids, x, in_row, in_len, m0, count, out, out_row, out_off, max_count):
        self.calls["resample_rings"] += 1
        cap, ocap = x.shape[1], out.shape[1]
        flat = x.reshape(-1).double().numpy()
        for b in range(plan_ids.numel()):
            a, r = self.plan_rates[int(plan_ids[b])]
            row, L, m, n = int(in_row[b]), int(in_len[b]), int(m0[b]), min(int(count[b]), max_count)
            sample = lambda J: np.where((J >= 0) & (J < L), flat[row * cap + J % cap], 0.0)  # noqa: E731
            ms = np.arange(m, m + n)
            y = fake_outputs(a, r, ms, sample)
            y[ms >= n_out(plan(a, r), L)] = 0
            out[int(out_row[b]), torch.from_numpy((int(out_off[b]) + np.arange(n)) % ocap)] = torch.from_numpy(y)


class FakeConverter(M.FakeConverter):
    def __init__(self):
        self.model = M.FakeModel()
        self.model.native = FakeNative()


@pytest.fixture(autouse=True)
def cpu_resampler(monkeypatch):
    """StreamingResampler uploads to the converter's CUDA device; here the stand-in runs on the CPU."""
    from openvoice_b200 import streaming as S
    init = S.StreamingResampler.__init__

    def cpu_init(self, *args, **kw):
        init(self, *args, **kw)
        self.dev = torch.device("cpu")
    monkeypatch.setattr(S.StreamingResampler, "__init__", cpu_init)


def test_plan_replica_matches_the_library():
    for a, b in ((48000, SR), (SR, 48000), (8000, SR), (SR, 44100), (16000, SR)):
        p = plan(a, b)
        for m in (0, 1, 7, 1000, 12345):
            _, _, lo, hi = resample_span(a, b, 0, m, m + 1)
            assert support(p, m) == (lo, hi - 1)
        assert n_out(p, 12345) == resample_span(a, b, 12345)[0]


SPECS = [  # (input_sr, output_sr, seconds, chunk sizes, step of open)
    (48000, 48000, 1.6, [960], 0),
    (16000, 16000, 1.3, [320, 5000], 0),
    (8000, None, 2.0, [160, 37, 999], 3),
    (None, 44100, 1.7, [441, 2000], 5),
    (SR, SR, 1.2, [441], 6),
    (None, None, 1.4, [700, 5], 8),
    (48000, 48000, 0.05, [10 ** 9], 10),            # shorter than window + halo
]


def test_multirate_sessions_equal_their_own_streaming_converters():
    from openvoice_b200.streaming import StreamingConverter, StreamingSessions
    W = 32
    conv = FakeConverter()
    ss = StreamingSessions(conv, window_frames=W, rates=(48000, 16000, 8000, 44100, SR))
    waves = [M.wave(max(1, int(sec * (i or SR))), 30 + k) for k, (i, o, sec, _, _) in enumerate(SPECS)]
    refs = [StreamingConverter(FakeConverter(), M.se(0), M.se(1), tau=0.3, window_frames=W, input_sr=i, output_sr=o,
                               request_seed=100 + k) for k, (i, o, *_rest) in enumerate(SPECS)]
    ids, pos, turn, done, step, biggest = {}, [0] * len(SPECS), [0] * len(SPECS), set(), 0, [0] * len(SPECS)
    total = [0] * len(SPECS)
    while len(done) < len(SPECS):
        for k, (i, o, _, _, start) in enumerate(SPECS):
            if step == start:
                ids[k] = ss.open(M.se(0), M.se(1), tau=0.3, seed=100 + k, input_sr=i, output_sr=o)
        chunks, owner, ending = {}, {}, []
        for k, sid in ids.items():
            if k in done:
                continue
            if pos[k] >= len(waves[k]):
                ending.append(k)
                continue
            sizes = SPECS[k][3]
            n = min(sizes[turn[k] % len(sizes)], len(waves[k]) - pos[k])
            chunks[sid], owner[sid] = waves[k][pos[k]:pos[k] + n], k
            pos[k], turn[k], biggest[k] = pos[k] + n, turn[k] + 1, max(biggest[k], n)
        for sid, y in ss.push(chunks).items():
            k = owner[sid]
            ref = refs[k].push(chunks[sid])
            assert y.shape == ref.shape, (k, step)
            assert np.allclose(y, ref, rtol=1e-5, atol=1e-5), (k, step)
            assert ss.sessions[sid].n_in == refs[k].n_in and ss.sessions[sid].emitted == refs[k].emitted, k
            total[k] += len(y)
            i, o = SPECS[k][:2]
            if i not in (None, SR):                       # raw ring: the next model sample's support and the push
                lo, hi = resample_span(i, SR, 0, 0, 1)[2:]
                assert ss.raw_state_samples(sid) <= (hi - lo) + biggest[k], k
            if o not in (None, SR):
                lo, hi = resample_span(SR, o, 0, 0, 1)[2:]
                assert ss.out_state_samples(sid) <= hi - lo, k
        for k in ending:
            y = ss.close([ids[k]])[ids[k]]
            ref = refs[k].flush()
            assert y.shape == ref.shape and np.allclose(y, ref, rtol=1e-5, atol=1e-5), k
            total[k] += len(y)
            done.add(k)
        step += 1
    for k, (i, o, *_rest) in enumerate(SPECS):         # whole model-rate frames, resampled to the output rate
        n_model = resample_span(i, SR, len(waves[k]))[0] if i not in (None, SR) else len(waves[k])
        T = n_model // M.HOP
        assert total[k] == (resample_span(SR, o, M.HOP * T)[0] if o not in (None, SR) else M.HOP * T), k


def count_step(ss, chunks):
    calls = ss.native.calls
    before = dict(calls)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU]) as prof:
        ss.push(chunks)
    splices = sum(e.count for e in prof.key_averages() if e.key == "aten::index_copy_")
    return {k: calls[k] - before[k] for k in calls}, splices


@pytest.mark.parametrize("S", [1, 8, 64])
def test_native_calls_per_step(S):
    """S sessions at 48 kHz in and out plus S at the model's rate: a step naming the 48 kHz ones (alone or with the
    others) adds at most two splices and two ring resamples to a model-rate step; a step naming only model-rate sessions
    makes exactly the calls of a StreamingSessions without rates."""
    from openvoice_b200.streaming import StreamingSessions
    W = 16
    ss = StreamingSessions(FakeConverter(), window_frames=W, rates=(48000,))
    plain = StreamingSessions(FakeConverter(), window_frames=W)
    fast = [ss.open(M.se(k), M.se(k + 1), seed=k, input_sr=48000, output_sr=48000) for k in range(S)]
    model = [ss.open(M.se(k), M.se(k + 1), seed=k) for k in range(S)]
    ref = [plain.open(M.se(k), M.se(k + 1), seed=k) for k in range(S)]
    x48, x22 = M.wave(48000 * 6, 1), M.wave(SR * 6, 2)
    n48, n22 = 2 * M.HOP * (W + 128) * 48000 // SR, 2 * M.HOP * (W + 128)     # past window + halo
    ss.push({**{sid: x48[:n48] for sid in fast}, **{sid: x22[:n22] for sid in model}})
    plain.push({sid: x22[:n22] for sid in ref})
    emitted = 0
    for p in range(4):
        a48, a22 = n48 + 9000 * p, n22 + 4400 * p         # about one window per step
        calls, splices = count_step(ss, {sid: x48[a48:a48 + 9000] for sid in fast})
        assert calls["resample_rings"] <= 2 and splices <= 2, (p, calls, splices)
        assert calls["voice_conversion"] <= 1 and calls["resample_plan"] == calls["resample"] == 0
        emitted += calls["voice_conversion"]
        c_ss, sp_ss = count_step(ss, {sid: x22[a22:a22 + 4400] for sid in model})
        c_pl, sp_pl = count_step(plain, {sid: x22[a22:a22 + 4400] for sid in ref})
        assert c_ss == c_pl and sp_ss == sp_pl, (p, c_ss, c_pl)
        assert c_ss["resample_rings"] == 0 and c_ss["voice_conversion"] >= 1
    both, splices_b = count_step(ss, {**{sid: x48[-960:] for sid in fast}, **{sid: x22[-441:] for sid in model}})
    assert both["resample_rings"] <= 2 and splices_b <= 3, (both, splices_b)
    assert emitted >= 3


def test_refusals_launch_nothing_and_change_nothing():
    from openvoice_b200.streaming import StreamingSessions
    conv = FakeConverter()
    calls = conv.model.native.calls
    for bad in ((44101,), (0,), (-8000,), (48000.5,), (True,)):
        with pytest.raises(ValueError):
            StreamingSessions(conv, window_frames=32, rates=bad)
    with pytest.raises(ValueError, match="44101"):
        StreamingSessions(conv, window_frames=32, rates=(48000, 44101))
    assert calls["resample_plan"] == 0                    # checked before any bank is built
    ss = StreamingSessions(conv, window_frames=32, rates=(48000,))
    assert calls["resample_plan"] == 2 and ss.rates == (48000,)
    a = ss.open(M.se(0), M.se(1), seed=1, input_sr=48000, output_sr=48000)
    ss.push({a: M.wave(700, 1)})
    state = {sid: (s.n_in, s.raw_n, s.out_n, s.emitted, s.row) for sid, s in ss.sessions.items()}
    rings = [t.clone() for t in (ss.rings, ss.raw, ss.orings)]
    calls0 = dict(calls)
    for kw, name in (({"input_sr": 16000}, "input_sr"), ({"output_sr": 8000}, "output_sr"), ({"input_sr": -5}, "input_sr"),
                     ({"output_sr": 0}, "output_sr"), ({"input_sr": 44101}, "input_sr")):
        with pytest.raises(ValueError, match=f"{name}.*declared: 48000"):
            ss.open(M.se(0), M.se(1), **kw)
    with pytest.raises(ValueError, match="audio too short"):
        ss.close([a])                                      # 700 samples at 48 kHz: 322 at the model's rate
    assert calls == calls0
    assert {sid: (s.n_in, s.raw_n, s.out_n, s.emitted, s.row) for sid, s in ss.sessions.items()} == state
    assert all(torch.equal(t, u) for t, u in zip(rings, (ss.rings, ss.raw, ss.orings)))
    assert ss.rows_in_use == 1
