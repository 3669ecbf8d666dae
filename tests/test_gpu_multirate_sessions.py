"""-m gpu: live sessions at other rates than the model's.  ovc_resample_rings against the whole-signal ovc_resample bit
for bit; StreamingSessions(rates=...) sessions against their own StreamingConverter(input_sr=, output_sr=) push by push;
company, launches per step, graph replay, push_device and refusals; CloneSessions(output_rates=) against the model-rate
session resampled by StreamingResampler.  fp32 and f16x3."""
import numpy as np
import pytest
import torch

from test_gpu_clone import models, requests
from test_gpu_multistream import conv, emb, wave  # noqa: F401  (conv: fixture)

pytestmark = pytest.mark.gpu

SR, HOP, H = 22050, 256, 128
OPEN = 2 ** 63 - 1
PAIRS = [(48000, SR), (SR, 48000), (8000, SR), (SR, 16000), (44100, SR), (SR, SR)]


# ------------------------------------------------------------------------------------------------ 1. the kernel
def test_resample_rings_equal_whole_signal(conv):
    """One launch over every pair: open items (the outputs ready so far), closed items (the tail and outputs past n_out,
    written as 0), input windows that wrap their ring row, outputs into wrapping ring rows and packed into one row.
    Every output equals ovc_resample of the whole signal; everything outside each item's outputs stays NaN."""
    from openvoice_b200._native import resample_span
    nat = conv.model.native
    rng = np.random.default_rng(1)
    plans = [nat.resample_plan(a, b) for a, b in PAIRS]
    assert plans == [nat.resample_plan(a, b) for a, b in PAIRS]          # one id per pair
    in_cap, out_cap = 3400, 4096
    items, sig = [], []
    for k, (a, b) in enumerate(PAIRS):
        L = int(rng.integers(20000, 40000))
        sig.append((0.3 * rng.standard_normal(L)).astype(np.float32))
        ready, n_all = resample_span(a, b, L - int(rng.integers(100, 3000)))[1], resample_span(a, b, L)[0]
        items += [(k, OPEN, ready - 1500, 1500, False), (k, L, n_all - 1400, 1500, False), (k, OPEN, 501, 600, True),
                  (k, L, n_all - 40, 80, True)]
    B = len(items)
    rings = torch.full((B, in_cap), float("nan"), device="cuda")
    out = torch.full((B + 1, out_cap), float("nan"), device="cuda")
    desc, at, wrapped = [], 0, 0
    for r, (k, ln, m0, n, pk) in enumerate(items):
        a, b = PAIRS[k]
        x = sig[k]
        _, _, lo, hi = resample_span(a, b, 0, m0, m0 + n)
        lo, hi = max(lo, 0), min(hi, len(x))
        rings[r, torch.from_numpy(np.arange(lo, hi) % in_cap).cuda()] = torch.from_numpy(x[lo:hi]).cuda()
        wrapped += (lo // in_cap) != ((hi - 1) // in_cap)
        desc.append((plans[k], r, ln, m0, n, B if pk else r, at if pk else m0))
        at += n if pk else 0
    assert wrapped >= 3 and at <= out_cap
    i64 = lambda c: torch.tensor([d[c] for d in desc], dtype=torch.int64, device="cuda")   # noqa: E731
    plan = torch.tensor([d[0] for d in desc], dtype=torch.int32, device="cuda")
    nat.resample_rings(plan, rings, i64(1), i64(2), i64(3), i64(4), out, i64(5), i64(6), max(d[4] for d in desc))
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    seen = np.zeros(got.shape, bool)
    wrapped_out = 0
    for (k, ln, m0, n, pk), d in zip(items, desc):
        a, b = PAIRS[k]
        x = torch.from_numpy(sig[k]).cuda()[None]
        ref = nat.resample(x, torch.tensor([len(sig[k])], dtype=torch.int64, device="cuda"), a, b)[0].cpu().numpy()
        ms = np.arange(m0, m0 + n)
        want = np.where(ms < len(ref), ref[np.minimum(ms, len(ref) - 1)], 0).astype(np.float32)
        cols = (d[6] + np.arange(n)) % out_cap
        wrapped_out += (not pk) and cols[0] > cols[-1]
        assert np.array_equal(got[d[5], cols], want), (a, b, ln == OPEN, m0, pk)
        seen[d[5], cols] = True
    assert np.isnan(got[~seen]).all() and wrapped_out >= 1


# ------------------------------------------------------------------------------------------------ sessions
def reference(conv, script_k, W):
    from openvoice_b200.streaming import StreamingConverter
    w, sizes, src, tgt, tau, seed, _, i, o = script_k
    sc = StreamingConverter(conv, src, tgt, tau, W, input_sr=i, output_sr=o, request_seed=seed)
    outs, pos, t = [], 0, 0
    while pos < len(w):
        n = min(sizes[t % len(sizes)], len(w) - pos)
        outs.append(sc.push(w[pos:pos + n]))
        pos, t = pos + n, t + 1
    return outs + [sc.flush()]


def drive(ss, script):
    """Pushes (wave, sizes, src, tgt, tau, seed, step of open, input_sr, output_sr) sessions, closing each in the step
    after its last push; returns each session's list of returns (one per push, then the close)."""
    ids, pos, turn, done, step = {}, [0] * len(script), [0] * len(script), set(), 0
    outs = {k: [] for k in range(len(script))}
    while len(done) < len(script):
        for k, (_, _, src, tgt, tau, seed, start, i, o) in enumerate(script):
            if step == start:
                ids[k] = ss.open(src, tgt, tau=tau, seed=seed, input_sr=i, output_sr=o)
        owner = {sid: k for k, sid in ids.items() if k not in done}
        chunks, ending = {}, []
        for sid, k in owner.items():
            w, sizes = script[k][0], script[k][1]
            if pos[k] >= len(w):
                ending.append(sid)
                continue
            n = min(sizes[turn[k] % len(sizes)], len(w) - pos[k])
            chunks[sid] = w[pos[k]:pos[k] + n]
            pos[k], turn[k] = pos[k] + n, turn[k] + 1
        res = ss.push(chunks)
        for sid in chunks:
            outs[owner[sid]].append(res[sid])
        if ending:
            for sid, y in ss.close(ending).items():
                outs[owner[sid]].append(y)
            done.update(owner[sid] for sid in ending)
        step += 1
    return outs


def test_sessions_equal_their_own_converters(conv):
    """Seven staggered sessions (rows reused): (48 k, 48 k), (16 k, 16 k), (8 k, None), (None, 44.1 k) over 20 s in one
    push, (22.05 k, 22.05 k) given explicitly, (None, None), and a 48 kHz one shorter than window + halo.  Every push's
    and close's return equals the session's own StreamingConverter(input_sr=, output_sr=) bit for bit."""
    from openvoice_b200.streaming import StreamingSessions
    W = 64
    rates = [(48000, 48000, 3.1, [960]), (16000, 16000, 2.7, [320]), (8000, None, 3.3, [160, 1000, 37]),
             (None, 44100, 20.5, [10 ** 9]), (SR, SR, 2.2, [441, 5000]), (None, None, 2.5, [700, 13]),
             (48000, 48000, 0.5, [960])]
    starts = [0, 0, 2, 3, 40, 60, 70]
    script = [(wave(int(sec * (i or SR)), 70 + k), sz, emb(2 * k), emb(2 * k + 1), 0.3 * (k % 3), 11 + k, starts[k], i, o)
              for k, (i, o, sec, sz) in enumerate(rates)]
    assert len(script[6][0]) * SR // 48000 < HOP * (W + H)
    ss = StreamingSessions(conv, window_frames=W, rates=(48000, 16000, 8000, 44100))
    got = drive(ss, script)
    assert ss.rows < len(script) and ss.rows_in_use == 0
    for k in range(len(script)):
        ref = reference(conv, script[k], W)
        assert len(got[k]) == len(ref), k
        for t, (g, r) in enumerate(zip(got[k], ref)):
            assert g.shape == r.shape and np.array_equal(g, r), (k, t)


def test_company_does_not_matter(conv):
    from openvoice_b200.streaming import StreamingSessions
    W = 32
    me = (wave(48000 * 4 + 99, 1), [960], emb(1), emb(2), 0.3, 4242, 0, 48000, 48000)
    rng = np.random.default_rng(5)
    mix = [(48000, 48000), (16000, None), (None, 8000), (None, None), (44100, 16000)]
    others = []
    for k in range(31):
        i, o = mix[k % len(mix)]
        others.append((wave(int(rng.integers(2, 4) * (i or SR)), 50 + k), [int(v) for v in rng.integers(100, 3000, 3)],
                       emb(10 + k), emb(40 + k), 0.3, 1000 + k, int(rng.integers(0, 100)), i, o))
    rates = (48000, 16000, 8000, 44100)
    alone = drive(StreamingSessions(conv, window_frames=W, rates=rates), [me])[0]
    crowd = drive(StreamingSessions(conv, window_frames=W, rates=rates), others[:15] + [me] + others[15:])[15]
    assert np.array_equal(np.concatenate(alone), np.concatenate(crowd))


def counting(ss, names=("splice", "resample_rings", "spectrogram_ring", "voice_conversion", "resample",
                        "resample_plan", "spectrogram")):
    counts = {n: 0 for n in names}
    for name in names:
        def counted(*args, _f=getattr(ss.native, name), _n=name, **kw):
            counts[_n] += 1
            return _f(*args, **kw)
        setattr(ss.native, name, counted)
    return counts


def uncount(ss, names=("splice", "resample_rings", "spectrogram_ring", "voice_conversion", "resample", "resample_plan",
                       "spectrogram")):
    for name in names:
        delattr(ss.native, name)


@pytest.mark.parametrize("S", [1, 8, 32])
def test_launches_per_step(conv, S):
    """S sessions at 48 kHz in and out: at most two splices and two ring resamples per step on top of one ring
    spectrogram and one conversion; model-rate sessions in the same object: exactly the calls of a plain step."""
    from openvoice_b200.streaming import StreamingSessions
    ss = StreamingSessions(conv, window_frames=32, rates=(48000,))
    fast = [ss.open(emb(k), emb(k + 1), seed=k, input_sr=48000, output_sr=48000) for k in range(S)]
    slow = [ss.open(emb(k), emb(k + 1), seed=k) for k in range(S)]
    x48, x22 = wave(48000 * 6, 1), wave(SR * 6, 2)
    counts = counting(ss)
    try:
        produced = 0
        for p in range(0, 48000 * 5, 4800):
            before = dict(counts)
            out = ss.push({sid: x48[p:p + 4800] for sid in fast})
            d = {k: counts[k] - before[k] for k in counts}
            assert d["splice"] <= 2 and d["resample_rings"] <= 2 and d["voice_conversion"] <= 1, d
            assert d["resample"] == d["resample_plan"] == d["spectrogram"] == 0, d
            produced += sum(len(v) for v in out.values())
            before = dict(counts)
            ss.push({sid: x22[p * SR // 48000:(p + 4800) * SR // 48000] for sid in slow})
            d = {k: counts[k] - before[k] for k in counts}
            assert d["resample_rings"] == 0 and d["splice"] == 1 and d["voice_conversion"] <= 1, d
        assert produced > 0
    finally:
        uncount(ss)
    ss.close(fast + slow)


def test_steady_lockstep_replays_its_graph(conv):
    from openvoice_b200.streaming import StreamingSessions
    ss = StreamingSessions(conv, window_frames=32, rates=(48000,))
    sids = [ss.open(emb(k), emb(k + 9), tau=0.3, seed=k, input_sr=48000, output_sr=48000) for k in range(8)]
    ws = [wave(48000 * 5, k) for k in range(8)]
    nat = conv.model.native
    before, emitted = nat.graph_replays, 0
    for p in range(0, 48000 * 5, 960):
        out = ss.push({sid: w[p:p + 960] for sid, w in zip(sids, ws)})
        emitted += sum(len(v) for v in out.values())
    assert emitted > 0 and nat.graph_replays >= before + 3, (before, nat.graph_replays)
    ss.close(sids)


def test_push_device_equals_push(conv):
    from openvoice_b200.streaming import StreamingSessions
    x = wave(48000 * 3 + 17, 3)
    rows = np.zeros((2, 96000), np.float32)                # the clip in two device rows
    rows[0], rows[1, :len(x) - 96000] = x[:96000], x[96000:]
    src = torch.from_numpy(rows).cuda()
    runs = [[(0, 0, 30000)], [(0, 30000, 66000)], [(1, 0, len(x) - 96000)]]
    outs = []
    for dev in (False, True):
        ss = StreamingSessions(conv, window_frames=32, rates=(48000,))
        a = ss.open(emb(1), emb(2), seed=5, input_sr=48000, output_sr=48000)
        got, at = [], 0
        for k, r in enumerate(runs):
            last = k == len(runs) - 1
            n = sum(c for _, _, c in r)
            if dev:
                got.append(ss.push_device({a: r}, src, close=[a] if last else ())[a])
            else:
                got.append(ss.push({a: x[at:at + n]})[a])
                if last:
                    got.append(ss.close([a])[a])
            at += n
        outs.append(np.concatenate(got))
    assert at == len(x) and np.array_equal(outs[0], outs[1])


def test_refusals_launch_nothing(conv):
    from openvoice_b200.streaming import StreamingSessions
    for bad in ((44101,), (0,), (-16000,)):
        with pytest.raises(ValueError):
            StreamingSessions(conv, window_frames=32, rates=bad)
    ss = StreamingSessions(conv, window_frames=32, rates=(48000,))
    a = ss.open(emb(1), emb(2), seed=1, input_sr=48000, output_sr=48000)
    b = ss.open(emb(3), emb(4), seed=2)
    ss.push({a: wave(700, 1), b: wave(9000, 2)})
    torch.cuda.synchronize()
    counts = counting(ss)
    try:
        state = {sid: (s.n_in, s.raw_n, s.out_n, s.emitted, s.row) for sid, s in ss.sessions.items()}
        rings = [t.clone() for t in (ss.rings, ss.raw, ss.orings)]
        for kw, name in (({"input_sr": 16000}, "input_sr"), ({"output_sr": 44100}, "output_sr"),
                         ({"input_sr": -48000}, "input_sr"), ({"output_sr": 0}, "output_sr")):
            with pytest.raises(ValueError, match=f"{name}.*declared: 48000"):
                ss.open(emb(5), emb(6), **kw)
        with pytest.raises(ValueError, match="audio too short"):
            ss.close([b, a])                               # a: 700 samples at 48 kHz, 322 at the model's rate
        with pytest.raises(ValueError, match="unknown or closed"):
            ss.push({a: wave(960, 3), 999: wave(441, 3)})
        assert all(v == 0 for v in counts.values()), counts
        assert {sid: (s.n_in, s.raw_n, s.out_n, s.emitted, s.row) for sid, s in ss.sessions.items()} == state
        assert all(torch.equal(t, u) for t, u in zip(rings, (ss.rings, ss.raw, ss.orings)))
    finally:
        uncount(ss)


# ------------------------------------------------------------------------------------------------ CloneSessions
@pytest.fixture(params=["fp32", "f16x3"])
def pair(request, tmp_path_factory):
    return models(tmp_path_factory, request.param)


def run_clone(cs, reqs, out_sr):
    ids = [cs.open(**{k: q[k] for k in ("speaker", "src_se", "tgt_se", "tau", "seed", "convert_seed", "speed",
                                        "noise_scale")}, output_sr=o) for q, o in zip(reqs, out_sr)]
    for sid, q in zip(ids, reqs):
        cs.say(sid, ids=q["ids"])
        cs.end(sid)
    steps = []
    while cs.sessions:
        steps.append({ids.index(sid): c for sid, c in cs.step().items()})
    return steps


def test_clone_sessions_output_rates(pair):
    """A session with output_sr = r returns, step by step, what StreamingResampler(conv, 22050, r) gives for the chunks
    of the same session at the model's rate (flushed at its end); sessions without output_sr are unchanged."""
    from openvoice_b200.streaming import CloneSessions, StreamingResampler
    tts, conv = pair
    reqs = requests(4)
    out_sr = [8000, None, 48000, 16000]
    got = run_clone(CloneSessions(conv, tts, window_frames=64, first_window_frames=16, output_rates=(8000, 16000, 48000)),
                    reqs, out_sr)
    base = run_clone(CloneSessions(conv, tts, window_frames=64, first_window_frames=16), reqs, [None] * 4)
    assert len(got) == len(base)
    rs = {r: StreamingResampler(conv.model, SR, o) for r, o in enumerate(out_sr) if o}
    last = {r: max(t for t, st in enumerate(base) if r in st) for r in range(4)}
    for t, (g, b) in enumerate(zip(got, base)):
        for r in range(4):
            if r not in rs:
                assert (r in g) == (r in b) and (r not in b or np.array_equal(g[r], b[r])), (t, r)
                continue
            want = rs[r].push(b[r]) if r in b else np.zeros(0, np.float32)
            if t == last[r]:
                want = np.concatenate([want, rs[r].flush()])
            assert np.array_equal(g.get(r, np.zeros(0, np.float32)), want), (t, r)
    cs = CloneSessions(conv, tts, output_rates=(48000,))
    with pytest.raises(ValueError, match="output_sr.*declared: 48000"):
        cs.open(**{k: reqs[0][k] for k in ("speaker", "src_se", "tgt_se")}, output_sr=16000)
    with pytest.raises(ValueError, match="output_sr.*declared: none"):
        CloneSessions(conv, tts).open(**{k: reqs[0][k] for k in ("speaker", "src_se", "tgt_se")}, output_sr=48000)
    assert not cs.sessions
