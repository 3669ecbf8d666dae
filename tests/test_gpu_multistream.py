"""-m gpu: multi-session streaming (openvoice_b200.streaming.StreamingSessions) and its front end,
ovc_spectrogram_ring.  Ring spectrogram frames equal the whole clip's, and every session equals its own
StreamingConverter(request_seed=...) bit for bit, whatever company it keeps."""
import json

import numpy as np
import pytest
import torch

from oracle import vc_oracle as O

pytestmark = pytest.mark.gpu

HOP, PAD, H = 256, 384, 128

_convs = {}


@pytest.fixture(params=["fp32", "f16x3"])
def conv(request, tmp_path_factory):
    from openvoice_b200.api import ToneColorConverter
    if request.param not in _convs:
        cfg = tmp_path_factory.mktemp("cfg") / "config.json"
        cfg.write_text(json.dumps(O.DEFAULT_HPARAMS))
        c = ToneColorConverter(str(cfg), device="cuda:0", enable_watermark=False, precision=request.param)
        c.model.load_state_dict(O.synthetic_state_dict(1234))
        _convs[request.param] = c
    return _convs[request.param]


def rel_err(got, ref):
    ref = np.asarray(ref, dtype=np.float64)
    return float(np.abs(np.asarray(got, dtype=np.float64) - ref).max() / (np.sqrt((ref ** 2).mean()) + 1e-30))


def wave(n, seed):
    rng = np.random.default_rng(seed)
    return (0.5 * (2 * rng.random(n, dtype=np.float32) - 1)).astype(np.float32)


def emb(seed):
    return 0.1 * torch.randn(1, 256, 1, generator=torch.Generator().manual_seed(seed))


def streaming_converter(conv, w, sizes, W, src, tgt, tau, seed):
    from openvoice_b200.streaming import StreamingConverter
    sc = StreamingConverter(conv, src, tgt, tau=tau, window_frames=W, request_seed=seed)
    outs, pos, i = [], 0, 0
    while pos < len(w):
        n = min(sizes[i % len(sizes)], len(w) - pos)
        outs.append(sc.push(w[pos:pos + n]))
        pos, i = pos + n, i + 1
    return np.concatenate(outs + [sc.flush()])


class Driver:
    """Runs StreamingSessions over scripted sessions: (wave, chunk sizes, src, tgt, tau, seed, step of open).  Each
    session is closed in the step after its last push; collects every session's output, rows in use and the audio each
    session keeps beyond its largest push."""

    def __init__(self, ss, script):
        self.ss, self.script = ss, script
        self.outs = {k: [] for k in range(len(script))}
        self.max_rows, self.max_keep = 0, 0

    def run(self):
        ss, script = self.ss, self.script
        ids, pos, turn, done, biggest, step = {}, [0] * len(script), [0] * len(script), set(), [0] * len(script), 0
        while len(done) < len(script):
            for k, (_, _, src, tgt, tau, seed, start) in enumerate(script):
                if step == start:
                    ids[k] = ss.open(src, tgt, tau=tau, seed=seed)
            owner = {sid: k for k, sid in ids.items() if k not in done}
            chunks, ending = {}, []
            for sid, k in owner.items():
                w, sizes = script[k][0], script[k][1]
                if pos[k] >= len(w):
                    ending.append(sid)
                    continue
                n = min(sizes[turn[k] % len(sizes)], len(w) - pos[k])
                chunks[sid] = w[pos[k]:pos[k] + n]
                pos[k], turn[k], biggest[k] = pos[k] + n, turn[k] + 1, max(biggest[k], n)
            for sid, y in ss.push(chunks).items():
                self.outs[owner[sid]].append(y)
            for sid in chunks:
                self.max_keep = max(self.max_keep, ss.state_samples(sid) - biggest[owner[sid]])
            self.max_rows = max(self.max_rows, ss.rows_in_use)
            if ending:
                for sid, y in ss.close(ending).items():
                    self.outs[owner[sid]].append(y)
                done.update(owner[sid] for sid in ending)
            step += 1
        return [np.concatenate(self.outs[k]) for k in range(len(script))]


# ------------------------------------------------------------------------------------------------ 1. ring spectrogram
def test_ring_spectrogram_equals_whole_clip(conv):
    """Windows at the stream start (reflect), in the middle across a ring wraparound, and at the end of a closed stream,
    in one batch mixing open and closed streams: array_equal to the matching columns of the whole clip's spectrogram,
    zeros after each item's frames."""
    from openvoice_b200._native import STREAM_OPEN
    nat = conv.model.native
    L, cap = 22050 * 4 + 77, 8192
    x = torch.from_numpy(wave(L, 1)).cuda()
    whole, _ = nat.spectrogram(x[None].contiguous(), torch.tensor([L], dtype=torch.int64, device="cuda"))
    T = L // HOP
    items = ((0, 20, 30 * HOP, False), (120, 24, 150 * HOP, False), (T - 15, 15, L, True), (T - 25, 25, L, True))
    rings = torch.full((len(items), cap), float("nan"), device="cuda")
    for r, (lo, n, upto, _) in enumerate(items):
        a = max(0, lo * HOP - PAD)
        rings[r, torch.from_numpy(np.arange(a, upto) % cap).cuda()] = x[a:upto]
    assert (120 * HOP - PAD) // cap != (143 * HOP - PAD + 1023) // cap     # item 1 wraps around its ring row
    assert all(upto - max(0, lo * HOP - PAD) <= cap for lo, _, upto, _ in items)   # every window's samples fit its row
    i64 = lambda v: torch.tensor(v, dtype=torch.int64, device="cuda")   # noqa: E731
    Tmax = 32
    spec = nat.spectrogram_ring(rings, i64(list(range(len(items)))), i64([it[0] for it in items]),
                                i64([it[1] for it in items]), i64([L if it[3] else STREAM_OPEN for it in items]), Tmax)
    torch.cuda.synchronize()
    for b, (lo, n, _, _) in enumerate(items):
        assert torch.equal(spec[b, :, :n], whole[0, :, lo:lo + n]), b
        assert torch.equal(spec[b, :, n:], torch.zeros_like(spec[b, :, n:])), b


# ------------------------------------------------------------------------------------------------ 2. = StreamingConverter
def test_sessions_equal_streaming_converters(conv):
    """Six staggered sessions (rows reused after closes): one shorter than window + halo, one ending exactly on a window
    edge, one over 20 s; 441-sample, irregular and whole-clip pushes; distinct embeddings, taus (one 0) and seeds.  Each
    equals its own StreamingConverter bit for bit and convert(seed=...) within the streaming bound, and state stays
    bounded."""
    from openvoice_b200.streaming import StreamingSessions
    W = 64
    lens = (22050 + 5, HOP * 6 * W + 100, 22050 * 21 + 313, 22050 * 3 + 17, 22050 * 4 + 1, 22050 * 5 + 201)
    sizes = ([441], [441, 1000, 37, 5000], [441], [10 ** 9], [4096, 17, 8191], [441])
    taus = (0.3, 0.0, 0.3, 1.0, 0.5, 0.0)
    seeds = (7, 2 ** 64 - 1, 123456789, 0, 2 ** 40 + 3, 99)
    starts = (0, 0, 3, 5, 150, 700)
    script = [(wave(n, 10 + k), sizes[k], emb(2 * k), emb(2 * k + 1), taus[k], seeds[k], starts[k])
              for k, n in enumerate(lens)]
    assert lens[0] < HOP * (W + H) and (lens[1] // HOP) % W == 0 and lens[2] > 22050 * 20
    ss = StreamingSessions(conv, window_frames=W)
    d = Driver(ss, script)
    got = d.run()
    assert ss.rows < len(script)                    # later sessions took closed sessions' rows
    for k, (w, sz, src, tgt, tau, seed, _) in enumerate(script):
        ref = streaming_converter(conv, w, sz, W, src, tgt, tau, seed)
        assert got[k].shape == ref.shape == (HOP * (len(w) // HOP),), k
        assert np.array_equal(got[k], ref), (k, rel_err(got[k], ref))
        whole = conv.convert(w, src, tgt, tau=tau, seed=seed)
        assert whole.shape == got[k].shape and rel_err(got[k], whole) <= 2e-6, k
    # state: rows of the open sessions only; per session the two halos, one window and the STFT lead beyond its largest
    # push (test_streaming_equals_whole_clip's frame bound, in samples)
    assert d.max_rows <= len(script)
    assert d.max_keep <= HOP * (W + 2 * H + 8), d.max_keep


# ------------------------------------------------------------------------------------------------ 3. company
def test_company_does_not_matter(conv):
    from openvoice_b200.streaming import StreamingSessions
    W = 32
    me = (wave(22050 * 5 + 99, 1), [441], emb(1), emb(2), 0.3, 4242, 0)
    rng = np.random.default_rng(5)
    others = [(wave(int(rng.integers(22050 * 2, 22050 * 4)), 50 + k), [int(v) for v in rng.integers(100, 3000, 3)],
               emb(10 + k), emb(40 + k), float(rng.choice([0.0, 0.3, 0.7])), 1000 + k, int(rng.integers(0, 200)))
              for k in range(31)]
    alone = Driver(StreamingSessions(conv, window_frames=W), [me]).run()[0]
    crowd = Driver(StreamingSessions(conv, window_frames=W), others[:15] + [me] + others[15:]).run()[15]
    assert np.array_equal(alone, crowd)


# ------------------------------------------------------------------------------------------------ 4. graph replay
def test_steady_lockstep_step_replays_its_graph(conv):
    from openvoice_b200.streaming import StreamingSessions
    ss = StreamingSessions(conv, window_frames=32)
    sids = [ss.open(emb(k), emb(k + 9), tau=0.3, seed=k) for k in range(8)]
    ws = [wave(22050 * 5, k) for k in range(8)]
    nat = conv.model.native
    before, emitted = nat.graph_replays, 0
    for p in range(0, 22050 * 5, 441):
        out = ss.push({sid: w[p:p + 441] for sid, w in zip(sids, ws)})
        emitted += sum(len(v) for v in out.values())
    assert emitted > 0 and nat.graph_replays >= before + 3, (before, nat.graph_replays)
    ss.close(sids)


# ------------------------------------------------------------------------------------------------ 5. refusals
def test_refusals_launch_nothing(conv):
    from openvoice_b200.streaming import StreamingSessions
    with pytest.raises(ValueError, match="window_frames"):
        StreamingSessions(conv, window_frames=0)
    ss = StreamingSessions(conv, window_frames=32)
    a = ss.open(emb(1), emb(2), seed=1)
    b = ss.open(emb(3), emb(4), seed=2)
    ss.push({a: wave(300, 1), b: wave(9000, 2)})
    torch.cuda.synchronize()
    nat, counts = ss.native, {}
    for name in ("spectrogram_ring", "voice_conversion", "spectrogram", "convert_waveform"):
        def counted(*args, _f=getattr(nat, name), _n=name, **kw):
            counts[_n] = counts.get(_n, 0) + 1
            return _f(*args, **kw)
        setattr(nat, name, counted)
    try:
        state = {sid: (s.n_in, s.emitted, s.row) for sid, s in ss.sessions.items()}
        rings = ss.rings.clone()
        with pytest.raises(ValueError, match="unknown or closed"):
            ss.push({a: wave(441, 3), 999: wave(441, 3)})
        with pytest.raises(ValueError, match="audio too short"):
            ss.close([b, a])
        for bad in (2 ** 64, -5, 0.5):
            with pytest.raises(ValueError, match="seed"):
                ss.open(emb(5), emb(6), seed=bad)
        with pytest.raises(ValueError, match="src_se"):
            ss.open(torch.zeros(1, 255, 1), emb(6))
        with pytest.raises(ValueError, match="input_sr"):
            ss.open(emb(5), emb(6), input_sr=48000)
        assert counts == {}
        assert {sid: (s.n_in, s.emitted, s.row) for sid, s in ss.sessions.items()} == state
        assert torch.equal(ss.rings, rings)
        ss.close([b])
        with pytest.raises(ValueError, match="unknown or closed"):
            ss.push({b: wave(441, 4)})
        assert counts.get("voice_conversion", 0) >= 1
    finally:
        for name in ("spectrogram_ring", "voice_conversion", "spectrogram", "convert_waveform"):
            delattr(nat, name)
