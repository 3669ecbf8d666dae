"""-m gpu: a live stream's source embedding learned from its own audio.

``ovc_reference_encoder_stream`` advances per-stream reference-encoder state rows as audio arrives in device rings; a
snapshot of a prefix equals ``reference_encoder`` on that prefix's spectrogram bit for bit.  ``StreamingSessions`` /
``StreamingConverter`` with ``enroll=`` retarget a session to its snapshots, and equal a plain converter retargeted by
hand to ``extract_se`` of the same prefixes."""
import json

import numpy as np
import pytest
import torch

from oracle import vc_oracle as O

pytestmark = pytest.mark.gpu

HOP, PAD = 256, 384
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


def wave(n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 22050.0
    f = 110 + 40 * seed
    x = 0.3 * np.sin(2 * np.pi * f * t * (1 + 0.2 * np.sin(2 * np.pi * 0.7 * t))) + 0.05 * rng.standard_normal(n)
    return x.astype(np.float32)


def emb(seed):
    return 0.1 * torch.randn(1, 256, 1, generator=torch.Generator().manual_seed(seed))


def prefix_se(conv, y, n):
    """``reference_encoder(spectrogram(y[:n]), lengths)`` -- what ``extract_se`` computes for the prefix."""
    nat = conv.model.native
    w = torch.from_numpy(np.ascontiguousarray(y[:n]))[None].cuda()
    spec, frames = nat.spectrogram(w, torch.tensor([n], dtype=torch.int64, device="cuda"))
    return nat.reference_encoder(spec, frames)[0].cpu()


def rel_err(got, ref):
    ref = np.asarray(ref, dtype=np.float64)
    return float(np.abs(np.asarray(got, dtype=np.float64) - ref).max() / (np.sqrt((ref ** 2).mean()) + 1e-30))


def test_stream_snapshots_equal_prefix_encoder(conv):
    """Streams in mixed chunk sizes, one batched call per round with rows in arbitrary order and small wrapping rings:
    every snapshot equals the whole-prefix encoder bit for bit, and the fp64 oracle within the extract_se gate."""
    nat = conv.model.native
    sizes = [[1, 769, 4000, 22050], [22050, 1, 4000], [769, 769, 1, 4000], [4000, 22050, 22050]]
    lens = [60 * 22050 + 131, 200000, 23456, 100001]
    ys = [wave(n, k + 1) for k, n in enumerate(lens)]
    points = [sorted({385, 512, 640, 641, 767, 1000, 1280, 5003, 12345, 23000, 44100, 100000, 150001, 199999, 300000,
                      600000, 60 * 22050} | {n})
              for n in lens]
    points = [[p for p in pts if p <= n] for pts, n in zip(points, lens)]
    S = len(lens)
    cap, M = 32768, 128
    rings = torch.zeros(S + 1, cap, device="cuda")
    F = nat.refenc_state_floats
    state = torch.zeros(S + 2, F, device="cuda")
    srow, rrow = [2, 0, 3, 1], [3, 1, 0, 2]            # arbitrary state and ring rows
    pos, turn, pend = [0] * S, [0] * S, [list(p) for p in points]
    got, calls = [], 0
    while any(pos[k] < lens[k] for k in range(S)):
        desc, who = [], []
        for k in range(S):
            if pos[k] >= lens[k]:
                continue
            end = min(lens[k], pos[k] + sizes[k][turn[k] % len(sizes[k])])
            crossing = [p for p in pend[k] if p <= end]
            if len(crossing) > 1:                       # one snapshot per call: stop before the second
                end = crossing[1] - 1
            # the ring: samples [pos, end) of stream k at s % cap
            idx = np.arange(pos[k], end)
            rings[rrow[k], torch.from_numpy(idx % cap).cuda()] = torch.from_numpy(ys[k][pos[k]:end]).cuda()
            snap = pend[k].pop(0) if pend[k] and pend[k][0] <= end else 0
            desc.append([srow[k], rrow[k], end, snap])
            who.append((k, snap))
            pos[k], turn[k] = end, turn[k] + 1
        d = torch.tensor(desc, dtype=torch.int64, device="cuda")
        out = nat.reference_encoder_stream(rings, state, d, M)
        calls += 1
        for b, (k, snap) in enumerate(who):
            if snap:
                got.append((k, snap, out[b].cpu()))
    assert sum(len(p) for p in points) == len(got) and all(not p for p in pend)
    sd = O.synthetic_state_dict(1234)
    for k, n, g in got:
        ref = prefix_se(conv, ys[k], n)
        assert torch.equal(g, ref), (k, n, (g - ref).abs().max().item())
    for k, n, g in got[::5]:
        with torch.no_grad():
            spec = O.spectrogram(torch.from_numpy(ys[k][:n].astype(np.float64))[None]).float()
            ref = O.reference_encoder(sd, spec.transpose(1, 2))[0]
        assert rel_err(g.numpy(), ref.numpy()) <= 1e-4, (k, n)


def test_descriptors_are_clamped(conv):
    """Out-of-range descriptor values stay inside rings / state / out: guard regions are untouched, a stale snapshot
    gives NaN and a row that is not named keeps its state."""
    nat = conv.model.native
    F, gin = nat.refenc_state_floats, 256
    cap, R, S, B = 4096, 2, 6, 6
    y = wave(20000, 9)
    rings = torch.zeros(R, cap, device="cuda")
    rings[0] = torch.from_numpy(y[:cap]).cuda()
    rings[1] = torch.from_numpy(y[:cap][::-1].copy()).cuda()
    guard = 7.0
    sbuf = torch.full((F * (S + 2),), guard, device="cuda")
    state = sbuf[F:F * (S + 1)].view(S, F)
    state.zero_()
    obuf = torch.full((gin * (B + 2),), guard, device="cuda")
    out = obuf[gin:gin * (B + 1)].view(B, gin)
    big = 2 ** 62
    desc = torch.tensor([[-5, -7, 3000, 0],                # rows below range -> state row 0, ring row 0
                         [big, big, big, 0],               # above range (state row 5), far-future n_adv -> capped frames
                         [1, 0, -big, -big],               # negative lengths: no advance, no snapshot
                         [5, 1, 2000, big],                # snapshot past what the call can reach -> NaN
                         [4, 1, 2000, 100],                # snapshot too short -> NaN
                         [3, 1, 2000, 385]], dtype=torch.int64, device="cuda")
    nat.reference_encoder_stream(rings, state, desc[:2].contiguous(), 8, out=out[:2])
    torch.cuda.synchronize()
    row1 = state[1].clone()
    nat.reference_encoder_stream(rings, state, desc[2:].contiguous(), 8, out=out[2:])
    stale = torch.tensor([[0, 0, 3000, 1000]], dtype=torch.int64, device="cuda")   # row 0 consumed past 1000 samples
    o1 = nat.reference_encoder_stream(rings, state, stale, 8)
    torch.cuda.synchronize()
    assert torch.all(sbuf[:F] == guard) and torch.all(sbuf[F * (S + 1):] == guard)
    assert torch.all(obuf[:gin] == guard) and torch.all(obuf[gin * (B + 1):] == guard)
    assert torch.all(out[:3] == guard)                     # no snapshot asked: out untouched
    assert torch.isnan(out[3]).all() and torch.isnan(out[4]).all() and torch.isfinite(out[5]).all()
    assert torch.isnan(o1).all()
    assert torch.equal(state[1], row1) and torch.all(state[2] == 0)
    assert torch.isfinite(state).all()
    c0 = state[:, :2].contiguous().view(torch.int64)[:, 0].tolist()
    assert c0 == [10, 0, 0, 6, 6, 8], c0     # the stale call still advanced row 0 to 3000 samples
    ref = prefix_se(conv, y[:cap][::-1].copy(), 385)
    assert torch.equal(out[5].cpu(), ref)
    with pytest.raises(ValueError):
        nat.reference_encoder_stream(rings, state, desc[:, :3].contiguous(), 8)
    with pytest.raises(ValueError):
        nat.reference_encoder_stream(rings, state[:, :-4].contiguous(), desc, 8)
    with pytest.raises(ValueError):
        nat.reference_encoder_stream(rings, state, desc, 0)


# ---------------------------------------------------------------------------------------------- live sessions
W_FR = 64
ENR = dict(every_frames=40, until_frames=130, ramp_frames=8)   # snapshots at 10240, 20480 and 30720 samples


def model_rate(conv, w, sr):
    """The whole stream at the model's rate (what a session's input resampler produces, prefix for prefix)."""
    if sr is None:
        return w
    nat = conv.model.native
    x = torch.from_numpy(w)[None].cuda()
    return nat.resample(x, torch.tensor([len(w)], dtype=torch.int64, device="cuda"), sr, 22050)[0].cpu().numpy()


def chunked(n, sizes):
    out, pos, i = [], 0, 0
    while pos < n:
        out.append((pos, min(n, pos + sizes[i % len(sizes)])))
        pos, i = out[-1][1], i + 1
    return out


@pytest.mark.parametrize("rates", [(None, None), (48000, 16000)])
def test_sessions_with_prior_equal_hand_retargeted_converter(conv, rates):
    """Each enrolling session equals, push by push, a plain StreamingConverter retargeted by hand to extract_se of the
    prefix after the step that crosses it; a non-enrolling session in the same steps equals its plain conversion."""
    from openvoice_b200.streaming import Enrollment, StreamingConverter, StreamingSessions
    enr = Enrollment(**ENR)
    srs = [rates[0], rates[1], None]
    lens = [(48000 if r == 48000 else 16000 if r == 16000 else 22050) * 3 + 77 for r in srs]
    ws = [wave(n, 20 + k) for k, n in enumerate(lens)]
    ys = [model_rate(conv, w, r) for w, r in zip(ws, srs)]
    sizes = [[4000, 769, 22050], [1, 769, 30000], [3000]]
    flags = [True, True, False]
    src, tgt = emb(1), emb(2)
    ss = StreamingSessions(conv, window_frames=W_FR, rates=[r for r in srs if r])
    ids = [ss.open(src, tgt, seed=10 + k, input_sr=srs[k], enroll=enr if flags[k] else None) for k in range(3)]
    refs = [StreamingConverter(conv, src, tgt, window_frames=W_FR, request_seed=10 + k, input_sr=srs[k]) for k in range(3)]
    plans = [chunked(n, sz) for n, sz in zip(lens, sizes)]
    E = enr.every_frames * HOP
    snapped = 0
    for step in range(max(len(p) for p in plans) + 1):
        chunks = {ids[k]: ws[k][plans[k][step][0]:plans[k][step][1]] for k in range(3) if step < len(plans[k])}
        closing = [ids[k] for k in range(3) if step == len(plans[k])]
        got = ss.push(chunks) if chunks else {}
        got.update(ss.close(closing) if closing else {})
        for k in range(3):
            sid, rc = ids[k], refs[k]
            if step < len(plans[k]):
                n0 = rc.n_in
                want = rc.push(chunks[sid])
                kk = enr.snapshot(n0, rc.n_in, HOP) if flags[k] else 0
                if kk:
                    rc.retarget(src_se=prefix_se(conv, ys[k], kk * E)[None, :, None], ramp_frames=enr.ramp_frames)
                    snapped += 1
            elif step == len(plans[k]):
                want = rc.flush()
            else:
                continue
            assert np.array_equal(got[sid], want), (k, step)
    assert snapped >= 3


def test_sessions_without_prior_equal_convert_with_their_track(conv):
    """No prior: nothing is converted before the first snapshot; the whole output equals convert with the session's
    source track, whose first key is (0, extract_se of the first every_frames * hop samples)."""
    from openvoice_b200.streaming import Enrollment, StreamingSessions
    enr = Enrollment(**ENR)
    w = wave(22050 * 3 + 500, 31)
    tgt = emb(3)
    ss = StreamingSessions(conv, window_frames=W_FR)
    sid = ss.open(None, tgt, seed=77, enroll=enr)
    other = ss.open(emb(4), tgt, seed=78)
    outs, E = [], enr.every_frames * HOP
    for a, b in chunked(len(w), [769, 4000]):
        got = ss.push({sid: w[a:b], other: w[a:b]})
        if b < E:
            assert len(got[sid]) == 0
        outs.append(got[sid])
    tr = ss.tone_track(sid, "src")
    outs.append(ss.close([sid, other])[sid])
    assert tr.frames[0] == 0 and torch.equal(tr.se[0].reshape(-1), prefix_se(conv, w, E))
    assert len(tr.frames) > 1
    want = conv.convert(w, tr, tgt, seed=77)
    assert np.array_equal(np.concatenate(outs), want)
    with pytest.raises(ValueError):
        ss.open(None, tgt)
    short = ss.open(None, tgt, enroll=enr)
    ss.push({short: w[:5000]})
    with pytest.raises(ValueError):                       # no source before the first snapshot: nothing to read
        ss.tone_track(short, "src")
    with pytest.raises(ValueError):                       # ... or to ramp from
        ss.retarget(short, src_se=emb(9))
    ss.retarget(short, tgt_se=emb(9))
    with pytest.raises(ValueError):
        ss.close([short])
    ss.discard([short])


def test_source_se_and_converter_equal_the_session(conv):
    """source_se after arbitrary pushes equals extract_se of everything received, and StreamingConverter(enroll=)
    equals the same session push by push (with and without a prior)."""
    from openvoice_b200.streaming import Enrollment, StreamingConverter, StreamingSessions
    enr = Enrollment(**ENR)
    w = wave(22050 * 2 + 999, 41)
    tgt = emb(5)
    ss = StreamingSessions(conv, window_frames=W_FR)
    for prior in (emb(6), None):
        sid = ss.open(prior, tgt, seed=5, enroll=enr)
        sc = StreamingConverter(conv, prior, tgt, window_frames=W_FR, request_seed=5, enroll=enr)
        n = 0
        for a, b in chunked(len(w), [1, 5000, 769, 22050, 3]):
            got, want = ss.push({sid: w[a:b]})[sid], sc.push(w[a:b])
            assert np.array_equal(got, want), (a, b)
            n = b
            if n > 400 and (a // 769) % 3 == 0:
                se, m = ss.source_se(sid)
                assert m == n and torch.equal(se.reshape(-1), prefix_se(conv, w, n)), n
                se2, _ = sc.source_se()
                assert torch.equal(se2, se)
        assert np.array_equal(ss.close([sid])[sid], sc.flush())
    plain = ss.open(emb(6), tgt)
    with pytest.raises(ValueError):
        ss.source_se(plain)


def test_one_encoder_call_per_step(conv, monkeypatch):
    """A step naming 1 or 16 enrolling sessions makes exactly one reference_encoder_stream call; one naming none
    makes no call."""
    from openvoice_b200.streaming import Enrollment, StreamingSessions
    nat = conv.model.native
    calls = []
    real = type(nat).reference_encoder_stream
    monkeypatch.setattr(type(nat), "reference_encoder_stream",
                        lambda self, *a, **k: (calls.append(1), real(self, *a, **k))[1])
    ss = StreamingSessions(conv, window_frames=W_FR)
    enr = Enrollment(**ENR)
    plain = [ss.open(emb(7), emb(8)) for _ in range(3)]
    enrolled = [ss.open(emb(7), emb(8), enroll=enr) for _ in range(16)]
    w = wave(12000, 50)
    for group in ([enrolled[0]], enrolled, plain):
        calls.clear()
        ss.push({sid: w[:11000] if group is not plain else w[:3000] for sid in group})
        assert len(calls) == (0 if group is plain else 1)
    calls.clear()
    ss.push({plain[0]: w[:100], enrolled[1]: w[:100]})
    assert len(calls) == 1


def test_first_snapshot_next_to_a_ramping_session(conv):
    """A session without a prior takes its first snapshot in a step whose launch is per-frame because another session
    is inside a source ramp: both equal their own StreamingConverter push by push (the new source reaches the
    per-frame conditioning too)."""
    from openvoice_b200.streaming import Enrollment, StreamingConverter, StreamingSessions
    enr = Enrollment(every_frames=200, until_frames=400, ramp_frames=8)   # first snapshot at 51 200 samples
    ws = [wave(22050 * 4 + 300, 51), wave(22050 * 4 + 300, 52)]
    src, tgt = emb(10), emb(11)
    ss = StreamingSessions(conv, window_frames=W_FR)
    a = ss.open(src, tgt, seed=1)
    b = ss.open(None, tgt, seed=2, enroll=enr)
    ra = StreamingConverter(conv, src, tgt, window_frames=W_FR, request_seed=1)
    rb = StreamingConverter(conv, None, tgt, window_frames=W_FR, request_seed=2, enroll=enr)
    plan = chunked(len(ws[0]), [22050])
    firsts = 0
    for step, (p, q) in enumerate(plan):
        got = ss.push({a: ws[0][p:q], b: ws[1][p:q]})
        want_a, want_b = ra.push(ws[0][p:q]), rb.push(ws[1][p:q])
        if p < enr.every_frames * HOP <= q:
            firsts += 1
            assert len(got[a]) and len(got[b])                # both convert windows in the first-snapshot step
            assert ss.tone_track(a, "src").frames[-1] > q // HOP   # a's windows in this step are inside its ramp
        assert np.array_equal(got[a], want_a), step
        assert np.array_equal(got[b], want_b), step
        if step == 0:                                         # a long source ramp that covers the snapshot step
            assert ss.retarget(a, src_se=emb(12), ramp_frames=600) == ra.retarget(src_se=emb(12), ramp_frames=600)
    out = ss.close([a, b])
    assert np.array_equal(out[a], ra.flush()) and np.array_equal(out[b], rb.flush())
    assert firsts == 1


def test_converter_snapshot_in_the_flush_lands_after_the_last_window(conv):
    """At another input rate, the resampler's tail pushed at flush can cross a snapshot boundary.  The snapshot then
    takes effect after the stream's last window, in StreamingConverter as in the session's closing step: both equal
    convert with the prior."""
    from openvoice_b200._native import resample_span
    from openvoice_b200.streaming import Enrollment, StreamingConverter, StreamingSessions
    enr = Enrollment(**ENR)
    E = enr.every_frames * HOP
    L = next(n for n in range(E * 48000 // 22050 - 64, E * 48000 // 22050 + 64)
             if resample_span(48000, 22050, n)[1] < E <= resample_span(48000, 22050, n)[0])
    w = wave(L, 61)
    src, tgt = emb(13), emb(14)
    ss = StreamingSessions(conv, window_frames=W_FR, rates=[48000])
    sid = ss.open(src, tgt, seed=3, input_sr=48000, enroll=enr)
    sc = StreamingConverter(conv, src, tgt, window_frames=W_FR, request_seed=3, input_sr=48000, enroll=enr)
    outs_s, outs_c = [], []
    for p, q in chunked(L, [4000, 769]):
        outs_s.append(ss.push({sid: w[p:q]})[sid])
        outs_c.append(sc.push(w[p:q]))
    assert sc.tone_track("src").frames[-1] == 0           # no snapshot before the flush
    outs_s.append(ss.close([sid])[sid])
    outs_c.append(sc.flush())
    got_s, got_c = np.concatenate(outs_s), np.concatenate(outs_c)
    assert np.array_equal(got_s, got_c)
    assert np.array_equal(got_c, conv.convert(w, src, tgt, seed=3, sr=48000))
