"""-m gpu: staged live sessions (openvoice_b200.streaming.StagedSessions) and the library pieces under them: the latent
half of ovc_voice_conversion_frames (o_hat NULL), ovc_generate_frames and ovc_splice's source wrap.  The two halves
compose to the whole conversion bit for bit; sessions are within the streaming bound of convert on the whole clip and
depend on their own stream only."""
import json

import numpy as np
import pytest
import torch
from scipy.signal import firwin

from oracle import vc_oracle as O

pytestmark = pytest.mark.gpu

HOP, SR = 256, 22050
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


def i64(v):
    return torch.tensor(v, dtype=torch.int64, device="cuda")


def run(ss, script, device_src=False):
    """Drives sessions (wave, chunk sizes, src, tgt, seed, step of open, open kwargs), closing each in the step after its
    last push; returns each session's concatenated output.  ``device_src``: push every step's chunks with push_device
    from one device array."""
    ids, pos, turn, done, step = {}, [0] * len(script), [0] * len(script), set(), 0
    outs = {k: [] for k in range(len(script))}
    while len(done) < len(script):
        for k, (_, _, src, tgt, seed, start, kw) in enumerate(script):
            if step == start:
                ids[k] = ss.open(src, tgt, seed=seed, **kw)
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
        if device_src and chunks:
            flat = np.concatenate(list(chunks.values()) + [np.zeros(1, np.float32)])
            at = np.cumsum([0] + [len(c) for c in chunks.values()])
            res = ss.push_device({sid: [(0, int(at[j]), len(c))] for j, (sid, c) in enumerate(chunks.items())},
                                 torch.from_numpy(flat).cuda()[None].contiguous())
        else:
            res = ss.push(chunks)
        for sid in chunks:
            outs[owner[sid]].append(res[sid])
        if ending:
            for sid, y in ss.close(ending).items():
                outs[owner[sid]].append(y)
            done.update(owner[sid] for sid in ending)
        step += 1
    return [np.concatenate(outs[k]) for k in range(len(script))]


# ------------------------------------------------------------------------------------------------ 1. the two halves
@pytest.mark.parametrize("per_frame", [False, True])
def test_latent_and_generator_halves_compose_bit_for_bit(conv, per_frame):
    """A ragged batch with per-item seeds and frame offsets: the latent half's z_hat equals the whole call's z_hat and
    the generator on it equals the whole call's o_hat, array_equal, with per-item or per-frame target embeddings."""
    nat = conv.model.native
    B, T = 3, 96
    lens = i64([96, 61, 17])
    x = torch.from_numpy(np.stack([wave(HOP * T + 768, k) for k in range(B)])).cuda()
    spec, _ = nat.spectrogram(x, i64([HOP * T + 768] * B))
    spec = spec[:, :, :T].contiguous()
    gs = torch.cat([emb(k) for k in range(B)]).reshape(B, 256).cuda()
    gt = torch.cat([emb(10 + k) for k in range(B)]).reshape(B, 256).cuda()
    if per_frame:
        ramp = torch.linspace(0, 1, T, device="cuda")
        gt = (gt[:, :, None] * (1 - ramp) + gs[:, :, None] * ramp).contiguous()
    items = {"seed": i64([5, 2 ** 40, 7]), "stream": i64([0, 0, 0]), "frame0": i64([0, 300, 12]),
             "tau": torch.tensor([0.3, 0.0, 0.7], device="cuda")}
    o, (_, _, zh) = nat.voice_conversion(spec, lens, gs, gt, ragged=True, items=items)
    z = nat.latent(spec, lens, gs, gt, items=items)
    g = nat.generate(z, lens, gt)
    torch.cuda.synchronize()
    assert torch.equal(z, zh)
    assert torch.equal(g, o)
    with pytest.raises(Exception, match="target side only"):
        _generate_src_frames(nat, z, lens, gt)


def _generate_src_frames(nat, z, lens, gt):
    """ovc_generate_frames asked for a per-frame source side, which the generator never reads."""
    import ctypes as C
    from openvoice_b200._native import SE_FRAMES_SRC, _check
    o = torch.empty(z.shape[0], 1, HOP * z.shape[2], device="cuda")
    rc = nat.lib.ovc_generate_frames(nat.handle, C.c_void_p(z.data_ptr()), C.c_void_p(lens.data_ptr()),
                                     C.c_void_p(gt.data_ptr()), SE_FRAMES_SRC, z.shape[0], z.shape[2],
                                     C.c_void_p(o.data_ptr()), None)
    _check(nat.lib, rc, "ovc_generate_frames")


# ------------------------------------------------------------------------------------------------ 2. source wrap
def test_splice_source_wrap_equals_indexing(conv):
    """Segments reading across a source ring's wrap, with offsets past the pitch and negative, counts past the pitch,
    rows out of range and gaps: equal to torch indexing of the clamp rules, bit for bit; the guard regions around both
    buffers stay untouched."""
    nat = conv.model.native
    rows, pitch, drows, dcap, guard = 3, 50, 4, 70, 64
    sbuf = torch.full((guard + rows * pitch + guard,), 7.0, device="cuda")
    src = sbuf[guard:guard + rows * pitch].view(rows, pitch)
    src.copy_(torch.randn(rows, pitch, generator=torch.Generator().manual_seed(1)).cuda())
    dbuf = torch.full((guard + drows * dcap + guard,), float("nan"), device="cuda")
    dst = dbuf[guard:guard + drows * dcap].view(drows, dcap)
    dst.zero_()
    segs = [(0, 45, 12, 0, 0), (1, 120, 10, 1, 65), (2, -7, 5, 2, 3), (9, 3, 55, 3, 0), (-1, 0, 6, 0, 30),
            (1, 10, 0, 1, 0), (-5, 2, 4, 7, -10)]            # no two segments write one slot
    nat.splice(src.contiguous(), i64(segs), dst.contiguous(), src_wrap=True)
    torch.cuda.synchronize()
    want = torch.zeros(drows, dcap)
    s_h = src.cpu()
    for r, off, n, dr, do in segs:
        dr = min(max(dr, 0), drows - 1)
        n = min(max(n, 0), dcap)
        for i in range(n):
            v = 0.0 if r < 0 else s_h[min(r, rows - 1), (off % pitch + i) % pitch]
            want[dr, (do % dcap + i) % dcap] = v
    assert torch.equal(dst.cpu(), want)
    assert (sbuf[:guard] == 7).all() and (sbuf[guard + rows * pitch:] == 7).all()
    assert torch.isnan(dbuf[:guard]).all() and torch.isnan(dbuf[guard + drows * dcap:]).all()


# ------------------------------------------------------------------------------------------------ 3. against convert
@pytest.mark.parametrize("W", [8, 16, 32, 256])
def test_sessions_within_streaming_bound_of_convert(conv, W):
    """Five staggered sessions: 441-sample and random chunkings, a clip shorter than one window, one shorter than both
    halos, and one ending on a window edge.  Each is within 2e-6 * rms of convert on the whole clip with its seed."""
    from openvoice_b200.streaming import StagedSessions
    rng = np.random.default_rng(W)
    lens = (22050 * 3 + 5, 22050 * 2 + 301, HOP * (W // 2 + 3) + 11, HOP * 60 + 400, HOP * 4 * W)
    sizes = ([441], [int(v) for v in rng.integers(1, 5000, 17)], [441], [700, 13], [441])
    script = [(wave(n, 100 + k), sizes[k], emb(2 * k), emb(2 * k + 1), 31 + k, 2 * k, {"tau": 0.3 * (k % 3)})
              for k, n in enumerate(lens)]
    ss = StagedSessions(conv, window_frames=W)
    got = run(ss, script)
    assert ss.rows_in_use == 0
    for k, (w, _, src, tgt, seed, _, kw) in enumerate(script):
        whole = conv.convert(w, src, tgt, tau=kw["tau"], seed=seed)
        assert got[k].shape == whole.shape, k
        assert rel_err(got[k], whole) <= 2e-6, (k, rel_err(got[k], whole))


# ------------------------------------------------------------------------------------------------ 4. independence
def test_chunking_and_company_do_not_matter(conv):
    """A session's audio is bit-identical under 441-sample, random and whole-clip pushes, run alone or among 7 others
    that open and close at other times; push_device gives the same audio as push."""
    from openvoice_b200.streaming import StagedSessions
    W = 32
    w = wave(22050 * 4 + 77, 9)
    rng = np.random.default_rng(3)
    me = [(w, sz, emb(1), emb(2), 4242, 0, {}) for sz in ([441], [int(v) for v in rng.integers(1, 9000, 11)], [10 ** 9])]
    alone = [run(StagedSessions(conv, window_frames=W), [m])[0] for m in me]
    assert all(np.array_equal(a, alone[0]) for a in alone[1:])
    others = [(wave(int(rng.integers(22050, 22050 * 5)), 50 + k), [int(v) for v in rng.integers(100, 3000, 3)],
               emb(10 + k), emb(40 + k), 1000 + k, int(rng.integers(0, 150)), {"tau": 0.5}) for k in range(7)]
    crowd = run(StagedSessions(conv, window_frames=W), others[:3] + [me[0]] + others[3:])
    assert np.array_equal(crowd[3], alone[0])
    dev = run(StagedSessions(conv, window_frames=W), others[:3] + [me[0]] + others[3:], device_src=True)
    assert all(np.array_equal(a, b) for a, b in zip(dev, crowd))


# ------------------------------------------------------------------------------------------------ 5. tone colour
def test_retarget_and_enrollment_follow_their_tracks(conv):
    """A session retargeted mid-stream (hard, then ramped) and one enrolling its source without a prior: each equals
    convert with its tone tracks within the streaming bound.  retarget returns the ready frames, as StreamingSessions
    does."""
    from openvoice_b200.streaming import Enrollment, StagedSessions, ready_frames
    W = 16
    ss = StagedSessions(conv, window_frames=W)
    w1, w2 = wave(22050 * 4 + 31, 1), wave(22050 * 3 + 500, 2)
    a = ss.open(emb(1), emb(2), seed=5)
    b = ss.open(None, emb(3), seed=6, enroll=Enrollment(every_frames=40, until_frames=130, ramp_frames=8))
    outs = {a: [], b: []}
    for p in range(0, len(w1), 441):
        chunks = {a: w1[p:p + 441]}
        if p < len(w2):
            chunks[b] = w2[p:p + 441]
        for sid, y in ss.push(chunks).items():
            outs[sid].append(y)
        if p == 441 * 60:
            assert ss.retarget(a, tgt_se=emb(7)) == ready_frames(p + 441, HOP, 1024, False)
        if p == 441 * 120:
            ss.retarget(a, src_se=emb(8), tgt_se=emb(9), ramp_frames=20)
        if p + 441 >= len(w2) and b in chunks:
            tb = (ss.tone_track(b, "src"), ss.tone_track(b, "tgt"))
            outs[b].append(ss.close([b])[b])
    ta = (ss.tone_track(a, "src"), ss.tone_track(a, "tgt"))
    outs[a].append(ss.close([a])[a])
    for sid, w, (src, tgt), seed in ((a, w1, ta, 5), (b, w2, tb, 6)):
        assert len(src.frames) > 1 or len(tgt.frames) > 1
        whole = conv.convert(w, src, tgt, seed=seed)
        got = np.concatenate(outs[sid])
        assert got.shape == whole.shape and rel_err(got, whole) <= 2e-6, (sid, rel_err(got, whole))


# ------------------------------------------------------------------------------------------------ 6. rates
def test_other_rates(conv):
    """Sessions at 48 kHz and 8 kHz in and out: within the model-rate bound times the output filter's error gain of
    convert on the whole clip resampled to the session's rate."""
    from openvoice_b200.streaming import StagedSessions
    nat = conv.model.native
    ss = StagedSessions(conv, window_frames=32, rates=(48000, 8000))
    script = [(wave(int(2.5 * r), 60 + k), [r // 50], emb(k), emb(k + 5), 70 + k, 0, {"input_sr": r, "output_sr": r})
              for k, r in enumerate((48000, 8000))]
    got = run(ss, script)
    for k, (w, _, src, tgt, seed, _, kw) in enumerate(script):
        r = kw["input_sr"]
        whole = conv.convert(w, src, tgt, seed=seed, sr=r)
        x = torch.from_numpy(whole).cuda()[None]
        ref = nat.resample(x, i64([len(whole)]), SR, r)[0].cpu().numpy()
        from math import gcd
        up, down = r // gcd(SR, r), SR // gcd(SR, r)
        q = max(up, down)
        h = firwin(20 * q + 1, 1.0 / q, window=("kaiser", 5.0)) * up
        gain = max(np.abs(h[p::up]).sum() for p in range(up))
        assert got[k].shape == ref.shape, k
        assert rel_err(got[k], ref) <= 2e-6 * gain, (r, rel_err(got[k], ref), gain)


# ------------------------------------------------------------------------------------------------ 7. discard
def test_discard_frees_both_rings_rows(conv):
    """A discarded session's row (audio ring and latent ring) is the next open's, and the new session's audio is the
    same as on a fresh StagedSessions."""
    from openvoice_b200.streaming import StagedSessions
    ss = StagedSessions(conv, window_frames=16)
    a = ss.open(emb(1), emb(2), seed=1)
    ss.push({a: wave(22050, 1)})
    row = ss.sessions[a].row
    ss.discard([a])
    assert ss.rows_in_use == 0
    w = wave(22050 * 2 + 3, 2)
    script = [(w, [441], emb(3), emb(4), 9, 0, {})]
    got = run(ss, script)[0]
    assert ss.free_rows.count(row) == 1 and ss.lrings.shape[0] == ss.rows * ss.C
    assert np.array_equal(got, run(StagedSessions(conv, window_frames=16), script)[0])
