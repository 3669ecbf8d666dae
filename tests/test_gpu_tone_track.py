"""-m gpu: time-varying tone colour -- per-frame source / target embeddings ([B, gin, T], the reference's
SynthesizerTrn.voice_conversion form) and keyframe tracks (``ToneTrack``, include/ovc.h: ovc_tone_track_expand).

Against the CPU oracle (which takes per-frame embeddings exactly as the reference does: every conditioning layer is a
1x1 conv added to per-frame activations) within the gates of test_gpu_parity.py; everything else bit for bit: a
constant per-frame embedding against the per-item call, a track against its dense form, batches and windows against
``convert``."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import vc_oracle as O

pytestmark = pytest.mark.gpu
GIN = 256
REL = 1e-4
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def rel_err(got, ref):
    ref = np.asarray(ref, dtype=np.float64)
    return float(np.abs(np.asarray(got, dtype=np.float64) - ref).max() / (np.sqrt((ref ** 2).mean()) + 1e-30))


def se(seed, n=1):
    gen = torch.Generator().manual_seed(seed)
    return [0.1 * torch.randn(1, GIN, 1, generator=gen) for _ in range(n)]


def morph(a, b, T):
    """[1, gin, T]: a linear morph from a to b over the clip."""
    w = torch.linspace(0, 1, T).view(1, 1, T)
    return (a + w * (b - a)).contiguous()


def switch(a, b, T, s):
    """[1, gin, T]: a before frame s, b from s on."""
    g = a.expand(1, GIN, T).clone()
    g[:, :, s:] = b
    return g


_convs = {}


def converter(tmp_path_factory, precision):
    from openvoice_b200.api import ToneColorConverter
    if precision not in _convs:
        cfg = tmp_path_factory.mktemp("cfg") / "config.json"
        cfg.write_text(json.dumps(O.DEFAULT_HPARAMS))
        conv = ToneColorConverter(str(cfg), device="cuda:0", enable_watermark=False, precision=precision)
        conv.model.load_state_dict(O.synthetic_state_dict(1234))
        _convs[precision] = conv
    return _convs[precision]


@pytest.fixture(params=["fp32", "f16x3"])
def conv(request, tmp_path_factory):
    return converter(tmp_path_factory, request.param)


def waves(lens, seed):
    rng = np.random.default_rng(seed)
    return [(0.5 * (2 * rng.random(n, dtype=np.float32) - 1)).astype(np.float32) for n in lens]


def run(m, spec, lengths, gs, gt, noise, ragged=False):
    o, _, lat = m.voice_conversion(spec.cuda(), lengths.cuda(), gs.cuda(), gt.cuda(), tau=0.3, noise=noise.cuda(),
                                   ragged=ragged)
    torch.cuda.synchronize()
    return o.cpu(), tuple(t.cpu() for t in lat)


# ------------------------------------------------------------------ the expansion kernel
def test_track_kernel_equals_host_rule(native):
    from openvoice_b200.api import ToneTrack
    a, b, c, d = se(1, 4)
    tracks = [
        ToneTrack([(0, a)]),
        ToneTrack([(10, a), (10, b)]),                         # hard switch
        ToneTrack([(5, a), (40, b), (40, c), (41, d)]),        # ramp, switch, one-frame ramp
        ToneTrack([(3, a), (7, b), (90, c)]),
        ToneTrack([(0, a), (1, b), (2, c), (3, d)]),
    ]
    frame0 = [0, 4, 30, 0, 0]
    frames = [60, 20, 33, 61, 2]
    Tmax = 61
    key_frame = np.concatenate([t.frames for t in tracks])
    key_se = torch.cat([t.se for t in tracks])
    key0 = np.cumsum([0] + [len(t.frames) for t in tracks[:-1]])
    nkeys = [len(t.frames) for t in tracks]
    i64 = lambda v: torch.tensor(np.asarray(v, dtype=np.int64), device="cuda")  # noqa: E731
    out = native.native.tone_track_expand(i64(key_frame), key_se.cuda(), i64(key0), i64(nkeys), i64(frame0), i64(frames),
                                          Tmax).cpu()
    for i, t in enumerate(tracks):
        want = torch.zeros(GIN, Tmax)
        want[:, : frames[i]] = t.dense(frames[i], frame0[i])[0]
        assert torch.equal(out[i], want), i
    # descriptors past the key arrays are clamped: key0 to the last key, nkeys to what is left
    out = native.native.tone_track_expand(i64(key_frame), key_se.cuda(), i64([99, -3]), i64([5, 99]), i64([0, 0]),
                                          i64([Tmax, Tmax]), Tmax).cpu()
    assert torch.equal(out[0], key_se[-1].view(GIN, 1).expand(GIN, Tmax))
    assert torch.isfinite(out[1]).all()   # key0 -3 -> 0 and every key from there: reads stay inside the arrays


# ------------------------------------------------------------------ voice_conversion with per-frame embeddings
@pytest.mark.parametrize("mode", ["fp32", "f16x3", "f16"])
@pytest.mark.parametrize("zero_g", [False, True])
def test_constant_per_frame_equals_per_item(mode, zero_g):
    """A per-frame embedding that is the same at every frame converts bit for bit like the per-item call, whichever
    side is per frame (both sides, source only, target only)."""
    from conftest import get_native
    m = get_native(zero_g)
    B, T = 2, 75
    spec, lengths, gs, gt, noise = O.synthetic_inputs(B, T, 5, lengths=[75, 52])
    m.native.set_precision(mode)
    try:
        for ragged in (False, True):
            ref_o, ref_lat = run(m, spec, lengths, gs, gt, noise, ragged)
            for fs, ft in ((True, True), (True, False), (False, True)):
                s = gs.expand(B, GIN, T).contiguous() if fs else gs
                t = gt.expand(B, GIN, T).contiguous() if ft else gt
                o, lat = run(m, spec, lengths, s, t, noise, ragged)
                assert torch.equal(o, ref_o), (mode, ragged, fs, ft)
                for x, y in zip(lat, ref_lat):
                    assert torch.equal(x, y), (mode, ragged, fs, ft)
    finally:
        m.native.set_precision(m.precision)


@pytest.mark.parametrize("zero_g", [False, True])
def test_per_frame_parity_with_oracle(native, zero_g, synthetic_sd):
    """Source morph + target hard switch at B = 1 and on a padded B = 2 batch, against the oracle in float64."""
    from conftest import get_native
    m = get_native(zero_g)
    m.native.set_precision(native.native.precision)
    try:
        _parity_cases(m, zero_g, synthetic_sd)
    finally:
        m.native.set_precision(m.precision)


def _parity_cases(m, zero_g, synthetic_sd):
    for B, T, lens in ((1, 67, [67]), (2, 64, [64, 41])):
        spec, lengths, gs, gt, noise = O.synthetic_inputs(B, T, 7, lengths=lens)
        a2, b2 = se(11, 2)
        g_src = torch.cat([morph(gs[b:b + 1], a2, T) for b in range(B)])
        g_tgt = torch.cat([switch(gt[b:b + 1], b2, T, 30) for b in range(B)])
        with torch.no_grad():
            sd64 = {k: v.double() for k, v in synthetic_sd.items()}
            ro, _, rlat = O.voice_conversion(sd64, spec.double(), lengths, g_src.double(), g_tgt.double(),
                                             noise.double(), 0.3, zero_g)
            co, _, _ = O.voice_conversion(sd64, spec.double(), lengths, gs.double(), gt.double(), noise.double(), 0.3,
                                          zero_g)
        o, lat = run(m, spec, lengths, g_src, g_tgt, noise)
        mask = torch.arange(T * 256).view(1, 1, -1) < (lengths * 256).view(-1, 1, 1)
        assert rel_err(o * mask, ro * mask) <= REL, (B, zero_g)
        for x, y in zip(lat, rlat):
            assert rel_err(x, y) <= REL
        assert float((ro - co).abs().max()) > 0.1 * float(ro.pow(2).mean().sqrt())   # the variation matters


@pytest.mark.parametrize("name", ["vc_frames_b1_t67", "vc_frames_b2_padded", "vc_frames_b1_t67_v2"])
def test_golden_reference_per_frame_vectors(name, native):
    """The real reference's voice_conversion with a source morph and a target hard switch ([B, 256, T] embeddings;
    oracle/make_golden_frames.py)."""
    from conftest import get_native
    d = np.load(os.path.join(GOLD, name + ".npz"))
    c = json.loads(str(d["meta"]))
    m = get_native(c["zero_g"])
    m.native.set_precision(native.native.precision)
    try:
        t = {k: torch.from_numpy(d[k]) for k in ("spec", "lengths", "g_src", "g_tgt", "noise")}
        o, lat = run(m, t["spec"], t["lengths"], t["g_src"], t["g_tgt"], t["noise"])
    finally:
        m.native.set_precision(m.precision)
    assert rel_err(o, d["o_hat"]) <= REL, name
    for x, k in zip(lat, ("z", "z_p", "z_hat")):
        assert rel_err(x, d[k]) <= REL, (name, k)


def test_golden_reference_convert_with_per_frame_embeddings(conv):
    d = np.load(os.path.join(GOLD, "convert_frames.npz"))
    a = conv.convert(d["wav"], torch.from_numpy(d["g_src"]), torch.from_numpy(d["g_tgt"]), tau=0.3,
                     noise=torch.from_numpy(d["noise"]))
    assert a.shape == d["audio"].shape and rel_err(a, d["audio"]) <= REL


def test_per_frame_f16_mode_has_its_own_gate(synthetic_sd):
    from conftest import get_native
    m = get_native(False)
    spec, lengths, gs, gt, noise = O.synthetic_inputs(2, 90, 21, lengths=[90, 57])
    a2, b2 = se(12, 2)
    g_src = torch.cat([morph(gs[b:b + 1], a2, 90) for b in range(2)])
    g_tgt = torch.cat([switch(gt[b:b + 1], b2, 90, 45) for b in range(2)])
    with torch.no_grad():
        ro, _, (_, _, rzh) = O.voice_conversion(synthetic_sd, spec, lengths, g_src, g_tgt, noise, 0.3)
    m.native.set_precision("f16")
    try:
        o, (_, _, zh) = run(m, spec, lengths, g_src, g_tgt, noise)
    finally:
        m.native.set_precision(m.precision)
    err = (o - ro).double()
    snr = 10 * np.log10(float(ro.double().pow(2).mean() / err.pow(2).mean()))
    assert snr >= 30.0
    assert rel_err(zh.numpy(), rzh.numpy()) <= 2e-2


def test_wrong_per_frame_shapes_are_refused(native):
    spec, lengths, gs, gt, noise = O.synthetic_inputs(1, 40, 3)
    for bad in (gs.expand(1, GIN, 39).contiguous(), torch.zeros(1, GIN, 2, 40), torch.zeros(1, GIN + 1)):
        with pytest.raises(ValueError):
            native.native.voice_conversion(spec.cuda(), lengths.cuda(), bad.cuda(), gt.cuda(), noise=noise.cuda())
        with pytest.raises(ValueError):
            native.voice_conversion(spec.cuda(), lengths.cuda(), gs.cuda(), bad.cuda(), noise=noise.cuda())


# ------------------------------------------------------------------ convert paths
def test_switch_is_local(conv):
    """A target hard switch at frame s of a 10 s clip: away from the switch by more than the receptive-field halo the
    audio is the constant-first / constant-second conversion, bit for bit."""
    from openvoice_b200.api import ToneTrack
    hop, H = 256, 128
    w = waves([220500], 3)[0]
    T = len(w) // hop
    s = T // 2
    src, a, b = se(21, 3)
    tr = ToneTrack([(s, a), (s, b)])
    got = conv.convert(w, src, tr, seed=5)
    first = conv.convert(w, src, a, seed=5)
    second = conv.convert(w, src, b, seed=5)
    assert np.array_equal(got[: (s - H) * hop], first[: (s - H) * hop])
    assert np.array_equal(got[(s + H) * hop:], second[(s + H) * hop:])
    assert not np.array_equal(got, first) and not np.array_equal(got, second)
    dense = torch.cat([a.expand(1, GIN, s), b.expand(1, GIN, T - s)], 2)
    assert np.array_equal(conv.convert(w, src, dense, seed=5), got)     # a track means its dense form


def test_convert_long_with_track_equals_convert(conv):
    from openvoice_b200.api import ToneTrack
    w = waves([256 * 700 + 77], 4)[0]
    a, b, c, d = se(31, 4)
    src = ToneTrack([(100, a), (400, b)])
    tgt = ToneTrack([(0, c), (250, c), (250, d), (600, c)])
    ref = conv.convert(w, src, tgt, seed=9)
    for wf in (128, 300):
        assert np.array_equal(conv.convert_long(w, src, tgt, window_frames=wf, seed=9), ref), wf
    T = len(w) // 256
    assert np.array_equal(conv.convert_long(w, src.dense(T), tgt, window_frames=200, seed=9), ref)


def test_mixed_batch_items_equal_their_own_convert(conv):
    from openvoice_b200.api import ToneTrack
    ws = waves([22050, 30000, 40000, 9999], 6)
    e = se(41, 6)
    T2 = len(ws[2]) // 256
    src = [e[0], ToneTrack([(0, e[0]), (50, e[1])]), e[2], e[3]]
    tgt = [e[4], e[5], morph(e[4], e[5], T2), ToneTrack([(20, e[5]), (20, e[4])])]
    seeds = [1, 2, 3, 4]
    got = conv.convert_batch(ws, src, tgt, seeds=seeds)
    for i in range(4):
        assert np.array_equal(got[i], conv.convert(ws[i], src[i], tgt[i], seed=seeds[i])), i
    assert np.array_equal(got[0], conv.convert(ws[0], e[0], e[4], seed=1))   # a per-item item stays per item
    conc = conv.convert_concurrent(ws, src, tgt, seeds=seeds, streams=2)
    for i in range(4):
        assert np.array_equal(conc[i], got[i]), i
    o, n = conv.convert_batch_device(ws, src, tgt, seeds=seeds)
    o = o.cpu().numpy()
    for i in range(4):
        assert np.array_equal(o[i, : n[i]], got[i]), i
    with pytest.raises(ValueError):     # one dense [1, gin, T] for a batch whose items differ in length
        conv.convert_batch(ws, morph(e[0], e[1], T2), e[4])


def test_repeated_per_frame_call_replays_and_follows_contents(native):
    nat = native.native
    B, L = 2, 256 * 64
    wav = torch.from_numpy(np.stack(waves([L, L], 8))).cuda()
    wl = torch.tensor([L, L - 3000], dtype=torch.int64, device="cuda")
    T = L // 256
    g1 = torch.cat([morph(*se(51, 2), T), morph(*se(52, 2), T)]).cuda()
    g2 = torch.cat([switch(*se(53, 2), T, 10), morph(*se(54, 2), T)]).cuda()
    gs = se(55)[0].expand(B, GIN, 1).reshape(B, GIN).contiguous().cuda()
    g, out, fr = g1.clone(), torch.empty(B, L, device="cuda"), torch.empty(B, dtype=torch.int64, device="cuda")
    for _ in range(3):
        nat.convert_waveform(wav, wl, gs, g, seed=3, out=out, frames_out=fr)
    r0 = nat.graph_replays
    g.copy_(g2)
    nat.convert_waveform(wav, wl, gs, g, seed=3, out=out, frames_out=fr)
    assert nat.graph_replays == r0 + 1
    want, _ = nat.convert_waveform(wav, wl, gs, g2.clone(), seed=3)
    torch.cuda.synchronize()
    assert torch.equal(out, want)


# ------------------------------------------------------------------ live streams
@pytest.mark.parametrize("chunks", [[22050], [4000, 9000], [769]])
def test_streaming_retarget_equals_convert_with_track(conv, chunks):
    """Retargets between pushes (a hard target switch, then both sides over a 40-frame ramp): the stream equals
    ``convert`` on the whole clip with the tracks the stream reports, bit for bit."""
    from openvoice_b200.streaming import StreamingConverter
    w = waves([22050 * 6 + 123], 13)[0]
    src, a, b, c = se(61, 4)
    plan = {2: dict(tgt_se=b), 4: dict(src_se=c, tgt_se=a, ramp_frames=40)}
    sc = StreamingConverter(conv, src, a, tau=0.3, window_frames=64, request_seed=17)
    outs, pos, k, at = [], 0, 0, []
    while pos < len(w):
        n = chunks[k % len(chunks)]
        outs.append(sc.push(w[pos: pos + n]))
        pos, k = pos + n, k + 1
        if k in plan:
            at.append(sc.retarget(**plan[k]))
    outs.append(sc.flush())
    assert len(at) == 2 and at[0] <= at[1]
    want = conv.convert(w, sc.tone_track("src"), sc.tone_track("tgt"), seed=17)
    assert np.array_equal(np.concatenate(outs), want)
    assert not np.array_equal(want, conv.convert(w, src, a, seed=17))


@pytest.mark.parametrize("rates", [(48000, None), (None, 48000), (16000, 48000)])
def test_streaming_retarget_at_other_rates(conv, rates):
    from openvoice_b200.streaming import StreamingConverter
    i_sr, o_sr = rates
    n = 22050 * 4 if i_sr is None else i_sr * 4
    w = waves([n + 77], 14)[0]
    src, a, b = se(71, 3)
    sc = StreamingConverter(conv, src, a, window_frames=128, request_seed=5, input_sr=i_sr, output_sr=o_sr)
    outs = []
    for k, pos in enumerate(range(0, len(w), 7000)):
        outs.append(sc.push(w[pos: pos + 7000]))
        if k == 5:
            sc.retarget(tgt_se=b, ramp_frames=16)
    outs.append(sc.flush())
    want = conv.convert(w, src, sc.tone_track("tgt"), seed=5, sr=i_sr)
    if o_sr is not None:
        x = torch.from_numpy(want)[None].cuda()
        want = conv.model.native.resample(x, torch.tensor([x.shape[1]], dtype=torch.int64, device="cuda"), 22050,
                                          o_sr)[0].cpu().numpy()
    assert np.array_equal(np.concatenate(outs), want)


@pytest.mark.parametrize("chunks,rates", [([5000], (None, None)), ([2048, 9000], (None, None)),
                                          ([7000], (48000, None)), ([6000, 2500], (16000, 48000))])
def test_sessions_retarget_equals_streaming_converter(conv, chunks, rates):
    """Two of four sessions retarget mid-stream (a hard target switch; a source ramp): each session equals its own
    retargeted StreamingConverter push by push (at the model's rate and at other input / output rates) and ``convert``
    with its tracks; the untouched sessions of the same steps equal their plain conversions, bit for bit."""
    from openvoice_b200.streaming import StreamingConverter, StreamingSessions
    i_sr, o_sr = rates
    S, n = 4, (i_sr or 22050) * 4
    e = se(81, 7)
    ws = waves([n] * S, 15)
    ss = StreamingSessions(conv, window_frames=64, rates=tuple(r for r in rates if r))
    ids = [ss.open(e[k], e[k + 1], seed=k, input_sr=i_sr, output_sr=o_sr) for k in range(S)]
    refs = [StreamingConverter(conv, e[k], e[k + 1], window_frames=64, request_seed=k, input_sr=i_sr, output_sr=o_sr)
            for k in range(S)]
    got, want = [[] for _ in range(S)], [[] for _ in range(S)]
    plan = {3: (1, dict(tgt_se=e[5])), 6: (2, dict(src_se=e[6], ramp_frames=30))}
    pos, step = 0, 0
    while pos < n:
        chunk = chunks[step % len(chunks)]
        res = ss.push({ids[k]: ws[k][pos: pos + chunk] for k in range(S)})
        for k in range(S):
            got[k].append(res[ids[k]])
            want[k].append(refs[k].push(ws[k][pos: pos + chunk]))
            assert np.array_equal(got[k][-1], want[k][-1]), (step, k)
        if step in plan:
            k, kw = plan[step]
            assert ss.retarget(ids[k], **kw) == refs[k].retarget(**kw)
        pos, step = pos + chunk, step + 1
    res = ss.close(ids)
    for k in range(S):
        got[k].append(res[ids[k]])
        want[k].append(refs[k].flush())
        a = np.concatenate(got[k])
        assert np.array_equal(a, np.concatenate(want[k])), k
        if o_sr is not None:
            continue                       # StreamingConverter(output_sr=) against convert: test_streaming_retarget_at_other_rates
        if k in (1, 2):
            tr = (refs[k].tone_track("src"), refs[k].tone_track("tgt"))
            assert np.array_equal(a, conv.convert(ws[k], *tr, seed=k, sr=i_sr)), k
        else:
            assert np.array_equal(a, conv.convert(ws[k], e[k], e[k + 1], seed=k, sr=i_sr)), k
