"""CPU: the tone-track rule (``ToneTrack.dense``, the host statement the device expansion kernel is held to bit for bit
in tests/test_gpu_tone_track.py) and the shape rules every embedding argument follows."""
import numpy as np
import pytest
import torch

from openvoice_b200 import _native
from openvoice_b200.api import NativeSynthesizer, ToneColorConverter, ToneTrack, is_per_frame_se, pack_tone_keys

GIN = 8


def rule(frames, ses, t):
    """The rule spelt out one frame at a time in fp32 (include/ovc.h: ovc_tone_track_expand)."""
    f32 = np.float32
    if t < frames[0]:
        return ses[0]
    k = max(i for i in range(len(frames)) if frames[i] <= t)
    if k == len(frames) - 1:
        return ses[k]
    u = f32(t - frames[k]) / f32(frames[k + 1] - frames[k])
    return np.array([f32(a) + f32(u) * (f32(b) - f32(a)) for a, b in zip(ses[k], ses[k + 1])], dtype=np.float32)


def keys(frames, seed):
    rng = np.random.default_rng(seed)
    return [(f, rng.standard_normal(GIN).astype(np.float32)) for f in frames]


@pytest.mark.parametrize("frames", [[0], [7], [10, 10], [3, 20], [3, 20, 20, 21, 40], [0, 1, 2, 3], [5, 5, 5, 9]])
def test_dense_follows_the_rule(frames):
    ks = keys(frames, len(frames))
    tr = ToneTrack(ks)
    T = 50
    d = tr.dense(T)[0].numpy()
    assert d.shape == (GIN, T) and d.dtype == np.float32
    for t in range(T):
        assert np.array_equal(d[:, t], rule([f for f, _ in ks], [s for _, s in ks], t)), t
    for f0 in (1, 9, 20, 33):     # a window at frame0 is the whole clip's slice, bit for bit
        assert np.array_equal(tr.dense(T - f0, f0)[0].numpy(), d[:, f0:])


def test_hard_switch_takes_the_later_key():
    a, b, c = (np.full(GIN, v, np.float32) for v in (1.0, 2.0, 3.0))
    d = ToneTrack([(4, a), (4, b), (4, c)]).dense(8)[0].numpy()
    assert (d[:, :4] == 1).all() and (d[:, 4:] == 3).all()


def test_ramp_endpoints_are_exact():
    a, b = (np.random.default_rng(s).standard_normal(GIN).astype(np.float32) for s in (1, 2))
    d = ToneTrack([(10, a), (17, b)]).dense(30)[0].numpy()
    assert np.array_equal(d[:, 10], a) and np.array_equal(d[:, 17], b) and np.array_equal(d[:, 29], b)
    assert np.array_equal(d[:, 0], a)


@pytest.mark.parametrize("bad", [[], [(3, np.zeros(GIN)), (2, np.zeros(GIN))], [(-1, np.zeros(GIN))],
                                 [(1.5, np.zeros(GIN))], [(0, np.zeros(GIN)), (1, np.zeros(GIN + 1))]])
def test_track_refusals(bad):
    with pytest.raises(ValueError):
        ToneTrack(bad)


def test_se_arg_shapes():
    B, T, G = 2, 30, GIN
    g, pf = _native.se_arg(torch.zeros(B, G, 1), B, G, T, "g")
    assert not pf and tuple(g.shape) == (B, G)
    g, pf = _native.se_arg(torch.zeros(B, G), B, G, T, "g")
    assert not pf and tuple(g.shape) == (B, G)
    g, pf = _native.se_arg(torch.zeros(B, G, T), B, G, T, "g")
    assert pf and tuple(g.shape) == (B, G, T)
    g, pf = _native.se_arg(torch.zeros(B, 1, G), B, G, T, "g")          # row vectors stay per item
    assert not pf and tuple(g.shape) == (B, G)
    for bad in (torch.zeros(B, G, T - 1), torch.zeros(B, G, T + 1), torch.zeros(1, G, T), torch.zeros(B, G + 1),
                torch.zeros(B * G * T), torch.zeros(B, T, G), torch.zeros(1, G, B)):   # [1, gin, B]: B * gin values
        with pytest.raises(ValueError):
            _native.se_arg(bad, B, G, T, "g")


class _Native:
    class hp:
        gin_channels = GIN


def test_synthesizer_expand_se_shapes():
    m = NativeSynthesizer.__new__(NativeSynthesizer)
    m.device, m.native = "cpu", _Native
    assert tuple(m._expand_se(torch.zeros(1, GIN, 1), 3).shape) == (3, GIN)
    assert tuple(m._expand_se(torch.zeros(1, 1, GIN), 3, 20).shape) == (3, GIN)     # a row vector: one embedding
    assert tuple(m._expand_se(torch.zeros(1, GIN, 20), 3, 20).shape) == (3, GIN, 20)
    assert tuple(m._expand_se(torch.zeros(3, GIN, 20), 3, 20).shape) == (3, GIN, 20)
    with pytest.raises(ValueError):
        m._expand_se(torch.zeros(1, GIN, 19), 3, 20)
    with pytest.raises(ValueError):
        m._expand_se(torch.zeros(2, GIN, 20), 3, 20)


class _Hps:
    class model:
        gin_channels = GIN


def _converter():
    c = ToneColorConverter.__new__(ToneColorConverter)
    c.hps, c.device = _Hps, "cpu"
    return c


def test_converter_embedding_forms():
    c = _converter()
    a = torch.zeros(1, GIN, 1)
    assert torch.is_tensor(c._se_items(a, 3, "src_se"))            # per item: today's stacked tensor
    assert torch.is_tensor(c._se_items([a, a, a], 3, "src_se"))
    tr = ToneTrack([(0, np.zeros(GIN)), (5, np.ones(GIN))])
    items = c._se_items([a, tr, torch.zeros(1, GIN, 12)], 3, "src_se")
    assert items[0].shape == (GIN,) and items[1] is tr and items[2].shape == (GIN, 12)
    assert len(c._se_items(tr, 2, "tgt_se")) == 2
    for bad in ([a, tr], [torch.zeros(1, GIN + 1, 1), tr, tr], [torch.zeros(2, GIN, 12), tr, tr],
                [ToneTrack([(0, np.zeros(GIN + 1))]), tr, tr]):
        with pytest.raises(ValueError):
            c._se_items(bad, 3, "src_se")
    with pytest.raises(ValueError):        # a dense embedding must cover the item's frames exactly
        pack_tone_keys([torch.zeros(GIN, 12)], [0], [13])


def test_per_item_only_paths_refuse_per_frame():
    from openvoice_b200 import distributed
    c = _converter()
    tr = ToneTrack([(0, np.zeros(GIN))])
    for se in (tr, torch.zeros(1, GIN, 5), [torch.zeros(1, GIN, 1), tr]):
        assert is_per_frame_se(se)
        with pytest.raises(ValueError):     # StreamingConverter and the other per-item paths stack through this
            c._stack_se(se, 2)
        with pytest.raises(ValueError):
            distributed.convert_sharded(lambda *a, **k: [], [np.zeros(1000, np.float32)], se, torch.zeros(1, GIN, 1))
    assert not is_per_frame_se(torch.zeros(1, GIN, 1)) and not is_per_frame_se([torch.zeros(1, GIN)])
    row = torch.zeros(1, 1, GIN)                       # [1, 1, gin] is one embedding, as it always was
    assert not is_per_frame_se(row) and not is_per_frame_se(row, GIN)
    assert torch.equal(c._stack_se(row, 2), torch.zeros(2, GIN))
    assert torch.is_tensor(c._se_items([row, row], 2, "src_se"))


def test_clone_paths_refuse_per_frame_embeddings():
    c = _converter()
    tr = ToneTrack([(0, np.zeros(GIN))])
    ok = torch.zeros(1, GIN, 1)
    assert c._clone_keys(dict(src_se=ok, tgt_se=ok), "request 0")["src_se"].shape == (1, GIN)
    for bad in (tr, torch.zeros(1, GIN, 7)):
        for name in ("src_se", "tgt_se"):
            q = dict(src_se=ok, tgt_se=ok)
            q[name] = bad
            with pytest.raises(ValueError):    # clone_batch, clone_stream_batch and CloneSessions.open validate here
                c._clone_keys(q, "request 0")


def test_sessions_refuse_tracks():
    from openvoice_b200.streaming import StreamingSessions
    with pytest.raises(ValueError):
        StreamingSessions._per_item_se("tgt_se", ToneTrack([(0, np.zeros(GIN))]))


@pytest.mark.parametrize("windows", [1, 8, 32])
def test_packed_keys_do_not_grow_with_the_clip_or_the_windows(windows):
    """convert_long packs one chunk of windows of a long clip: a dense per-frame embedding gives the windows' own
    frames, a track only the keys around each window, and items that read the same keys share them."""
    T, W = 300_000, 256
    dense = torch.zeros(GIN, T)
    f0 = [100_000 + W * i for i in range(windows)]
    kf, ks, k0, nk = pack_tone_keys([dense] * windows, f0, [W] * windows, clip=T)
    assert len(kf) == windows * W and ks.shape == (windows * W, GIN)
    tr = ToneTrack([(f, np.full(GIN, f, np.float32)) for f in range(0, T, 1000)])
    kf, ks, k0, nk = pack_tone_keys([tr] * windows, f0, [W] * windows)
    assert len(kf) <= 3 * windows and max(nk) <= 3
    kf, ks, k0, nk = pack_tone_keys([tr] * windows, [f0[0]] * windows, [W] * windows)
    assert len(kf) <= 3 and k0 == [k0[0]] * windows                     # the same window: one shared key set
    # the packed keys give the track's values at the windows' frames
    keys = ToneTrack(list(zip(kf.tolist(), ks)))
    assert np.array_equal(keys.dense(W, f0[0])[0].numpy(), tr.dense(W, f0[0])[0].numpy())


@pytest.mark.parametrize("f", [0, 1, 6, 12, 13, 25, 40, 80])
@pytest.mark.parametrize("ramp", [0, 1, 9])
def test_retarget_track_keeps_the_past_and_reaches_the_new_embedding(f, ramp):
    from openvoice_b200.streaming import retarget_track
    old = ToneTrack(keys([2, 12, 30, 30, 45], 3))
    new = np.random.default_rng(9).standard_normal(GIN).astype(np.float32)
    tr = retarget_track(old, f, new, ramp)
    T = f + ramp + 20
    d_old, d_new = old.dense(T)[0].numpy(), tr.dense(T)[0].numpy()
    assert np.array_equal(d_new[:, :f], d_old[:, :f])                    # frames windows may already have read
    assert (d_new[:, f + ramp:] == new[:, None]).all()
    if ramp:
        assert np.array_equal(d_new[:, f], d_old[:, f])                  # the ramp starts from the old value at f
    assert len(tr.frames) <= len(old.frames) + 30                         # pinned frames: only inside an old ramp
    tr2 = retarget_track(tr, f + ramp + 5, d_old[:, 0], 0)                # a second retarget keeps the first one's frames
    assert np.array_equal(tr2.dense(f + ramp + 5)[0].numpy(), tr.dense(f + ramp + 5)[0].numpy())


def test_retarget_track_refusals():
    from openvoice_b200.streaming import retarget_track
    old = ToneTrack(keys([0], 1))
    for f, ramp in ((-1, 0), (3, -2)):
        with pytest.raises(ValueError):
            retarget_track(old, f, np.zeros(GIN), ramp)
