"""-m gpu: time-varying speaking style for the base-speaker TTS (include/ovc.h: ovc_tts_encode_g,
ovc_tts_encode_state_tokens, ovc_tts_decode_windows_tokens).  A speaker is a style id, one vector (a blend of emb_g rows)
or per-token vectors (a ToneTrack over token positions or a [1, gin, N] tensor).  Every comparison is bit for bit
unless it names a bound."""
import copy
import json

import numpy as np
import pytest
import torch

from oracle import tts_oracle as T
from oracle import vc_oracle as O

pytestmark = pytest.mark.gpu

HOP = 256


def rms(a):
    return float(np.sqrt((np.asarray(a, dtype=np.float64) ** 2).mean()))


_engines = {}


def engine(tmp_path_factory, precision):
    from openvoice_b200.api import BaseSpeakerTTS, ToneColorConverter
    if precision not in _engines:
        d = tmp_path_factory.mktemp("style")
        hp = copy.deepcopy(O.DEFAULT_HPARAMS)
        hp["data"]["n_speakers"] = T.TTS_HPARAMS["n_speakers"]
        hp["speakers"] = {"default": 1, "whispering": 2}
        (d / "tts.json").write_text(json.dumps(hp))
        torch.save({"model": T.synthetic_tts_state_dict()}, d / "tts.pth")
        tts = BaseSpeakerTTS(str(d / "tts.json"), device="cuda:0", precision=precision)
        tts.load_ckpt(str(d / "tts.pth"))
        (d / "vc.json").write_text(json.dumps(O.DEFAULT_HPARAMS))
        conv = ToneColorConverter(str(d / "vc.json"), device="cuda:0", enable_watermark=False, precision=precision)
        conv.model.load_state_dict(O.synthetic_state_dict(1234))
        _engines[precision] = (tts, conv)
    return _engines[precision]


@pytest.fixture(params=["fp32", "f16x3"])
def pair(request, tmp_path_factory):
    return engine(tmp_path_factory, request.param)


def sentences(k, seed, lo=20, hi=70):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, T.TTS_HPARAMS["n_vocab"], int(rng.integers(lo, hi))).tolist() for _ in range(k)]


def ramp_track(tts, n_tokens):
    """default -> whispering ramp over the first half of the tokens, then a hard switch to style 0."""
    from openvoice_b200.api import ToneTrack
    a, b, c = tts.style("default"), tts.style("whispering"), tts.style(0)
    h = n_tokens // 2
    return ToneTrack([(3, a), (h, b), (h + 7, b), (h + 7, c)])


def se(seed):
    return 0.1 * torch.randn(1, 256, 1, generator=torch.Generator().manual_seed(seed))


# ------------------------------------------------------------------------------------------------ identity
def test_identity_forms_equal_the_style_id(pair):
    """speaker=style(k), a one-key track at style(k) and a constant per-token tensor all give speaker=k's audio."""
    from openvoice_b200.api import ToneTrack
    tts, _ = pair
    ids = sentences(3, 1)
    n = sum(len(q) for q in ids)
    v = tts.style("whispering")
    forms = [v, v[None, :, None], ToneTrack([(0, v)]), v[None, :, None].expand(1, -1, n).contiguous()]
    ref = tts.tts_batch([dict(ids=ids, speaker="whispering", seed=3, speed=0.9)])[0]
    ref_ids = tts.tts_from_ids(ids, "whispering", seed=3)
    for i, spk in enumerate(forms):
        got = tts.tts_batch([dict(ids=ids, speaker=spk, seed=3, speed=0.9)])[0]
        assert got.shape == ref.shape and np.array_equal(got, ref), i
        for a, b in zip(tts.tts_from_ids(ids, spk, seed=3), ref_ids):
            assert np.array_equal(a, b), i


def test_identity_in_streaming_and_clone(pair):
    from openvoice_b200.api import ToneTrack
    tts, conv = pair
    ids = sentences(2, 2)
    v = tts.style("default")
    q = dict(ids=ids, seed=11, src_se=se(1), tgt_se=se(2), tau=0.3, convert_seed=5)
    ref_stream = [c for _, c in tts.tts_stream_batch([dict(q, speaker="default")], window_frames=64, first_window_frames=16)]
    ref_clone = conv.clone_batch(tts, [dict(q, speaker="default")])[0]
    for spk in (v, ToneTrack([(0, v)])):
        got = [c for _, c in tts.tts_stream_batch([dict(q, speaker=spk)], window_frames=64, first_window_frames=16)]
        assert len(got) == len(ref_stream) and all(np.array_equal(a, b) for a, b in zip(got, ref_stream))
        assert np.array_equal(conv.clone_batch(tts, [dict(q, speaker=spk)])[0], ref_clone)


# ------------------------------------------------------------------------------------------------ batching
def test_mixed_ragged_batch_equals_solo_calls(pair):
    tts, _ = pair
    reqs = []
    for r in range(5):
        ids = sentences(1 + r % 3, 10 + r)
        n = sum(len(q) for q in ids)
        spk = ["default", 0.7 * tts.style("default") + 0.3 * tts.style(0), ramp_track(tts, n),
               torch.linspace(0, 1, n)[None, None, :] * tts.style("whispering")[None, :, None], 2][r]
        reqs.append(dict(ids=ids, speaker=spk, seed=40 + r, speed=[1.0, 0.8, 1.2, 1.0, 0.9][r]))
    together = tts.tts_batch(reqs)
    for r, q in enumerate(reqs):
        assert np.array_equal(together[r], tts.tts_batch([q])[0]), r


def test_track_changes_the_durations_and_the_audio(pair):
    tts, _ = pair
    ids = sentences(2, 5)
    n = sum(len(q) for q in ids)
    a = tts.tts_batch([dict(ids=ids, speaker="default", seed=1)])[0]
    b = tts.tts_batch([dict(ids=ids, speaker=ramp_track(tts, n), seed=1)])[0]
    assert a.shape != b.shape or not np.array_equal(a, b)


# ------------------------------------------------------------------------------------------------ streaming
def test_stream_with_a_track_follows_tts_batch(pair):
    tts, _ = pair
    reqs = [dict(ids=sentences(2, 20 + r), seed=60 + r, speed=1.0 + 0.1 * r) for r in range(3)]
    for r, q in enumerate(reqs):
        q["speaker"] = ramp_track(tts, sum(len(s) for s in q["ids"])) if r != 1 else "whispering"
    whole = tts.tts_batch(reqs)
    chunks = [[] for _ in reqs]
    for r, c in tts.tts_stream_batch(reqs, window_frames=48, first_window_frames=16):
        chunks[r].append(c)
    for r in range(len(reqs)):
        got = np.concatenate(chunks[r])
        assert got.shape == whole[r].shape
        assert np.abs(got - whole[r]).max() <= 2e-6 * rms(whole[r]), r


def test_whole_row_window_is_bit_identical(pair):
    tts, _ = pair
    m = tts.model
    ids = sentences(2, 7)
    x, lens = tts._pad_ids(ids)
    n = int(lens.sum())
    g = torch.zeros(2, 256, x.shape[1])
    tr = ramp_track(tts, n)
    g[0, :, :len(ids[0])] = tr.dense(len(ids[0]), 0)[0]
    g[1, :, :len(ids[1])] = tr.dense(len(ids[1]), len(ids[0]))[0]
    kw = dict(seeds=[4, 4], streams=[0, 1], noise_scale=0.667, noise_scale_w=0.6, length_scale=1.0, sdp_ratio=0.2)
    state = m.tts_encode(x, lens, g=g, **kw)
    assert state.g.shape == (2, 256, x.shape[1])
    o, frames = m.infer_ragged(x, lens, g=g, **kw)
    o = o.cpu().numpy()
    for b in range(2):
        w, _ = m.tts_decode_windows(state, [(b, 0, frames[b])])
        assert np.array_equal(w[0, : HOP * frames[b]].cpu().numpy(), o[b, : HOP * frames[b]]), b


def test_per_token_state_is_refused_where_rows_hold_one_vector(pair):
    from openvoice_b200._native import OvcError
    tts, conv = pair
    m = tts.model
    x, lens = tts._pad_ids(sentences(2, 8))
    g = torch.randn(2, 256, x.shape[1]) * 0.1
    m.tts_encode(x, lens, g=g, seed=1)
    with pytest.raises(OvcError):
        m.native.tts_encode_state(2, x.shape[1], m.device)          # OVC_ERR_STATE: never one silent vector
    N, Tp, dev = 4, x.shape[1] + 8, m.device
    pool = (torch.zeros(N, Tp, 2 * m.native.hp.inter_channels, device=dev), torch.zeros(N, Tp, dtype=torch.int32, device=dev),
            torch.zeros(N, 256, device=dev), torch.zeros(N, dtype=torch.int64, device=dev))
    with pytest.raises(OvcError):
        m.native.tts_state_rows([0, 1], *pool)                       # a per-row pool cannot take per-token rows


# ------------------------------------------------------------------------------------------------ clone
def test_clone_batch_with_a_track_equals_tts_then_convert(pair):
    tts, conv = pair
    reqs = []
    for r in range(3):
        ids = sentences(1 + r, 30 + r)
        spk = ramp_track(tts, sum(len(q) for q in ids)) if r != 2 else 0.5 * (tts.style(0) + tts.style("default"))
        reqs.append(dict(ids=ids, speaker=spk, seed=70 + r, src_se=se(3 * r), tgt_se=se(3 * r + 1), tau=0.3,
                         convert_seed=9 + r))
    got = conv.clone_batch(tts, reqs)
    for r, q in enumerate(reqs):
        ref = conv.convert(tts.tts_batch([q])[0], q["src_se"], q["tgt_se"], tau=q["tau"], seed=q["convert_seed"])
        assert got[r].shape == ref.shape and np.array_equal(got[r], ref), r


# ------------------------------------------------------------------------------------------------ sessions
def test_clone_stream_batch_with_tracks_follows_clone_batch(pair):
    tts, conv = pair
    reqs = []
    for r in range(3):
        ids = sentences(2, 80 + r)
        spk = [ramp_track(tts, sum(len(q) for q in ids)), 0.6 * tts.style(0) + 0.4 * tts.style(2), "default"][r]
        reqs.append(dict(ids=ids, speaker=spk, seed=90 + r, src_se=se(5 * r), tgt_se=se(5 * r + 1), tau=0.3,
                         convert_seed=3 + r))
    whole = conv.clone_batch(tts, reqs)
    chunks = [[] for _ in reqs]
    for r, c in conv.clone_stream_batch(tts, reqs, window_frames=64, first_window_frames=16):
        chunks[r].append(c)
    for r in range(len(reqs)):
        got = np.concatenate(chunks[r])
        assert got.shape == whole[r].shape
        assert np.abs(got - whole[r]).max() <= 1e-4 * rms(whole[r]), r


def test_session_whose_track_switches_at_a_later_say_equals_clone_batch(pair):
    """The track's switch falls in the second say: the session, stepped between says and beside an id session, gives
    its clone_stream_batch chunks, and those follow clone_batch on the whole text."""
    from openvoice_b200.streaming import CloneSessions
    tts, conv = pair
    first, second = sentences(1, 100), sentences(2, 101)
    n1, n = len(first[0]), len(first[0]) + sum(len(q) for q in second)
    from openvoice_b200.api import ToneTrack
    tr = ToneTrack([(0, tts.style("default")), (n1 + 5, tts.style("default")), (n1 + 5, tts.style("whispering"))])
    keys = dict(speaker=tr, src_se=se(20), tgt_se=se(21), tau=0.3, seed=7, convert_seed=8)
    other = dict(speaker=2, src_se=se(22), tgt_se=se(23), tau=0.3, seed=9, convert_seed=10)
    ref = [c for _, c in conv.clone_stream_batch(tts, [dict(keys, ids=first + second)], window_frames=64,
                                                 first_window_frames=16)]
    whole = conv.clone_batch(tts, [dict(keys, ids=first + second)])[0]
    cs = CloneSessions(conv, tts, window_frames=64, first_window_frames=16)
    a, b = cs.open(**keys), cs.open(**other)
    cs.say(a, ids=first)
    cs.say(b, ids=sentences(2, 102))
    cs.end(b)
    got = []
    got += [o[a] for o in [cs.step()] if a in o]
    cs.say(a, ids=second)
    cs.end(a)
    while a in cs.sessions:
        o = cs.step()
        if a in o:
            got.append(o[a])
    assert np.array_equal(np.concatenate(got), np.concatenate(ref))
    assert np.abs(np.concatenate(got) - whole).max() <= 1e-4 * rms(whole)


# ------------------------------------------------------------------------------------------------ parity
STYLE_CASES = ["tts_style_b1_t60", "tts_style_b2_padded", "tts_style_b1_blend"]


@pytest.mark.parametrize("precision", ["fp32", "f16x3"])
@pytest.mark.parametrize("name", STYLE_CASES)
def test_infer_with_style_matches_the_reference_fixtures(name, precision):
    """Fixtures of the reference's own modules with per-token g (oracle/make_golden_tts_style.py): a ramp and a hard
    switch, a padded batch of a track row and a sid row, a per-row blend."""
    from conftest import get_native_tts
    from test_tts_style_host import style_fixture
    m = get_native_tts()
    d, (tokens, lengths, noise_w, noise), g, kw = style_fixture(name)
    g_in = g[:, :, 0] if g.shape[-1] == 1 else g
    m.native.set_precision(precision)
    try:
        o, attn, y_mask, (z, z_p, _, _) = m.infer(tokens, lengths, g=g_in, noise_w=noise_w, noise=noise, **kw)
        _, _, logw = m.native.tts_encode(tokens.cuda(), lengths.cuda(), None, noise_w=noise_w.cuda(), g=g_in.cuda(),
                                         **{k: kw[k] for k in ("noise_scale_w", "length_scale", "sdp_ratio")})
        torch.cuda.synchronize()
    finally:
        m.native.set_precision(m.precision)
    ref_logw = (d["logw_sdp"] * kw["sdp_ratio"] + d["logw_dp"] * (1 - kw["sdp_ratio"]))[:, 0]
    assert np.abs(logw.cpu().numpy() - ref_logw).max() < 1e-4
    assert np.array_equal(attn[:, 0].sum(1).cpu().numpy(), d["w_ceil"])
    assert np.array_equal(y_mask[:, 0].sum(1).long().cpu().numpy(), d["y_lengths"])
    ym = y_mask.cpu().numpy()
    e = dict(z_p=np.abs(z_p.cpu().numpy() - d["z_p"] * ym).max() / rms(d["z_p"]),
             z=np.abs(z.cpu().numpy() * ym - d["z"] * ym).max() / rms(d["z"]),
             o=np.abs(o.cpu().numpy() - d["o"]).max() / rms(d["o"]))
    print(name, precision, e)
    assert all(v < 1e-4 for v in e.values()), e


def test_sid_row_as_vectors_equals_the_sid_call():
    from conftest import get_native_tts
    m = get_native_tts()
    tokens, lengths, _, noise_w = T.synthetic_tts_inputs(1, 31, 2)
    noise = torch.randn(1, 192, 2000, generator=torch.Generator().manual_seed(5))
    g = m._state_dict["emb_g.weight"].float()[2][None, :, None].expand(1, -1, 31).contiguous()
    kw = dict(noise_scale=0.667, length_scale=1.0, noise_scale_w=0.6, sdp_ratio=0.2, noise_w=noise_w, noise=noise,
              latents=False)
    o_sid = m.infer(tokens, lengths, sid=torch.tensor([2]), **kw)[0]
    o_g = m.infer(tokens, lengths, g=g, **kw)[0]
    assert np.array_equal(o_sid.cpu().numpy(), o_g.cpu().numpy())
