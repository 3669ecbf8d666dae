"""Host-side rules of time-varying speaking style (no GPU): speaker forms, their refusals before any launch, and the
token positions o_j at which a per-token speaker is read for each sentence of a request."""
import copy
import json
import os
import sys
import types

import numpy as np

import pytest
import torch

from oracle import tts_oracle as T
from oracle import vc_oracle as O

ORACLE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
STYLE_CASES = ["tts_style_b1_t60", "tts_style_b2_padded", "tts_style_b1_blend"]

GIN = 256


def _engine():
    from openvoice_b200.api import BaseSpeakerTTS
    from openvoice_b200.utils import HParams
    hp = copy.deepcopy(O.DEFAULT_HPARAMS)
    hp["data"]["n_speakers"] = T.TTS_HPARAMS["n_speakers"]
    hp["speakers"] = {"default": 1, "whispering": 2}
    eng = BaseSpeakerTTS.__new__(BaseSpeakerTTS)
    eng.hps = HParams(**hp)
    eng.device = "cuda:0"
    eng.text_frontend = lambda text, mark: [[ord(c) % 50 for c in w] for w in text.split(".") if w]
    emb = torch.randn(T.TTS_HPARAMS["n_speakers"], GIN, generator=torch.Generator().manual_seed(3))
    eng.model = types.SimpleNamespace(_state_dict={"emb_g.weight": emb})   # no infer: a launch would fail loudly
    return eng


def _track(eng):
    from openvoice_b200.api import ToneTrack
    return ToneTrack([(2, eng.style(0)), (9, eng.style("whispering")), (15, eng.style("whispering")),
                      (15, eng.style("default"))])


def test_style_and_tokenize():
    eng = _engine()
    emb = eng.model._state_dict["emb_g.weight"]
    assert torch.equal(eng.style("whispering"), emb[2]) and torch.equal(eng.style(0), emb[0])
    for bad in ("shouting", T.TTS_HPARAMS["n_speakers"], -1):
        with pytest.raises(ValueError, match="style"):
            eng.style(bad)
    assert eng.tokenize("ab.cde") == [[ord("a") % 50, ord("b") % 50], [ord(c) % 50 for c in "cde"]]


def test_malformed_speakers_are_refused_before_any_launch():
    from openvoice_b200.api import ToneTrack
    eng = _engine()
    ids = [[1, 2, 3], [4, 5]]
    ok = dict(ids=ids, speaker="default", seed=1)
    bad = [torch.zeros(GIN - 1), torch.zeros(1, GIN + 1, 1), torch.zeros(1, GIN, 4), torch.zeros(1, GIN, 6), "shouting",
           ToneTrack([(0, torch.zeros(GIN - 1))]), torch.zeros(2, GIN, 5)]
    for spk in bad:
        for call in (lambda q: eng.tts_batch(q), lambda q: eng.tts_stream_batch(q)):
            with pytest.raises(ValueError, match="request 1"):
                call([ok, dict(ok, speaker=spk)])
        with pytest.raises(ValueError, match="speaker"):
            eng.tts_from_ids(ids, spk, seed=1)


def test_sentences_read_the_track_at_their_token_offsets():
    eng = _engine()
    tr = _track(eng)
    ids = [[1] * 6, [2] * 4, [3] * 9]
    per_token = torch.randn(1, GIN, 19, generator=torch.Generator().manual_seed(5))
    reqs = [dict(ids=ids, speaker=tr, seed=1), dict(ids=[[4] * 3], speaker="whispering", seed=2),
            dict(ids=ids, speaker=per_token, seed=3), dict(ids=[[5] * 2], speaker=0.5 * eng.style(0), seed=4)]
    seqs, sid, owner, _, kw = eng._request_sentences(reqs)
    g = kw["g"]
    assert g.shape == (len(seqs), GIN, 9) and owner == [0, 0, 0, 1, 2, 2, 2, 3]
    offs = [0, 6, 10]
    for j in range(3):
        n = len(ids[j])
        assert torch.equal(g[j, :, :n], tr.dense(n, offs[j])[0])
        assert torch.equal(g[4 + j, :, :n], per_token[0, :, offs[j]:offs[j] + n])
        assert not g[j, :, n:].any()
    assert torch.equal(g[3, :, :3], eng.style("whispering")[:, None].expand(-1, 3))
    assert torch.equal(g[7, :, :2], (0.5 * eng.style(0))[:, None].expand(-1, 2))
    # one vector per request: [n, gin]; ids only: no g (the emb_g path)
    _, _, _, _, kw = eng._request_sentences([reqs[1], reqs[3]])
    assert kw["g"].shape == (2, GIN) and torch.equal(kw["g"][0], eng.style(2))
    _, sid, _, _, kw = eng._request_sentences([reqs[1]])
    assert "g" not in kw and sid == [2]


def test_tts_from_ids_places_the_track_over_the_whole_call():
    eng = _engine()
    tr = _track(eng)
    seen = {}

    def infer_sentences(seqs, sid, **kw):
        seen.update(kw)
        return []
    eng._infer_sentences = infer_sentences
    eng.tts_from_ids([[1] * 7, [2] * 5], tr, seed=1)
    assert torch.equal(seen["g"][1, :, :5], tr.dense(5, 7)[0])


def test_sessions_key_tracks_by_tokens_across_say_calls():
    """A session's sentence j reads its track at o_j, counted over every sentence said to it, whatever the steps."""
    from test_clone_sessions_host import keys, make_models
    from openvoice_b200.streaming import CloneSessions
    tts, conv = make_models()
    emb = torch.randn(3, GIN, generator=torch.Generator().manual_seed(9))
    tts.model._state_dict = {"emb_g.weight": emb}
    seen = []
    encode = tts.model.tts_encode

    def tts_encode(x, lens, **kw):
        seen.append((x.clone(), kw.pop("g", None)))
        return encode(x, lens, **kw)
    tts.model.tts_encode = tts_encode
    from openvoice_b200.api import ToneTrack
    tr = ToneTrack([(0, emb[0]), (8, emb[1]), (12, emb[1]), (12, emb[2])])
    cs = CloneSessions(conv, tts, window_frames=64)
    a = cs.open(**dict(keys(0), speaker=tr))
    b = cs.open(**dict(keys(1), speaker="default"))
    cs.say(a, ids=[[1] * 5, [2] * 4])
    cs.say(b, ids=[[3] * 6])
    cs.encode_pending()
    cs.say(a, ids=[[4] * 7])
    cs.encode_pending()
    (x1, g1), (x2, g2) = seen
    assert torch.equal(g1[0, :, :5], tr.dense(5, 0)[0]) and torch.equal(g1[1, :, :4], tr.dense(4, 5)[0])
    assert torch.equal(g1[2, :, :6], emb[1][:, None].expand(-1, 6))          # the id row rides as its emb_g row
    assert torch.equal(g2[0, :, :7], tr.dense(7, 9)[0])                        # the second say starts at token 9
    per_token = torch.zeros(1, GIN, 10)
    c = cs.open(**dict(keys(2), speaker=per_token))
    cs.say(c, ids=[[1] * 6])
    with pytest.raises(ValueError, match=f"session {c}: its per-token speaker tensor has 10 columns"):
        cs.say(c, ids=[[1] * 5])


def style_fixture(name):
    """(fixture arrays, inputs (tokens, lengths, noise_w, noise), g) of a reference-generated style case."""
    if ORACLE not in sys.path:
        sys.path.insert(0, ORACLE)
    import make_golden_tts_style as M
    d = np.load(os.path.join(GOLDEN, name + ".npz"))
    c = json.loads(str(d["meta"]))
    return d, M.inputs(c), torch.from_numpy(d["g"]), {k: c[k] for k in M.KW}


@pytest.mark.parametrize("name", STYLE_CASES)
def test_style_oracle_matches_the_reference_fixtures(name):
    if ORACLE not in sys.path:
        sys.path.insert(0, ORACLE)
    import tts_style_oracle as S
    d, (tokens, lengths, noise_w, noise), g, kw = style_fixture(name)
    with torch.no_grad():
        r = S.tts_infer_g(T.synthetic_tts_state_dict(), tokens, lengths, g, noise_w, noise, **kw)
    assert np.abs(r["logw_sdp"].numpy() - d["logw_sdp"]).max() < 1e-4
    assert np.abs(r["logw_dp"].numpy() - d["logw_dp"]).max() < 1e-4
    assert np.array_equal(r["w_ceil"].numpy(), d["w_ceil"]) and np.array_equal(r["y_lengths"].numpy(), d["y_lengths"])
    for k in ("z_p", "z", "o"):
        ref = d[k]
        assert np.abs(r[k].numpy() - ref).max() < 1e-4 * np.sqrt((ref.astype(np.float64) ** 2).mean()), k
