"""Host logic of CloneSessions on the CPU, with stand-in TTS and converter models: sentence numbering across ``say``
calls, the first-window rule, when a session closes, pool and converter rows being freed and reused, the calls a step
makes, and the refusals.  Each session's chunks must equal StreamingSessions fed its whole utterance at once."""
import copy
import types

import numpy as np
import pytest
import torch

from test_multistream_host import HOP, SR, FakeConverter, FakeModel

GIN, INTER = FakeConverter.hps.model.gin_channels, FakeConverter.hps.model.inter_channels


def sentence_audio(seed, stream, toks, t):
    """The stand-in decode: sample t of a sentence, a function of its key, stream and tokens only."""
    return (0.5 * np.sin(0.003 * t * (1 + stream) + seed % 97 + sum(toks) % 13)).astype(np.float32)


def n_frames(toks):
    return 3 * len(toks) + 2


class FakeTtsNative:
    hp = types.SimpleNamespace(inter_channels=INTER, gin_channels=GIN)

    def __init__(self, calls):
        self.calls = calls

    def tts_info(self):
        return {"has_tts": 1, "n_vocab": 50, "n_speakers": 3}

    def tts_state_rows(self, dst_row, stats, cum, g, y_lengths, src=None):
        """The library's copy and padding rule (include/ovc.h: ovc_tts_state_rows) on the host."""
        self.calls.append("tts_state_rows" if src is None else "repitch")
        s_stats, s_cum, s_g, s_len = src
        T = s_cum.shape[1]
        for b, r in enumerate(dst_row):
            stats[r].zero_()
            stats[r, :T] = s_stats[b]
            cum[r, :T] = s_cum[b]
            cum[r, T:] = s_cum[b, T - 1]
            g[r], y_lengths[r] = s_g[b], s_len[b]


class FakeTtsModel:
    device = torch.device("cpu")
    from openvoice_b200.api import NativeSynthesizer
    check_tts_input = NativeSynthesizer.check_tts_input  # the real checks, on the stand-in's tts_info
    del NativeSynthesizer

    def __init__(self):
        self.calls = []
        self.native = FakeTtsNative(self.calls)
        self.rows = {}                                   # pool row -> (seed, stream, tokens)
        self.encoded = []                                # (seed, stream) of every sentence encoded
        self.windows = []

    def tts_encode(self, x, lens, sid=None, pool=None, rows=None, seeds=None, streams=None, noise_scale=None, **kw):
        self.calls.append("tts_encode")
        self.check_tts_input(x, sid)                     # raises before anything is written, as the real encode does
        pool.fit(max(rows) + 1, x.shape[1])
        for b, r in enumerate(rows):                     # token sums in the pool, to see re-pitching keep them
            toks = tuple(int(v) for v in x[b, : int(lens[b])])
            self.rows[r] = (seeds[b], streams[b], toks)
            self.encoded.append((seeds[b], streams[b]))
            pool.stats[r].zero_()
            pool.stats[r, : len(toks), 0] = torch.tensor(toks, dtype=torch.float32)
        # what NativeSynthesizer.tts_encode returns: frames, and each row's decode key (the encode key + 1), stream and
        # noise scale
        return types.SimpleNamespace(frames=[n_frames(self.rows[r][2]) for r in rows], dec_keys=[k + 1 for k in seeds],
                                     dec_streams=list(streams), dec_noise_scale=list(noise_scale))

    def tts_decode_windows(self, state, wins):
        self.calls.append("tts_decode_windows")
        self.windows.append(list(wins))
        wmax = max(ln for _, _, ln in wins)
        o = torch.zeros(len(wins), HOP * wmax)
        for i, (r, f0, ln) in enumerate(wins):
            seed, stream, toks = self.rows[r]
            assert f0 + ln <= state.frames[r] == n_frames(toks)
            assert (state.dec_keys[r], state.dec_streams[r]) == (seed + 1, stream)
            assert state.stats[r, : len(toks), 0].tolist() == list(toks)
            o[i, : HOP * ln] = torch.from_numpy(sentence_audio(seed, stream, toks, np.arange(f0 * HOP, (f0 + ln) * HOP)))
        return o, None


def make_models(tts_sr=SR, tts_device="cpu"):
    from oracle import vc_oracle as O
    from openvoice_b200.api import BaseSpeakerTTS, ToneColorConverter
    from openvoice_b200.utils import HParams
    hp = copy.deepcopy(O.DEFAULT_HPARAMS)
    hp["data"].update(sampling_rate=tts_sr, hop_length=HOP, n_speakers=3)
    hp["speakers"] = {"default": 1}
    tts = BaseSpeakerTTS.__new__(BaseSpeakerTTS)
    tts.hps, tts.text_frontend = HParams(**hp), (lambda text, mark: [[ord(c) % 50 for c in w] for w in text.split(".") if w])
    tts.model = FakeTtsModel()
    tts.model.device = torch.device(tts_device)
    conv = ToneColorConverter.__new__(ToneColorConverter)
    conv.hps, conv.device, conv.watermark_model, conv.HALO_FRAMES = FakeConverter.hps, "cpu", None, 128
    conv.model = FakeModel()
    conv.model.device = torch.device("cpu")
    return tts, conv


def keys(i):
    return dict(speaker="default", src_se=torch.full((1, GIN, 1), 0.1 * i), tgt_se=torch.full((1, GIN, 1), -0.2 * i),
                tau=0.3 + 0.1 * i, seed=1000 + i, convert_seed=77 + i, speed=[1.0, 0.8, 1.25][i % 3])


def sentences(i, k):
    rng = np.random.default_rng(i)
    return [rng.integers(1, 50, int(rng.integers(15, 70))).tolist() for _ in range(k)]


def expected(conv, i, sents):
    """The session's utterance (sentences and 50 ms / speed gaps) through StreamingSessions in one push and a close."""
    from openvoice_b200.streaming import StreamingSessions
    q = keys(i)
    gap = np.zeros(int(SR * 0.05 / q["speed"]), np.float32)
    parts = []
    for j, toks in enumerate(sents):
        parts += [sentence_audio(q["seed"], j, tuple(toks), np.arange(n_frames(toks) * HOP)), gap]
    ss = StreamingSessions(conv, window_frames=64)
    sid = ss.open(q["src_se"], q["tgt_se"], tau=q["tau"], seed=q["convert_seed"])
    return np.concatenate([ss.push({sid: np.concatenate(parts)})[sid], ss.close([sid])[sid]])


def run(cs, script, steps=200):
    """Drive ``cs``: script[k] is a list of callables run before step k.  Returns {sid: concatenated chunks}."""
    out = {}
    for k in range(steps):
        for f in script.get(k, []):
            f()
        for sid, c in cs.step().items():
            assert c.dtype == np.float32 and len(c)
            out.setdefault(sid, []).append(c)
    assert not cs.sessions
    return {sid: np.concatenate(v) for sid, v in out.items()}


def sessions(tts, conv):
    from openvoice_b200.streaming import CloneSessions
    return CloneSessions(conv, tts, window_frames=64, first_window_frames=16)


# ------------------------------------------------------------------------------------------------ contract
def test_staggered_sessions_match_their_whole_utterance():
    tts, conv = make_models()
    cs = sessions(tts, conv)
    S = {i: sentences(i, 3) for i in range(4)}
    ids = {}

    def opener(i, say_all=False):
        def f():
            ids[i] = cs.open(**keys(i))
            if say_all:
                cs.say(ids[i], ids=S[i])
                cs.end(ids[i])
        return f

    script = {0: [opener(0, True), opener(1)],
              1: [lambda: cs.say(ids[1], ids=S[1][:1])],
              4: [opener(2), lambda: cs.say(ids[1], ids=S[1][1:2]), lambda: cs.say(ids[2], ids=S[2][:2])],
              5: [opener(3), lambda: cs.say(ids[3], ids=S[3])],
              9: [lambda: cs.say(ids[1], ids=S[1][2:]), lambda: cs.say(ids[2], ids=S[2][2:]), lambda: cs.end(ids[2])],
              14: [lambda: cs.end(ids[1])],
              30: [lambda: cs.end(ids[3])]}
    got = run(cs, script)
    for i in range(4):
        ref = expected(conv, i, S[i])
        assert got[ids[i]].shape == ref.shape and np.array_equal(got[ids[i]], ref), i
    # sentence j of a session was keyed (seed, stream j) however its text arrived
    for i in range(4):
        assert [(s, j) for s, j in tts.model.encoded if s == 1000 + i] == [(1000 + i, j) for j in range(3)]


def test_first_window_only_for_the_first_sentence():
    tts, conv = make_models()
    cs = sessions(tts, conv)
    sid = cs.open(**keys(0))
    cs.say(sid, ids=sentences(5, 2))
    cs.encode_pending()
    cs.say(sid, ids=sentences(6, 1))
    s = cs.sessions[sid]
    cs.encode_pending()
    firsts = [e1 - e0 for _, _, _, e0, e1, _, _ in s.plans if e0 == 0]
    assert firsts == [16, 64, 64]
    last = [g for *_, g, end in s.plans if end]
    assert len(last) == 3 and all(last)


# ------------------------------------------------------------------------------------------------ closing
def test_session_closes_in_the_step_that_writes_its_last_gap():
    tts, conv = make_models()
    cs = sessions(tts, conv)
    a = cs.open(**keys(0))
    cs.say(a, ids=sentences(1, 1))
    cs.end(a)
    steps = 0
    while a in cs.sessions:
        cs.step()
        steps += 1
    n_windows = sum(len(w) for w in tts.model.windows)
    assert steps == len(tts.model.windows) and n_windows >= steps
    # end after the last gap: the session stays open, then a later step closes it without decoding
    b = cs.open(**keys(1))
    cs.say(b, ids=sentences(2, 1))
    while cs.sessions[b].plans or cs.sessions[b].unencoded:
        cs.step()
    before = list(tts.model.calls)
    assert cs.step() == {} and tts.model.calls == before and b in cs.sessions     # nothing to advance: no calls
    cs.end(b)
    out = cs.step()
    assert b not in cs.sessions and tts.model.calls == before and set(out) <= {b}


def test_step_calls_at_most_one_of_each():
    tts, conv = make_models()
    cs = sessions(tts, conv)
    ids = [cs.open(**keys(i)) for i in range(3)]
    for i in ids:
        cs.say(i, ids=sentences(10 + i, 2))
    counts = {}
    from openvoice_b200.streaming import StreamingSessions
    pushes = []
    real = StreamingSessions.push_device

    def push_device(self, *a, **k):
        pushes.append(1)
        return real(self, *a, **k)
    StreamingSessions.push_device = push_device
    try:
        for k in range(40):
            n0, p0 = len(tts.model.calls), len(pushes)
            if k == 3:
                for i in ids:
                    cs.end(i)
            cs.step()
            new = tts.model.calls[n0:]
            for name in ("tts_encode", "tts_state_rows", "tts_decode_windows"):
                counts[name] = max(counts.get(name, 0), new.count(name))
            assert len(pushes) - p0 <= 1
            if not cs.sessions:
                break
    finally:
        StreamingSessions.push_device = real
    assert not cs.sessions and counts == {"tts_encode": 1, "tts_state_rows": 0, "tts_decode_windows": 1}, counts


# ------------------------------------------------------------------------------------------------ rows
def test_pool_rows_are_freed_reused_and_repitched():
    tts, conv = make_models()
    cs = sessions(tts, conv)
    a = cs.open(**keys(0))
    cs.say(a, ids=[[1] * 10, [2] * 12])
    cs.end(a)
    cs.encode_pending()
    assert cs.pool_rows_in_use == 2 and cs.rows == 2
    cs.step()                                            # both sentences decode whole in this step: their rows are free
    assert cs.pool_rows_in_use == 0
    b = cs.open(**keys(1))
    cs.say(b, ids=[[3] * 90])                            # a longer sentence: the pool is re-pitched, rows kept
    cs.end(b)
    while cs.sessions:
        cs.step()
    assert "repitch" in tts.model.calls and cs.pool.Tp >= 90
    assert cs.pool_rows_in_use == 0 and cs.ss.rows_in_use == 0
    rows = cs.rows
    c = cs.open(**keys(2))
    cs.say(c, ids=sentences(3, 2))
    cs.step()
    assert cs.rows == rows                               # freed rows are reused
    d = cs.open(**keys(0))
    cs.say(d, ids=sentences(4, 3))
    cs.step()
    cs.cancel(c)
    cs.cancel(d)
    assert not cs.sessions and cs.pool_rows_in_use == 0 and cs.ss.rows_in_use == 0 and not cs.pending
    assert cs.step() == {}


def test_cancel_leaves_the_neighbours_unchanged():
    tts, conv = make_models()
    cs = sessions(tts, conv)
    S = {i: sentences(20 + i, 6) for i in range(3)}
    ids = {i: cs.open(**keys(i)) for i in range(3)}
    for i in range(3):
        cs.say(ids[i], ids=S[i])
        cs.end(ids[i])

    def cancel():
        assert cs.sessions[ids[1]].plans                 # mid-stream
        cs.cancel(ids[1])
    got = run(cs, {2: [cancel]})
    assert ids[1] in got
    for i in (0, 2):
        assert np.array_equal(got[ids[i]], expected(conv, i, S[i])), i


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals():
    from openvoice_b200.streaming import CloneSessions
    tts, conv = make_models()
    cs = sessions(tts, conv)
    for kw, msg in ((dict(tau=float("nan")), "session 0: tau"), (dict(src_se=None), "session 0 has no src_se"),
                    (dict(tgt_se=torch.zeros(GIN + 1)), "tgt_se has"), (dict(speed=0.0), "session 0: speed"),
                    (dict(convert_seed=-1), "convert_seed"), (dict(seed=2 ** 64), "seed")):
        with pytest.raises(ValueError, match=msg):
            cs.open(**dict(keys(0), **kw))
    assert not cs.sessions
    sid = cs.open(**keys(0))
    with pytest.raises(ValueError, match="no sentences"):
        cs.say(sid, ids=[])
    with pytest.raises(ValueError, match="unknown"):
        cs.say(sid + 5, ids=[[1, 2]])
    cs.say(sid, text="ab cd.ef")
    assert [q for _, q in cs.pending] == [[ord(c) % 50 for c in "ab cd"], [ord(c) % 50 for c in "ef"]]
    cs.end(sid)
    with pytest.raises(ValueError, match="has ended"):
        cs.say(sid, ids=[[1, 2]])
    with pytest.raises(ValueError, match="unknown"):
        cs.cancel(sid + 1)
    tts48, conv48 = make_models(tts_sr=48000)
    with pytest.raises(ValueError, match="48000"):
        CloneSessions(conv48, tts48)
    tts_meta, conv_meta = make_models(tts_device="meta")
    with pytest.raises(ValueError, match="meta"):
        CloneSessions(conv_meta, tts_meta)
    with pytest.raises(ValueError, match="window_frames"):
        CloneSessions(conv, tts, window_frames=0)


def test_too_short_session_is_cancelled_and_the_others_continue():
    """The stand-in's shortest sentence (no tokens) decodes to 2 frames, which the real rule accepts, so the length rule is
    made stricter here: under 2000 samples is too short.  The failing session is cancelled in the step that encodes its
    last sentence, before that step's decode; the others then finish unchanged."""
    tts, conv = make_models()
    cs = sessions(tts, conv)
    S = {i: sentences(30 + i, 2) for i in range(2)}
    ids = {i: cs.open(**keys(i)) for i in range(2)}
    short = cs.open(**keys(2))
    for i in range(2):
        cs.say(ids[i], ids=S[i][:1])
    cs.step()
    cs.say(short, ids=[[]])                               # an empty sentence: 2 frames, then ended with no more text
    cs.end(short)
    orig = conv._check_clone_lengths

    def strict(lengths, rate, names=None):
        for n, who in zip(lengths, names):
            if n < 2000:
                raise ValueError(f"{who}: its utterance has {n} samples")
        return orig(lengths, rate, names)
    conv._check_clone_lengths = strict
    for i in range(2):
        cs.say(ids[i], ids=S[i][1:])
        cs.end(ids[i])
    before = list(tts.model.calls)
    with pytest.raises(ValueError, match=f"session {short}: its utterance"):
        cs.step()
    assert short not in cs.sessions and "tts_decode_windows" not in tts.model.calls[len(before):]   # no decode
    got = run(cs, {})
    for i in range(2):
        assert np.array_equal(got[ids[i]], expected(conv, i, S[i])), i


# ------------------------------------------------------------------------------------------------ ptxas
def test_state_rows_kernel_does_not_spill():
    """-Xptxas -v report of the library's translation unit (written by the build): the pool copy uses no stack and
    spills nothing."""
    import os
    import re
    log = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "openvoice_b200", "csrc", "build",
                       "ovc_lib.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("no ptxas report: the library has not been built")
    m = re.search(r"Compiling entry function '(_ZN3ovc21tts_state_rows_kernel\w*)' for 'sm_90a'\n(?:ptxas info[^\n]*\n)*?"
                  r"\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", open(log).read())
    assert m, "tts_state_rows_kernel not in the ptxas report"
    assert (int(m.group(2)), int(m.group(3)), int(m.group(4))) == (0, 0, 0), m.group(0)


def test_bad_text_names_its_session_and_the_others_run_on():
    tts, conv = make_models()
    cs = sessions(tts, conv)
    S = sentences(40, 2)
    a = cs.open(**keys(0))
    cs.say(a, ids=S)
    cs.end(a)
    b = cs.open(**keys(1))
    for bad, msg in (([[1, 2, 999]], f"session {b}: token ids"), ([[3, -1]], f"session {b}: token ids")):
        with pytest.raises(ValueError, match=msg):
            cs.say(b, ids=bad)
    assert [sid for sid, _ in cs.pending] == [a] * 2 and cs.sessions[b].said == 0
    c = cs.open(**dict(keys(2), speaker=7))
    with pytest.raises(ValueError, match=f"session {c}: speaker ids"):
        cs.say(c, ids=[[1, 2]])
    for kw, msg in ((dict(noise_scale=float("nan")), "noise_scale"), (dict(noise_scale_w=float("inf")), "noise_scale_w"),
                    (dict(sdp_ratio=float("nan")), "sdp_ratio")):
        with pytest.raises(ValueError, match=f"session {cs.next_id}: {msg}"):
            cs.open(**dict(keys(0), **kw))
    cs.cancel(c)
    cs.say(b, ids=S[:1])                                 # the session goes on with good text
    cs.end(b)
    got = run(cs, {})
    assert np.array_equal(got[a], expected(conv, 0, S)) and np.array_equal(got[b], expected(conv, 1, S[:1]))
    assert cs.pool_rows_in_use == 0


def test_a_failed_encode_takes_no_rows_and_keeps_the_text(monkeypatch):
    tts, conv = make_models()
    cs = sessions(tts, conv)
    S = sentences(41, 3)
    a = cs.open(**keys(0))
    cs.say(a, ids=S[:1])
    first = cs.step()
    rows, free = cs.rows, list(cs.free_rows)
    cs.say(a, ids=S[1:])
    cs.end(a)
    real = tts.model.tts_encode

    def failing(*args, **kw):
        raise RuntimeError("device out of memory")
    monkeypatch.setattr(tts.model, "tts_encode", failing)
    for _ in range(3):
        with pytest.raises(RuntimeError):
            cs.step()
        assert (cs.rows, cs.free_rows, len(cs.pending)) == (rows, free, 2)
    monkeypatch.setattr(tts.model, "tts_encode", real)
    rest = run(cs, {})
    got = np.concatenate([first[a], rest[a]] if a in first else [rest[a]])
    assert np.array_equal(got, expected(conv, 0, S)) and cs.pool_rows_in_use == 0
