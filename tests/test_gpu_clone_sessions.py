"""-m gpu: live text-to-cloned-voice sessions.  The pool copy (ovc_tts_encode_state_rows / ovc_tts_state_rows) against
ovc_tts_encode_state bit for bit, with its padding and its clamping; CloneSessions against clone_stream_batch (bit for
bit) and clone_batch (1e-4 of the rms) whatever the timing of the text; the launches of a step.  fp32 and f16x3."""
import numpy as np
import pytest
import torch

from test_gpu_clone import models, rel_err, requests

pytestmark = pytest.mark.gpu


@pytest.fixture(params=["fp32", "f16x3"])
def pair(request, tmp_path_factory):
    return models(tmp_path_factory, request.param)


# ------------------------------------------------------------------------------------------------ the pool copy
def encode(m, lengths, **kw):
    rng = np.random.default_rng(3)
    x = torch.zeros(len(lengths), max(lengths), dtype=torch.int64)
    for b, n in enumerate(lengths):
        x[b, :n] = torch.from_numpy(rng.integers(1, 40, n))
    return m.tts_encode(x, torch.tensor(lengths), sid=torch.tensor([1, 2, 0, 1][: len(lengths)]),
                        seeds=[5 + b for b in range(len(lengths))], streams=list(range(len(lengths))),
                        noise_scale=0.667, length_scale=1.0, noise_scale_w=0.6, sdp_ratio=0.2, **kw)


def test_pool_rows_equal_the_encode_state(pair):
    from openvoice_b200.api import TtsPool, TtsState
    m = pair[0].model
    lengths, rows = [37, 12, 60, 25], [5, 0, 3, 7]
    state = encode(m, lengths)
    pool = TtsPool(m.native, m.device)
    pool.fit(9, 100)
    ps = encode(m, lengths, pool=pool, rows=rows)
    assert ps.frames == state.frames and pool.Tp >= 100 and pool.N >= 9
    T = max(lengths)
    for b, r in enumerate(rows):
        assert torch.equal(pool.stats[r, :T], state.stats[b]), b
        assert torch.equal(pool.cum[r, :T], state.cum[b]), b
        assert torch.equal(pool.g[r], state.g[b]) and int(pool.y_lengths[r]) == state.frames[b], b
        assert not pool.stats[r, T:].any(), b                                      # padding: stats 0
        assert bool((pool.cum[r, T:] == state.cum[b, T - 1]).all()), b           # cum keeps its last value
    # the same windows over the pool and over the state: the same samples, bit for bit
    wins = [(b, 0, state.frames[b]) for b in range(4)] + [(2, 17, 40), (0, 3, state.frames[0] - 3)]
    o_ref, _ = m.tts_decode_windows(state, wins)
    o_ref = o_ref.clone()
    full = TtsState(pool.stats, pool.cum, pool.g, pool.y_lengths, [0] * pool.N, [0] * pool.N, [0] * pool.N, [0.0] * pool.N)
    for b, r in enumerate(rows):
        full.frames[r], full.dec_keys[r] = state.frames[b], state.dec_keys[b]
        full.dec_streams[r], full.dec_noise_scale[r] = state.dec_streams[b], state.dec_noise_scale[b]
    o_pool, _ = m.tts_decode_windows(full, [(rows[b], f0, ln) for b, f0, ln in wins])
    assert torch.equal(o_pool, o_ref)
    # a larger pitch re-pitches the rows with the same padding, and they still decode the same
    pool.fit(pool.N, 200)
    assert pool.Tp >= 200 and bool((pool.cum[rows[1], T:] == state.cum[1, T - 1]).all())
    full = full._replace(stats=pool.stats, cum=pool.cum, g=pool.g, y_lengths=pool.y_lengths)
    o_pool, _ = m.tts_decode_windows(full, [(rows[b], f0, ln) for b, f0, ln in wins])
    assert torch.equal(o_pool, o_ref)


def test_out_of_range_rows_stay_inside_the_pool(pair):
    m = pair[0].model
    state = encode(m, [20, 31])
    N, Tp, C2, gin = 3, 48, state.stats.shape[2], state.g.shape[1]
    big = [torch.full((N + 2,) + shape, fill, dtype=dt, device=m.device) for shape, fill, dt in
           (((Tp, C2), 7.0, torch.float32), ((Tp,), 7, torch.int32), ((gin,), 7.0, torch.float32), ((), 7, torch.int64))]
    pool = [t[1:N + 1] for t in big]
    m.native.tts_state_rows([-5, 10 ** 12], *pool, src=(state.stats, state.cum, state.g, state.y_lengths))
    torch.cuda.synchronize()
    for t in big:
        assert bool((t[0] == 7).all()) and bool((t[N + 1] == 7).all())          # nothing outside the pool
    assert torch.equal(pool[0][0, :31], state.stats[0]) and torch.equal(pool[2][2], state.g[1])   # clamped rows
    assert torch.equal(pool[1][2], torch.nn.functional.pad(state.cum[1], (0, Tp - 31), value=int(state.cum[1, -1])))


# ------------------------------------------------------------------------------------------------ the contract
def one_shot(tts, conv, q, W, W1):
    return np.concatenate([c for _, c in conv.clone_stream_batch(tts, [q], window_frames=W, first_window_frames=W1)])


OPEN = ("speaker", "src_se", "tgt_se", "tau", "seed", "convert_seed", "speed", "noise_scale")


def drive(cs, reqs, scenario):
    """Run the requests through ``cs`` with the text timing of ``scenario``; returns ({request: audio}, cancelled)."""
    ids, out, k = {}, {}, 0
    cancelled = set()
    while True:
        for r, q in enumerate(reqs):
            sents = q["ids"]
            if scenario == "at_open" and k == 0 or scenario == "late_end" and k == 0 or \
                    scenario == "staggered" and k == 3 * r or scenario == "cancel" and k == 0:
                ids[r] = cs.open(**{n: q[n] for n in OPEN})
                cs.say(ids[r], ids=sents)
                if scenario != "late_end":
                    cs.end(ids[r])
            if scenario == "one_per_step":
                if k == 0:
                    ids[r] = cs.open(**{n: q[n] for n in OPEN})
                if k % 2 == 0 and k // 2 < len(sents):
                    cs.say(ids[r], ids=[sents[k // 2]])
                    if k // 2 == len(sents) - 1:
                        cs.end(ids[r])
            if scenario == "late_end" and k == 12:
                cs.end(ids[r])
        if scenario == "cancel" and k == 1:                # a neighbour that is still mid-stream goes away
            mid = [r for r in (2, 1, 3, 0) if ids[r] in cs.sessions and cs.sessions[ids[r]].plans]
            assert mid, "no session is mid-stream at step 1"
            r = mid[0]
            assert cs.sessions[ids[r]].ss_id is not None and cs.ss.sessions[cs.sessions[ids[r]].ss_id].n_in > 0
            cs.cancel(ids[r])
            cancelled.add(r)
        for sid, c in cs.step().items():
            out.setdefault(sid, []).append(c)
        k += 1
        if k > 3 * len(reqs) + 13 and not cs.sessions:
            break
        assert k < 500
    back = {sid: r for r, sid in ids.items()}
    return {back[sid]: np.concatenate(v) for sid, v in out.items()}, cancelled


@pytest.mark.parametrize("scenario", ["at_open", "one_per_step", "staggered", "cancel", "late_end"])
def test_sessions_equal_the_one_shot_stream(pair, scenario):
    from openvoice_b200.streaming import CloneSessions
    tts, conv = pair
    W, W1 = 64, 16
    reqs = requests(4)
    cs = CloneSessions(conv, tts, window_frames=W, first_window_frames=W1)
    got, cancelled = drive(cs, reqs, scenario)
    assert cs.pool_rows_in_use == 0 and cs.ss.rows_in_use == 0
    for r, q in enumerate(reqs):
        if r in cancelled:
            continue
        ref = one_shot(tts, conv, q, W, W1)
        assert got[r].shape == ref.shape and np.array_equal(got[r], ref), (scenario, r)
        whole = conv.clone_batch(tts, [q])[0]
        err = rel_err(got[r], whole)
        print(f"{scenario} request {r}: max|d|/rms vs clone_batch = {err:.2e}")
        assert got[r].shape == whole.shape and err <= 1e-4, (scenario, r, err)


# ------------------------------------------------------------------------------------------------ launches
def test_a_step_launches_at_most_one_of_each(pair, monkeypatch):
    from openvoice_b200.streaming import CloneSessions, StreamingSessions
    tts, conv = pair
    n = {"tts_encode": 0, "encode_rows": 0, "tts_decode_windows": 0, "push_device": 0, "conv_native": 0}
    nat = tts.model.native

    def count(name, fn):
        def f(*a, **k):
            n[name] += 1
            return fn(*a, **k)
        return f
    monkeypatch.setattr(nat, "tts_encode", count("tts_encode", nat.tts_encode))
    monkeypatch.setattr(nat, "tts_decode_windows", count("tts_decode_windows", nat.tts_decode_windows))
    real_rows = nat.tts_state_rows

    def state_rows(*a, **k):                               # the encode's copy; a re-pitch passes src
        n["encode_rows"] += k.get("src") is None
        return real_rows(*a, **k)
    monkeypatch.setattr(nat, "tts_state_rows", state_rows)
    monkeypatch.setattr(StreamingSessions, "push_device", count("push_device", StreamingSessions.push_device))
    for name in ("spectrogram_ring", "voice_conversion", "splice"):
        monkeypatch.setattr(conv.model.native, name, count("conv_native", getattr(conv.model.native, name)))
    reqs = requests(3)
    cs = CloneSessions(conv, tts, window_frames=64, first_window_frames=16)
    ids = [cs.open(**{k: q[k] for k in OPEN}) for q in reqs]
    for sid, q in zip(ids, reqs):
        cs.say(sid, ids=q["ids"][:1])
    steps = 0
    while any(s.plans or s.unencoded for s in cs.sessions.values()):
        before = dict(n)
        cs.step()
        d = {k: n[k] - before[k] for k in n}
        assert d["tts_encode"] <= 1 and d["encode_rows"] <= 1 and d["tts_decode_windows"] <= 1 and d["push_device"] <= 1, d
        steps += 1
    assert n["tts_encode"] == 1 and steps >= 1
    before = dict(n)
    assert cs.step() == {} and n == before                 # every session waits for text: nothing is launched
    for sid, q in zip(ids, reqs):
        cs.end(sid)
    while cs.sessions:
        cs.step()


def test_unindexed_cuda_device(tmp_path, tmp_path_factory):
    """Models built with device="cuda" (no index), as bench.py builds them: the same audio as on "cuda:0"."""
    import copy
    import json

    from oracle import tts_oracle as T
    from oracle import vc_oracle as O
    from openvoice_b200.api import BaseSpeakerTTS, ToneColorConverter
    from openvoice_b200.streaming import CloneSessions
    hp = copy.deepcopy(O.DEFAULT_HPARAMS)
    hp["data"]["n_speakers"] = T.TTS_HPARAMS["n_speakers"]
    hp["speakers"] = {"default": 1, "whispering": 2}
    (tmp_path / "tts.json").write_text(json.dumps(hp))
    torch.save({"model": T.synthetic_tts_state_dict()}, tmp_path / "tts.pth")
    (tmp_path / "vc.json").write_text(json.dumps(O.DEFAULT_HPARAMS))
    tts = BaseSpeakerTTS(str(tmp_path / "tts.json"), device="cuda", precision="f16x3")
    tts.load_ckpt(str(tmp_path / "tts.pth"))
    conv = ToneColorConverter(str(tmp_path / "vc.json"), device="cuda", enable_watermark=False, precision="f16x3")
    conv.model.load_state_dict(O.synthetic_state_dict(1234))
    tts0, conv0 = models(tmp_path_factory, "f16x3")
    reqs = requests(2)
    for q in reqs:
        ref = one_shot(tts0, conv0, q, 64, 16)
        assert np.array_equal(one_shot(tts, conv, q, 64, 16), ref)
        cs = CloneSessions(conv, tts, window_frames=64, first_window_frames=16)
        sid = cs.open(**{n: q[n] for n in OPEN})
        chunks = []
        for sent in q["ids"]:
            cs.say(sid, ids=[sent])
            chunks += list(cs.step().values())
        cs.end(sid)
        while cs.sessions:
            chunks += list(cs.step().values())
        assert np.array_equal(np.concatenate(chunks), ref)
