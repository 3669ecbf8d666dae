"""-m gpu: streaming base-speaker TTS (include/ovc.h: ovc_tts_encode_state / ovc_tts_decode_windows).  The decode half
runs in time windows of caller-owned encode state; the windows' interiors give the whole decode's audio.  Every
comparison is bit for bit unless it names a bound."""
import copy
import json

import numpy as np
import pytest
import torch

from oracle import tts_oracle as T
from oracle import vc_oracle as O

pytestmark = pytest.mark.gpu

HOP = 256


def rel_err(got, ref):
    ref = np.asarray(ref, dtype=np.float64)
    return float(np.abs(np.asarray(got, dtype=np.float64) - ref).max() / (np.sqrt((ref ** 2).mean()) + 1e-30))


# ------------------------------------------------------------------------------------------------ fixtures
@pytest.fixture(params=["fp32", "f16x3"])
def nat(request):
    from conftest import get_native_tts
    m = get_native_tts()
    m.native.set_precision(request.param)
    yield m
    m.native.set_precision(m.precision)


_engines = {}


def engine(tmp_path_factory, precision):
    from openvoice_b200.api import BaseSpeakerTTS
    if precision not in _engines:
        d = tmp_path_factory.mktemp("tts")
        hp = copy.deepcopy(O.DEFAULT_HPARAMS)
        hp["data"]["n_speakers"] = T.TTS_HPARAMS["n_speakers"]
        hp["speakers"] = {"default": 1, "whispering": 2}
        (d / "config.json").write_text(json.dumps(hp))
        torch.save({"model": T.synthetic_tts_state_dict()}, d / "checkpoint.pth")
        eng = BaseSpeakerTTS(str(d / "config.json"), device="cuda:0", precision=precision)
        eng.load_ckpt(str(d / "checkpoint.pth"))
        _engines[precision] = eng
    return _engines[precision]


@pytest.fixture(params=["fp32", "f16x3"])
def eng(request, tmp_path_factory):
    return engine(tmp_path_factory, request.param)


def sentences(k, seed, lo=5, hi=60, long_first=False):
    rng = np.random.default_rng(seed)
    out = [rng.integers(0, T.TTS_HPARAMS["n_vocab"], int(rng.integers(lo, hi))).tolist() for _ in range(k)]
    if long_first:
        out[0] = rng.integers(0, T.TTS_HPARAMS["n_vocab"], 300).tolist()
    return out


# three rows: a ~300-token sentence spoken slowly, a medium one and a short one, each with its own keys
ENC = dict(seeds=[5, 2 ** 64 - 1, 9], streams=[0, 3, 1], noise_scale=[0.667, 0.3, 1.0], length_scale=[1 / 0.7, 1.0, 1.2],
           noise_scale_w=0.6, sdp_ratio=0.2)


def encoded(m):
    tokens, lengths, sid, _ = T.synthetic_tts_inputs(3, 300, 21, [300, 120, 37])
    state = m.tts_encode(tokens, lengths, sid=sid, **ENC)
    o, _, y_mask, (_, z_p, _, _) = m.infer(tokens, lengths, sid=sid, ragged=True, latents=True, **ENC)
    return state, o[:, 0], z_p


def decode(m, state, wins, **kw):
    o, zp = m.tts_decode_windows(state, wins, **kw)
    return o.clone(), zp


def interiors(m, state, row, first, window, halo):
    from openvoice_b200.api import plan_tts_windows
    plan = plan_tts_windows(state.frames[row], first, window, halo)
    o, _ = decode(m, state, [(row, lo, hi - lo) for lo, hi, _, _ in plan])
    return torch.cat([o[k, (e0 - lo) * HOP: (e1 - lo) * HOP] for k, (lo, _, e0, e1) in enumerate(plan)]).cpu().numpy(), plan


# ------------------------------------------------------------------------------------------------ 1. whole decode
def test_whole_decode_as_windows_is_bit_identical(nat):
    state, o_whole, zp_whole = encoded(nat)
    F = state.frames
    assert F[0] > 32 + 256, F         # the long sentence spans several windows of both sizes
    Ty = max(F)
    o, zp = decode(nat, state, [(b, 0, F[b]) for b in range(3)], w_max=Ty, latents=True)
    assert torch.equal(o, o_whole) and torch.equal(zp, zp_whole)


# ------------------------------------------------------------------------------------------------ 2. expansion
def test_expansion_at_offsets_is_exact(nat):
    state, _, zp_whole = encoded(nat)
    F = state.frames
    wins = [(0, 0, 17), (0, 50, 100), (0, F[0] - 33, 33), (1, 5, 60), (2, 0, F[2]), (0, F[0] // 2, 1), (1, F[1] - 1, 1)]
    _, zp = decode(nat, state, wins, latents=True)
    for i, (r, f0, ln) in enumerate(wins):
        assert torch.equal(zp[i, :, :ln], zp_whole[r, :, f0: f0 + ln]), i
        assert not zp[i, :, ln:].any(), i


# ------------------------------------------------------------------------------------------------ 3. interiors
def test_interiors_match_the_whole_sentence(nat):
    from openvoice_b200.api import TTS_HALO_FRAMES
    state, o_whole, _ = encoded(nat)
    F0 = state.frames[0]
    ref = o_whole[0, : F0 * HOP].cpu().numpy()
    for first, window in ((32, 256), (20, 100), (256, 32)):
        got, plan = interiors(nat, state, 0, first, window, TTS_HALO_FRAMES)
        assert len(plan) >= 2 and got.shape == ref.shape
        err = rel_err(got, ref)
        print(f"{nat.native.precision} first {first} window {window}: {len(plan)} windows, max|d|/rms = {err:.2e}")
        assert err <= 2e-6, (first, window, err)
    got, plan = interiors(nat, state, 0, F0, 256, TTS_HALO_FRAMES)
    assert len(plan) == 1 and np.array_equal(got, ref)
    got, _ = interiors(nat, state, 0, 32, 256, 16)             # control: a halo short of the receptive field
    err = rel_err(got, ref)
    print(f"{nat.native.precision} halo 16: max|d|/rms = {err:.2e}")
    assert err > 2e-6


# ------------------------------------------------------------------------------------------------ 4. batch independence
def test_window_does_not_depend_on_its_batch(nat):
    state, _, _ = encoded(nat)
    F = state.frames
    target = (0, 100, 150)
    alone, _ = decode(nat, state, [target])
    n = target[2] * HOP
    for wins in ([(2, 0, F[2]), target, (1, 10, 40), (0, 0, 30)], [target, (0, 200, 84)], [(1, 0, F[1]), (1, 7, 9), target]):
        got, _ = decode(nat, state, wins)
        i = wins.index(target)
        assert torch.equal(got[i, :n], alone[0, :n]), wins


# ------------------------------------------------------------------------------------------------ 5. tts_stream
@pytest.mark.parametrize("k", [1, 4])
def test_stream_matches_tts(eng, k):
    ids = sentences(k, 30 + k, long_first=True)
    speed, seed = 0.8, 1234 + k
    ref_parts = eng.tts_from_ids(ids, "default", speed=speed, seed=seed)
    ref = eng.audio_numpy_concat(ref_parts, 22050, speed)
    chunks = list(eng.tts_stream(ids=ids, speaker="default", speed=speed, seed=seed, window_frames=256,
                                 first_window_frames=32))
    got = np.concatenate(chunks)
    assert got.shape == ref.shape
    err = rel_err(got, ref)
    print(f"{eng.model.precision} {k} sentences, {len(chunks)} chunks: max|d|/rms = {err:.2e}")
    assert err <= 2e-6
    gap, pos = int(22050 * 0.05 / speed), 0
    for p in ref_parts:
        pos += len(p)
        assert not got[pos: pos + gap].any()
        pos += gap
    assert len(ref_parts[0]) > 32 * HOP and len(chunks[0]) == 32 * HOP


# ------------------------------------------------------------------------------------------------ 6. tts_stream_batch
def test_stream_batch_equals_each_request_alone(eng):
    reqs = [dict(ids=sentences(1, 1, long_first=True), speaker="default", speed=0.7, seed=1),
            dict(ids=sentences(4, 2), speaker="whispering", speed=1.0, seed=2 ** 64 - 1, noise_scale=0.3, sdp_ratio=0.5),
            dict(ids=sentences(2, 3), speaker=0, speed=1.3, seed=2, noise_scale_w=0.9),
            dict(ids=sentences(3, 4, long_first=True), speaker="default", speed=1.0, seed=1, noise_scale=1.0,
                 noise_scale_w=0.2)]
    per = [[] for _ in reqs]
    order = []
    for r, chunk in eng.tts_stream_batch(reqs, window_frames=100, first_window_frames=20):
        per[r].append(chunk)
        order.append(r)
    for r, q in enumerate(reqs):
        kw = {k: q[k] for k in ("noise_scale", "noise_scale_w", "sdp_ratio") if k in q}
        alone = list(eng.tts_stream_batch([q], window_frames=100, first_window_frames=20))
        assert np.array_equal(np.concatenate(per[r]), np.concatenate([c for _, c in alone])), r
        parts = eng.tts_from_ids(q["ids"], q["speaker"], speed=q["speed"], seed=q["seed"], **kw)
        ref = eng.audio_numpy_concat(parts, 22050, q["speed"])
        assert np.concatenate(per[r]).shape == ref.shape and rel_err(np.concatenate(per[r]), ref) <= 2e-6, r
    # one chunk per unfinished request per step, in request order
    step, seen = 0, set()
    for r in order:
        if r in seen:
            step, seen = step + 1, set()
        assert not seen or r > max(seen)
        seen.add(r)


# ------------------------------------------------------------------------------------------------ 7. caller-owned state
def test_unrelated_tts_between_chunks_does_not_change_the_stream(eng):
    ids = sentences(2, 50, long_first=True)
    kw = dict(speaker="default", speed=0.9, seed=77, window_frames=100, first_window_frames=20)
    ref = list(eng.tts_stream(ids=ids, **kw))
    gen = eng.tts_stream(ids=ids, **kw)
    got = [next(gen)]
    eng.tts_from_ids(sentences(5, 51), "whispering", speed=1.2, seed=3)
    got.append(next(gen))
    eng.tts_batch([dict(ids=sentences(3, 52), speaker=0, seed=4)])
    got += list(gen)
    assert len(got) == len(ref)
    for a, b in zip(got, ref):
        assert np.array_equal(a, b)


# ------------------------------------------------------------------------------------------------ 8. graph replay
def test_graph_replay_is_bit_identical(eng):
    nat = eng.model.native
    ids = [sentences(1, 60, long_first=True)[0]]
    kw = dict(speaker="default", speed=0.6, seed=8, window_frames=64, first_window_frames=16)
    nat.set_option("graph", 0)
    direct = list(eng.tts_stream(ids=ids, **kw))
    nat.set_option("graph", 1)
    before = nat.graph_replays
    graphed = list(eng.tts_stream(ids=ids, **kw))
    assert len(direct) >= 6 and nat.graph_replays - before >= 2
    for a, b in zip(direct, graphed):
        assert np.array_equal(a, b)


# ------------------------------------------------------------------------------------------------ 9. cloned voice
def test_stream_into_streaming_converter(tmp_path_factory):
    from openvoice_b200.api import ToneColorConverter
    from openvoice_b200.streaming import StreamingConverter
    tts = engine(tmp_path_factory, "f16x3")
    cfg = tmp_path_factory.mktemp("vc") / "config.json"
    cfg.write_text(json.dumps(O.DEFAULT_HPARAMS))
    conv = ToneColorConverter(str(cfg), device="cuda:0", enable_watermark=False)
    conv.model.load_state_dict(O.synthetic_state_dict(1234))
    gen = torch.Generator().manual_seed(9)
    src, tgt = 0.1 * torch.randn(1, 256, 1, generator=gen), 0.1 * torch.randn(1, 256, 1, generator=gen)
    ids = sentences(3, 70, long_first=True)
    sc = StreamingConverter(conv, src, tgt, tau=0.3, window_frames=128, request_seed=21)
    outs = [sc.push(c) for c in tts.tts_stream(ids=ids, speaker="default", seed=5)]
    outs.append(sc.flush())
    got = np.concatenate(outs)
    whole = tts.audio_numpy_concat(tts.tts_from_ids(ids, "default", seed=5), 22050)
    ref = conv.convert(whole, src, tgt, tau=0.3, seed=21)
    assert got.shape == ref.shape
    err = rel_err(got, ref)
    print(f"tts_stream -> StreamingConverter vs convert(tts): max|d|/rms = {err:.2e}")
    assert err <= 1e-4
