"""-m gpu: duration fit (include/ovc.h: ovc_tts_encode_fit), in fp32 and f16x3.  The device's scale against the host
statement of the rule (g++ build of ovc_tts_ops.h) on the device's own logw and exp, bit for bit; a fitted encode
against an unfitted one given the fitted scales; the fixtures of oracle/make_golden_tts_fit.py; the length rule of
tts_batch; unfitted requests beside fitted ones; streaming; CloneSessions.say(duration=); the launches."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import tts_fit_oracle as FO
from oracle import tts_oracle as T
from test_gpu_clone import models, rel_err, requests
from test_tts_fit_host import CASES, hc, host_fit  # noqa: F401  (hc: the g++ build of the rule, a fixture)

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(params=["fp32", "f16x3"])
def pair(request, tmp_path_factory):
    return models(tmp_path_factory, request.param)


def tokens(lengths, seed=3):
    rng = np.random.default_rng(seed)
    x = torch.zeros(len(lengths), max(lengths), dtype=torch.int64)
    for b, n in enumerate(lengths):
        x[b, :n] = torch.from_numpy(rng.integers(1, T.TTS_HPARAMS["n_vocab"], n))
    return x, torch.tensor(lengths)


def encode(m, x, lens, **kw):
    B = len(lens)
    return m.tts_encode(x, lens, sid=torch.tensor([b % 3 for b in range(B)]), seeds=[5 + b for b in range(B)],
                        streams=list(range(B)), noise_scale=0.667, noise_scale_w=0.6, sdp_ratio=0.2, **kw)


def device_logw(m, x, lens, **kw):
    """(y_lengths, logw, scale) of the native encode with the same draws as ``encode``."""
    B = len(lens)
    a = m._tts_args(x, lens, torch.tensor([b % 3 for b in range(B)]), 0.667, kw.pop("length_scale", 1.0), 0.6, 0.2,
                    None, [5 + b for b in range(B)], list(range(B)))
    return m.native.tts_encode(a["x"], a["x_lengths"], a["sid"], seed=a["seed"], items=a["enc_items"], **kw,
                               **a["enc_scalars"])


def check_groups(hc, m, x, lens, fit):  # noqa: F811
    from openvoice_b200.api import fit_groups
    y, _, logw, scale = device_logw(m, x, lens, fit=fit_groups(fit, len(lens), m.device))
    e = torch.exp(logw).cpu().numpy()                  # the device's own expf, as the kernel evaluates it
    scale, y, L = scale.cpu().numpy(), y.cpu().numpy(), lens.numpy()
    for r0, r1, target in fit:
        s = host_fit(hc, e[r0:r1], L[r0:r1], target)
        assert s == FO.fit_scale(e[r0:r1], L[r0:r1], target)
        assert (scale[r0:r1] == s).all(), (r0, r1, target, scale[r0:r1], s)
        assert y[r0:r1].sum() == FO.group_frames(e[r0:r1], L[r0:r1], s)
    return scale, y


def test_device_scale_is_the_host_rule(pair, hc):  # noqa: F811
    m = pair[0].model
    rng = np.random.default_rng(5)
    lengths = rng.integers(5, 140, 24).tolist()
    x, lens = tokens(lengths)
    y1 = device_logw(m, x, lens)[0].cpu().numpy()
    fit, b = [], 0
    while b < 24:                                       # groups of 1-4 rows, gaps between some of them
        n = int(rng.integers(1, 5))
        if b + n > 24:
            break
        fit.append((b, b + n, max(1, int(y1[b:b + n].sum() * rng.uniform(0.3, 3.5)))))
        b += n + int(rng.integers(0, 2))
    fit[-1] = (fit[-1][0], fit[-1][1], int(y1[fit[-1][0]:fit[-1][1]].sum()) * 9)   # clamps at the top
    scale, _ = check_groups(hc, m, x, lens, fit)
    assert scale[fit[-1][0]] == np.float32(FO.SCALE_HI)
    covered = np.zeros(24, bool)
    for r0, r1, _ in fit:
        covered[r0:r1] = True
    assert (scale[~covered] == 1.0).all()
    # a request far longer than the CTA: 2700 tokens in one row, and beside a short one
    x, lens = tokens([2700, 40], seed=9)
    y1 = device_logw(m, x, lens)[0].cpu().numpy()
    check_groups(hc, m, x, lens, [(0, 2, int(y1.sum() * 0.7))])
    check_groups(hc, m, x, lens, [(0, 1, int(y1[0] * 1.6)), (1, 2, 3)])


def test_fitted_encode_equals_the_encode_at_its_scales(pair):
    m = pair[0].model
    x, lens = tokens([37, 12, 60, 25, 80])
    y1 = encode(m, x, lens).frames
    fit = [(0, 2, int((y1[0] + y1[1]) * 1.4)), (3, 5, int((y1[3] + y1[4]) * 0.6))]
    st = encode(m, x, lens, fit=fit)
    assert st.length_scale[2] == 1.0 and st.length_scale[0] == st.length_scale[1] != 1.0
    ref = encode(m, x, lens, length_scale=st.length_scale)
    assert ref.length_scale is None and st.frames == ref.frames
    for a, b in ((st.stats, ref.stats), (st.cum, ref.cum), (st.g, ref.g), (st.y_lengths, ref.y_lengths)):
        assert torch.equal(a, b)
    # w_ceil and logw of the native calls, and the audio of whole-row windows
    from openvoice_b200.api import fit_groups
    got = device_logw(m, x, lens, fit=fit_groups(fit, 5, m.device))
    want = device_logw(m, x, lens, length_scale=st.length_scale)
    for a, b in zip(got[:3], want[:3]):
        assert torch.equal(a, b)
    wins = [(b, 0, st.frames[b]) for b in range(5)]
    o1 = m.tts_decode_windows(st, wins)[0].clone()
    o2 = m.tts_decode_windows(ref, wins)[0]
    assert torch.equal(o1, o2)
    o3, f3 = m.infer_ragged(x, lens, sid=torch.tensor([b % 3 for b in range(5)]), seeds=[5 + b for b in range(5)],
                            streams=list(range(5)), noise_scale=0.667, noise_scale_w=0.6, sdp_ratio=0.2, fit=fit)
    o4, f4 = m.infer_ragged(x, lens, sid=torch.tensor([b % 3 for b in range(5)]), seeds=[5 + b for b in range(5)],
                            streams=list(range(5)), noise_scale=0.667, noise_scale_w=0.6, sdp_ratio=0.2,
                            length_scale=st.length_scale)
    assert f3 == f4 == st.frames and torch.equal(o3, o4)


@pytest.mark.parametrize("name", CASES)
def test_fixtures(name, pair):
    m = pair[0].model
    d = np.load(os.path.join(GOLD, name + ".npz"))
    c = json.loads(str(d["meta"]))
    x, lens, sid, noise_w = T.synthetic_tts_inputs(c["B"], c["T"], c["seed"], c["lengths"])
    noise = torch.randn(c["B"], 192, 40 * c["T"] + 64, generator=torch.Generator().manual_seed(30_000 + c["seed"]))
    dev = m.device
    fit = [torch.tensor(col, dtype=torch.int64, device=dev) for col in d["fit"].T.tolist()]
    y, w_ceil, logw, scale = m.native.tts_encode(x.to(dev), lens.to(dev), sid.to(dev), noise_w=noise_w.to(dev),
                                                 noise_scale_w=c["noise_scale_w"], length_scale=c["unfitted_scale"],
                                                 sdp_ratio=c["sdp_ratio"], fit=(*fit, FO.SCALE_LO, FO.SCALE_HI))
    y, scale = y.cpu().numpy(), scale.cpu().numpy()
    assert np.array_equal(y, d["y_lengths"])
    assert np.array_equal(w_ceil.cpu().numpy(), d["w_ceil"])
    # s* = k / exp(logw) of the token that reaches the target, so it moves with that token's logw: the device's scale
    # is within the largest logw difference of its group (plus 1e-6) of the reference's
    dlogw = np.abs(logw.cpu().numpy().astype(np.float64) - d["logw"])
    for r0, r1, _ in d["fit"]:
        ds = np.abs(scale[r0:r1].astype(np.float64) / d["scale"][r0:r1] - 1).max()
        print(f"{name}: scale {float(scale[r0])!r} vs {float(d['scale'][r0])!r}: rel {ds:.2e}, "
              f"max|dlogw| {dlogw[r0:r1].max():.2e}")
        assert ds <= dlogw[r0:r1].max() + 1e-6, (ds, dlogw[r0:r1].max())
    Ty = int(y.max())
    o, _ = m.native.tts_decode(c["B"], Ty, dev, noise=noise[:, :, :Ty].to(dev), noise_scale=c["noise_scale"],
                               ragged=True)
    o = o[:, 0].cpu().numpy()
    hop = o.shape[1] // Ty
    for b in range(c["B"]):
        n = y[b] * hop
        err = rel_err(o[b, :n], d["o"][b, :n])
        print(f"{name} row {b}: scale {float(scale[b]):.7f}, max|d|/rms {err:.2e}")
        assert err <= 1e-4, (name, b, err)


def fit_requests():
    reqs = requests(5)
    durations = [2.4, None, 6.0, None, 3.0]
    for q, dur in zip(reqs, durations):
        if dur is not None:
            q["duration"] = dur
    return reqs


def test_length_rule_and_unfitted_neighbours(pair):
    tts = pair[0]
    sr, hop = int(tts.hps.data.sampling_rate), int(tts.hps.data.hop_length)
    reqs = fit_requests()
    out = tts.tts_batch(reqs)
    plain = tts.tts_batch([q for q in reqs if "duration" not in q])
    k = 0
    for q, a in zip(reqs, out):
        if "duration" not in q:
            assert np.array_equal(a, plain[k])
            k += 1
            continue
        want = int(round(q["duration"] * sr))
        assert want <= len(a) < want + hop, (q["duration"], len(a), want)
        alone = tts.tts_batch([q])[0]
        assert np.array_equal(a, alone)                 # fitted requests do not depend on their neighbours either


def test_stream_concatenates_to_the_batch(pair):
    tts = pair[0]
    reqs = fit_requests()
    whole = tts.tts_batch(reqs)
    parts = [[] for _ in reqs]
    for r, c in tts.tts_stream_batch(reqs, window_frames=64, first_window_frames=16):
        parts[r].append(c)
    for r, a in enumerate(whole):
        got = np.concatenate(parts[r])
        assert got.shape == a.shape and rel_err(got, a) <= 2e-6, r


def test_single_request_entry_points(pair):
    tts = pair[0]
    sr, hop = int(tts.hps.data.sampling_rate), int(tts.hps.data.hop_length)
    q = fit_requests()[0]
    a = tts.tts_batch([q])[0]
    ids = q["ids"]
    b = np.concatenate(list(tts.tts_stream(ids=ids, speaker=q["speaker"], speed=q["speed"], seed=q["seed"],
                                           duration=q["duration"], window_frames=64, first_window_frames=16)))
    assert b.shape == a.shape
    speech = tts.tts_from_ids(ids, q["speaker"], speed=q["speed"], noise_scale=q["noise_scale"], seed=q["seed"],
                              duration=1.5)
    n = sum(len(s) for s in speech)
    assert int(round(1.5 * sr)) <= n < int(round(1.5 * sr)) + hop


def test_say_equals_the_one_shot_stream(pair):
    from openvoice_b200.streaming import CloneSessions
    tts, conv = pair
    W, W1 = 64, 16
    reqs = fit_requests()[:3]
    cs = CloneSessions(conv, tts, window_frames=W, first_window_frames=W1)
    keys = ("speaker", "src_se", "tgt_se", "tau", "seed", "convert_seed", "speed", "noise_scale")
    ids = [cs.open(**{k: q[k] for k in keys}) for q in reqs]
    for sid, q in zip(ids, reqs):
        cs.say(sid, ids=q["ids"], duration=q.get("duration"))
        cs.end(sid)
    out = {}
    while cs.sessions:
        for sid, c in cs.step().items():
            out.setdefault(sid, []).append(c)
    for sid, q in zip(ids, reqs):
        got = np.concatenate(out[sid])
        ref = np.concatenate([c for _, c in conv.clone_stream_batch(tts, [q], window_frames=W, first_window_frames=W1)])
        assert got.shape == ref.shape and np.array_equal(got, ref), sid
        whole = conv.clone_batch(tts, [q])[0]
        assert whole.shape == ref.shape and rel_err(ref, whole) <= 1e-4


def test_encode_without_fit_launches_what_it_did(pair):
    m = pair[0].model
    x, lens = tokens([30, 50])
    from openvoice_b200.api import fit_groups
    device_logw(m, x, lens)
    plain = m.native.last_launch_count
    device_logw(m, x, lens, fit=fit_groups([(0, 2, 300)], 2, m.device))
    fitted = m.native.last_launch_count
    device_logw(m, x, lens, fit=None)
    assert m.native.last_launch_count == plain and fitted == plain + 2   # the fit kernel and the second durations pass
