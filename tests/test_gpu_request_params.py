"""-m gpu: per-request seeds and sampling parameters (include/ovc.h: ovc_item_params).  A request's audio depends on
the request alone -- its input, embeddings, parameters and seed -- not on its batch, position, stream, shard or window.
Every comparison here is bit for bit unless it names a bound."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

from oracle import vc_oracle as O

pytestmark = pytest.mark.gpu

LENS = (22050, 30000, 66150, 256 * 7 + 5, 44100, 22050 * 2, 51200, 9999, 70000, 12345, 33333)


def rel_err(got, ref):
    ref = np.asarray(ref, dtype=np.float64)
    return float(np.abs(np.asarray(got, dtype=np.float64) - ref).max() / (np.sqrt((ref ** 2).mean()) + 1e-30))


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


def embeddings(seed):
    gen = torch.Generator().manual_seed(seed)
    return 0.1 * torch.randn(1, 256, 1, generator=gen), 0.1 * torch.randn(1, 256, 1, generator=gen)


def waves(lens, seed):
    rng = np.random.default_rng(seed)
    return [(0.5 * (2 * rng.random(n, dtype=np.float32) - 1)).astype(np.float32) for n in lens]


def items_of(dev, **kw):
    out = {}
    for k, v in kw.items():
        if k == "seed":
            from openvoice_b200.api import seed_array
            out[k] = torch.from_numpy(seed_array(v)).to(dev)
        elif k in ("stream", "frame0"):
            out[k] = torch.tensor(v, dtype=torch.int64, device=dev)
        else:
            out[k] = torch.tensor(v, dtype=torch.float32, device=dev)
    return out


# ------------------------------------------------------------------------------------------------ 1. default path
def test_voice_conversion_default_items_are_bit_identical(native):
    """ovc_voice_conversion_items with items NULL, a struct of NULLs, and arrays spelling out today's defaults equals
    ovc_voice_conversion; so does ovc_convert_waveform_items against ovc_convert_waveform."""
    nat = native.native
    nat.set_option("graph", 0)
    B, T, seed, tau = 3, 70, 4242, 0.3
    spec, lengths, gs, gt, _ = O.synthetic_inputs(B, T, 5, lengths=[70, 41, 64])
    spec, lengths, gs, gt = spec.cuda(), lengths.cuda(), gs.reshape(B, -1).cuda(), gt.reshape(B, -1).cuda()
    lib, p = nat.lib, (lambda t: C.c_void_p(t.data_ptr()))

    def old():
        o = torch.empty(B, 1, 256 * T, device="cuda")
        lat = [torch.empty(B, 192, T, device="cuda") for _ in range(3)]
        rc = lib.ovc_voice_conversion(nat.handle, p(spec), p(lengths), p(gs), p(gt), None, C.c_uint64(seed), C.c_float(tau),
                                      B, T, 1, p(o), p(lat[0]), p(lat[1]), p(lat[2]),
                                      C.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == 0
        return [o] + lat

    ref = old()
    spelled = items_of("cuda", seed=[seed] * B, stream=list(range(B)), frame0=[0] * B, tau=[tau] * B)
    for items in (None, {}, spelled):
        o, lat = nat.voice_conversion(spec, lengths, gs, gt, tau=tau, seed=seed, ragged=True, items=items)
        for a, b in zip([o] + list(lat), ref):
            assert torch.equal(a, b)
    L = 22050
    wav = torch.from_numpy(np.stack([w[:L] for w in waves((L, L), 1)])).cuda()
    wlen = torch.tensor([L, L - 3000], dtype=torch.int64, device="cuda")
    o_old = torch.empty(2, (L // 256) * 256, device="cuda")
    rc = lib.ovc_convert_waveform(nat.handle, p(wav), p(wlen), 2, L, p(gs[:2].contiguous()), p(gt[:2].contiguous()), None,
                                  C.c_uint64(seed), C.c_float(tau), p(o_old), None,
                                  C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    spelled = items_of("cuda", seed=[seed] * 2, stream=[0, 1], frame0=[0, 0], tau=[tau] * 2)
    for items in (None, {}, spelled):
        o, _ = nat.convert_waveform(wav, wlen, gs[:2], gt[:2], tau=tau, seed=seed, items=items)
        assert torch.equal(o, o_old)
    nat.set_option("graph", 1)


# ------------------------------------------------------------------------------------------------ 2. batch invariance
def test_batch_invariance_at_nonzero_tau(conv):
    src, tgt = embeddings(4)
    ws = waves(LENS, 3)
    n = len(ws)
    seeds = [1000 + 17 * i for i in range(n)]
    taus = [(0.0, 0.3, 1.0)[i % 3] for i in range(n)]
    solo = [conv.convert(w, src, tgt, tau=t, seed=s) for w, t, s in zip(ws, taus, seeds)]
    for mb in (3, 64):
        got = conv.convert_batch(ws, src, tgt, tau=taus, seeds=seeds, max_batch=mb)
        for a, b in zip(got, solo):
            assert np.array_equal(a, b), mb
    perm = np.random.default_rng(0).permutation(n)
    got = conv.convert_batch([ws[i] for i in perm], src, tgt, tau=[taus[i] for i in perm], seeds=[seeds[i] for i in perm])
    for j, i in enumerate(perm):
        assert np.array_equal(got[j], solo[i])
    got = conv.convert_concurrent(ws, src, tgt, tau=taus, seeds=seeds, streams=3)
    for a, b in zip(got, solo):
        assert np.array_equal(a, b)
    other = conv.convert(ws[1], src, tgt, tau=0.3, seed=seeds[1] + 1)
    assert taus[1] == 0.3 and not np.array_equal(other, solo[1])


def test_sharded_async_follows_seeds(tmp_path_factory):
    from openvoice_b200 import distributed as D
    conv = converter(tmp_path_factory, "f16x3")
    src, tgt = embeddings(3)
    ws = waves((22050, 9000, 30011, 4096), 31)
    seeds = [5, 2 ** 64 - 1, 77, 2 ** 33]
    solo = [conv.convert(w, src, tgt, tau=0.3, seed=s) for w, s in zip(ws, seeds)]
    res = D.convert_sharded_async(conv, ws, src, tgt, tau=0.3, seeds=seeds, copy=True).result()
    for a, b in zip(res, solo):
        assert np.array_equal(a, b)


# ------------------------------------------------------------------------------------------------ 3. windows, streams
def test_long_clip_and_streaming_with_request_seed(conv):
    from openvoice_b200.streaming import StreamingConverter
    src, tgt = embeddings(8)
    L = 22050 * 14 + 123
    wav = waves((L,), 11)[0]
    whole = conv.convert(wav, src, tgt, tau=0.3, seed=99)
    tiled = conv.convert_long(wav, src, tgt, tau=0.3, seed=99, window_frames=300)
    assert tiled.shape == whole.shape and rel_err(tiled, whole) <= 2e-6
    short = wav[: 256 * 90]
    assert np.array_equal(conv.convert_long(short, src, tgt, tau=0.3, seed=99, window_frames=2048),
                          conv.convert(short, src, tgt, tau=0.3, seed=99))
    Ls = 22050 * 9 + 77
    whole = conv.convert(wav[:Ls], src, tgt, tau=0.3, seed=7)
    for W, sizes in ((200, [100, 7000, 33, 66150, 12000, 256, 90001]), (64, [4096] * 60)):
        sc = StreamingConverter(conv, src, tgt, tau=0.3, window_frames=W, request_seed=7)
        outs, pos, i = [], 0, 0
        while pos < Ls:
            k = min(sizes[i % len(sizes)], Ls - pos)
            outs.append(sc.push(wav[pos: pos + k]))
            pos, i = pos + k, i + 1
        outs.append(sc.flush())
        stream = np.concatenate(outs)
        assert stream.shape == whole.shape and rel_err(stream, whole) <= 2e-6, W
        assert sc.noise.numel() == 0


def test_in_kernel_draws_equal_explicit_philox_noise(native):
    """voice_conversion keyed per item (mixed seeds, streams, frame offsets) == the same call given the stacked
    ovc_philox_normals tensors as explicit noise: o_hat and all three latents."""
    from openvoice_b200._native import philox_normals
    nat = native.native
    B, T = 3, 70
    spec, lengths, gs, gt, _ = O.synthetic_inputs(B, T, 6, lengths=[70, 41, 64])
    spec, lengths, gs, gt = spec.cuda(), lengths.cuda(), gs.cuda(), gt.cuda()
    seeds, streams, frame0, taus = [3, 2 ** 64 - 2, 3], [0, 5, 1], [0, 1000, 2 ** 32 - 70], [0.3, 1.0, 0.6]
    o, lat = nat.voice_conversion(spec, lengths, gs, gt, tau=0.0, seed=0, ragged=True,
                                  items=items_of("cuda", seed=seeds, stream=streams, frame0=frame0, tau=taus))
    noise = torch.stack([philox_normals(s, st, 0, 192, f, T) for s, st, f in zip(seeds, streams, frame0)])
    o2, lat2 = nat.voice_conversion(spec, lengths, gs, gt, noise=noise, tau=0.0, seed=0, ragged=True,
                                    items=items_of("cuda", tau=taus))
    assert torch.equal(o, o2)
    for a, b in zip(lat, lat2):
        assert torch.equal(a, b)
    # today's default draw is the same function at (seed; b, c, t)
    o3, lat3 = nat.voice_conversion(spec, lengths, gs, gt, tau=0.3, seed=11, ragged=True)
    noise = torch.stack([philox_normals(11, b, 0, 192, 0, T) for b in range(B)])
    o4, lat4 = nat.voice_conversion(spec, lengths, gs, gt, noise=noise, tau=0.3, ragged=True)
    assert torch.equal(o3, o4) and torch.equal(lat3[0], lat4[0])


# ------------------------------------------------------------------------------------------------ 4. graph replay
def test_graph_replay_follows_new_seeds_and_taus(tmp_path_factory):
    conv = converter(tmp_path_factory, "f16x3")
    nat = conv.model.native
    src, tgt = embeddings(2)
    ws = waves((30000, 22050, 26000), 5)
    calls = [([1, 2, 3], [0.3, 0.0, 1.0]), ([4, 5, 6], [1.0, 0.3, 0.3]), ([7, 8, 9], [0.5, 0.5, 0.0]),
             ([1, 2, 3], [0.3, 0.0, 1.0])]
    nat.set_option("graph", 0)
    direct = [conv.convert_batch(ws, src, tgt, tau=t, seeds=s) for s, t in calls]
    nat.set_option("graph", 1)
    before = nat.graph_replays
    graphed = [conv.convert_batch(ws, src, tgt, tau=t, seeds=s) for s, t in calls]
    assert nat.graph_replays - before >= 2
    for d, g in zip(direct, graphed):
        for a, b in zip(d, g):
            assert np.array_equal(a, b)
    assert not np.array_equal(direct[0][0], direct[1][0])


# ------------------------------------------------------------------------------------------------ 6. TTS
@pytest.fixture(scope="module")
def tts():
    from conftest import get_native_tts
    return get_native_tts()


def test_tts_default_items_are_bit_identical(tts):
    from oracle import tts_oracle as T
    nat = tts.native
    tokens, lengths, sid, _ = T.synthetic_tts_inputs(3, 40, 11, [40, 33, 9])
    tokens, lengths, sid = tokens.cuda(), lengths.cuda(), sid.cuda()
    kw = dict(seed=7, noise_scale_w=0.6, length_scale=1.1, sdp_ratio=0.2)
    ref = nat.tts_encode(tokens, lengths, sid, **kw)
    Ty = int(ref[0].max())
    ref_o = nat.tts_decode(3, Ty, "cuda", seed=8, noise_scale=0.667, ragged=True, latents=True)
    spelled_e = items_of("cuda", seed=[7] * 3, stream=[0, 1, 2], noise_scale_w=[0.6] * 3, length_scale=[1.1] * 3,
                         sdp_ratio=[0.2] * 3, frame0=[0] * 3, tau=[0.3] * 3)
    spelled_d = items_of("cuda", seed=[8] * 3, stream=[0, 1, 2], noise_scale=[0.667] * 3)
    for ie, idd in ((None, None), ({}, {}), (spelled_e, spelled_d)):
        got = nat.tts_encode(tokens, lengths, sid, items=ie, **kw)
        for a, b in zip(got, ref):
            assert torch.equal(a, b)
        o, lat = nat.tts_decode(3, Ty, "cuda", seed=8, noise_scale=0.667, ragged=True, latents=True, items=idd)
        assert torch.equal(o, ref_o[0]) and torch.equal(lat[0], ref_o[1][0]) and torch.equal(lat[1], ref_o[1][1])


def test_tts_in_kernel_draws_equal_explicit_noise(tts):
    from openvoice_b200._native import philox_normals
    from oracle import tts_oracle as T
    nat = tts.native
    B, Tn = 3, 40
    tokens, lengths, sid, _ = T.synthetic_tts_inputs(B, Tn, 12, [40, 20, 31])
    tokens, lengths, sid = tokens.cuda(), lengths.cuda(), sid.cuda()
    seeds, streams = [9, 2 ** 64 - 1, 9], [2, 0, 7]
    nsw, ls, sr, ns = [0.6, 0.8, 0.3], [1.0, 1 / 0.8, 1 / 1.3], [0.2, 0.5, 0.0], [0.667, 0.3, 1.0]
    ie = items_of("cuda", seed=seeds, stream=streams, noise_scale_w=nsw, length_scale=ls, sdp_ratio=sr)
    a = nat.tts_encode(tokens, lengths, sid, items=ie)
    noise_w = torch.stack([torch.cat([philox_normals(s, st, 0x7700, 1, 0, Tn), philox_normals(s, st, 0x7701, 1, 0, Tn)])
                           for s, st in zip(seeds, streams)])
    b = nat.tts_encode(tokens, lengths, sid, noise_w=noise_w,
                       items=items_of("cuda", noise_scale_w=nsw, length_scale=ls, sdp_ratio=sr))
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    Ty = int(a[0].max())
    dk = [(s + 1) % 2 ** 64 for s in seeds]
    o1, l1 = nat.tts_decode(B, Ty, "cuda", ragged=True, latents=True,
                            items=items_of("cuda", seed=dk, stream=streams, noise_scale=ns))
    noise = torch.stack([philox_normals(s, st, 0, 192, 0, Ty) for s, st in zip(dk, streams)])
    o2, l2 = nat.tts_decode(B, Ty, "cuda", noise=noise, ragged=True, latents=True, items=items_of("cuda", noise_scale=ns))
    assert torch.equal(o1, o2) and torch.equal(l1[1], l2[1])
    # the statistics of per-item keys: plausible normals, equal keys give equal draws, different keys do not
    big = philox_normals(2 ** 63 + 5, 3, 0, 192, 2 ** 32 - 1000, 4000)
    assert abs(float(big.mean())) < 0.01 and abs(float(big.std()) - 1.0) < 0.01
    assert torch.equal(noise_w[0, :, :20], philox_normals(9, 2, 0x7700, 2, 0, 20))
    assert not torch.equal(noise_w[0], noise_w[2])
    assert torch.equal(big[:, 1000:], philox_normals(2 ** 63 + 5, 3, 0, 192, 0, 3000))    # the frame counter wraps


def test_tts_batch_equals_each_request_alone(tmp_path):
    import copy
    from oracle import tts_oracle as T
    from openvoice_b200.api import BaseSpeakerTTS
    hp = copy.deepcopy(O.DEFAULT_HPARAMS)
    hp["data"]["n_speakers"] = T.TTS_HPARAMS["n_speakers"]
    hp["speakers"] = {"default": 1, "whispering": 2}
    (tmp_path / "config.json").write_text(json.dumps(hp))
    torch.save({"model": T.synthetic_tts_state_dict()}, tmp_path / "checkpoint.pth")
    eng = BaseSpeakerTTS(str(tmp_path / "config.json"), device="cuda:0")
    eng.load_ckpt(str(tmp_path / "checkpoint.pth"))
    rng = np.random.default_rng(4)
    nv = eng.model.native.tts_info()["n_vocab"]

    def sents(k):
        return [rng.integers(0, nv, int(rng.integers(5, 40))).tolist() for _ in range(k)]
    reqs = [dict(ids=sents(1), speaker="default", speed=0.8, seed=1),
            dict(ids=sents(4), speaker="whispering", speed=1.0, seed=2 ** 64 - 1, noise_scale=0.3, sdp_ratio=0.5),
            dict(ids=sents(2), speaker=0, speed=1.3, seed=2, noise_scale_w=0.9),
            dict(ids=sents(3), speaker="default", speed=1.0, seed=1, noise_scale=1.0, noise_scale_w=0.2)]
    got = eng.tts_batch(reqs)
    assert len(got) == len(reqs)
    for q, a in zip(reqs, got):
        kw = {k: q[k] for k in ("noise_scale", "noise_scale_w", "sdp_ratio") if k in q}
        parts = eng.tts_from_ids(q["ids"], q["speaker"], speed=q["speed"], seed=q["seed"], **kw)
        assert np.array_equal(a, eng.audio_numpy_concat(parts, 22050, q["speed"]))
    # durations: y_lengths / w_ceil of the mixed batch equal each request's own
    q = reqs[1]
    x = [s for r in reqs for s in r["ids"]]
    Tn = max(len(s) for s in x)
    tok = torch.zeros(len(x), Tn, dtype=torch.int64)
    for i, s in enumerate(x):
        tok[i, : len(s)] = torch.tensor(s)
    lens = torch.tensor([len(s) for s in x])
    _, attn, y_mask, _ = eng.model.infer(tok, lens, sid=torch.tensor([2] * len(x)), seeds=[q["seed"]] * len(x),
                                         streams=list(range(len(x))), length_scale=[1.0] * len(x), ragged=True,
                                         latents=False)
    _, attn1, y_mask1, _ = eng.model.infer(tok[:1, : len(x[0])], lens[:1], sid=torch.tensor([2]), seed=q["seed"],
                                           ragged=True, latents=False)
    assert np.array_equal(y_mask[0, 0].sum().cpu().numpy(), y_mask1[0, 0].sum().cpu().numpy())
    assert np.array_equal(attn[0, 0, :, : len(x[0])].sum(0).cpu().numpy(), attn1[0, 0].sum(0).cpu().numpy())
