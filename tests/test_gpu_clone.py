"""-m gpu: text to cloned voice joined on the device.  ``ovc_splice`` against the NumPy model of tests/test_clone_host.py,
``ToneColorConverter.clone_batch`` against the two-step ``tts_batch`` -> ``convert`` path (bit for bit), and
``clone_stream_batch`` against ``clone_batch`` (within 1e-4 of the rms), in fp32 and f16x3."""
import copy
import json

import numpy as np
import pytest
import torch

from oracle import tts_oracle as T
from oracle import vc_oracle as O
from test_clone_host import np_splice, q16, random_segments

pytestmark = pytest.mark.gpu

_models = {}


def models(tmp_path_factory, precision, conv_sr=None):
    """(BaseSpeakerTTS, ToneColorConverter) on synthetic checkpoints; the converter at ``conv_sr`` when given."""
    from openvoice_b200.api import BaseSpeakerTTS, ToneColorConverter
    key = (precision, conv_sr)
    if key not in _models:
        d = tmp_path_factory.mktemp("clone")
        hp = copy.deepcopy(O.DEFAULT_HPARAMS)
        hp["data"]["n_speakers"] = T.TTS_HPARAMS["n_speakers"]
        hp["speakers"] = {"default": 1, "whispering": 2}
        (d / "tts.json").write_text(json.dumps(hp))
        torch.save({"model": T.synthetic_tts_state_dict()}, d / "tts.pth")
        tts = BaseSpeakerTTS(str(d / "tts.json"), device="cuda:0", precision=precision)
        tts.load_ckpt(str(d / "tts.pth"))
        hv = copy.deepcopy(O.DEFAULT_HPARAMS)
        if conv_sr is not None:
            hv["data"]["sampling_rate"] = conv_sr
        (d / "vc.json").write_text(json.dumps(hv))
        conv = ToneColorConverter(str(d / "vc.json"), device="cuda:0", enable_watermark=False, precision=precision)
        conv.model.load_state_dict(O.synthetic_state_dict(1234))
        _models[key] = (tts, conv)
    return _models[key]


@pytest.fixture(params=["fp32", "f16x3"])
def pair(request, tmp_path_factory):
    return models(tmp_path_factory, request.param)


def se(seed):
    return 0.1 * torch.randn(1, 256, 1, generator=torch.Generator().manual_seed(seed))


def requests(n=5):
    """Mixed requests: speakers, speeds (0.9 and 1.3 among them), seeds, taus, embeddings and sentence counts."""
    rng = np.random.default_rng(17)
    speakers, speeds, taus = ["default", "whispering", 0, "default", 2], [1.0, 0.9, 1.3, 0.75, 1.1], [0.3, 0.0, 0.6, 1.0, 0.3]
    out = []
    for r in range(n):
        k = 1 + r % 3
        ids = [rng.integers(0, T.TTS_HPARAMS["n_vocab"], int(rng.integers(20, 90))).tolist() for _ in range(k)]
        out.append(dict(ids=ids, speaker=speakers[r % 5], speed=speeds[r % 5], seed=100 + r, src_se=se(2 * r),
                        tgt_se=se(2 * r + 1), tau=taus[r % 5], convert_seed=[7, 2 ** 64 - 1, 0, 12345, 99][r % 5],
                        noise_scale=0.667 if r % 2 else 0.5))
    return out


def two_step(tts, conv, q, pcm16=False, sr=None):
    audio = tts.tts_batch([q])[0]
    if pcm16:
        audio = q16(audio)[0]
    return conv.convert(audio, q["src_se"], q["tgt_se"], tau=q["tau"], seed=q["convert_seed"], sr=sr)


def rel_err(got, ref):
    ref = np.asarray(ref, dtype=np.float64)
    return float(np.abs(np.asarray(got, dtype=np.float64) - ref).max() / (np.sqrt((ref ** 2).mean()) + 1e-30))


# ------------------------------------------------------------------------------------------------ ovc_splice
@pytest.mark.parametrize("pcm16", [False, True])
def test_splice_matches_the_model(pcm16):
    from conftest import get_native_tts
    nat = get_native_tts().native
    rng = np.random.default_rng(8)
    src = rng.uniform(-1.2, 1.2, (6, 5000)).astype(np.float32)
    for dst_rows, cap, S in ((4, 4096, 4), (16, 1000, 16), (3, 9000, 3)):
        dst = rng.standard_normal((dst_rows, cap)).astype(np.float32)
        seg = random_segments(rng, S, 6, 5000, dst_rows, cap)
        ref = np_splice(src, dst, seg, pcm16)
        d = torch.from_numpy(dst).cuda()
        nat.splice(torch.from_numpy(src).cuda(), torch.from_numpy(seg).cuda(), d, pcm16=pcm16)
        assert np.array_equal(d.cpu().numpy(), ref), (dst_rows, cap)
    # a ring write that wraps, then a gap
    d = torch.zeros(2, 700, device="cuda")
    seg = np.asarray([(3, 100, 650, 1, 7 * 700 + 600), (-1, 0, 30, 1, 550)], np.int64)
    nat.splice(torch.from_numpy(src).cuda(), torch.from_numpy(seg).cuda(), d, pcm16=pcm16)
    assert np.array_equal(d.cpu().numpy(), np_splice(src, np.zeros((2, 700), np.float32), seg, pcm16))


# ------------------------------------------------------------------------------------------------ clone_batch
def test_clone_batch_equals_tts_then_convert(pair):
    tts, conv = pair
    reqs = requests()
    refs = [two_step(tts, conv, q) for q in reqs]
    got = conv.clone_batch(tts, reqs)
    for r, (g, ref) in enumerate(zip(got, refs)):
        assert g.dtype == np.float32 and g.shape == ref.shape and np.array_equal(g, ref), r
    order = [3, 0, 4, 2, 1]
    again = conv.clone_batch(tts, [reqs[i] for i in order], max_batch=2)
    for k, i in enumerate(order):
        assert np.array_equal(again[k], refs[i]), i
    alone = conv.clone_batch(tts, [reqs[2]])[0]
    assert np.array_equal(alone, refs[2])


def test_clone_batch_pcm16_equals_converting_the_16_bit_wav(pair):
    tts, conv = pair
    reqs = requests(3)
    got = conv.clone_batch(tts, reqs, pcm16=True)
    for r, q in enumerate(reqs):
        ref = two_step(tts, conv, q, pcm16=True)
        assert np.array_equal(got[r], ref), r
    assert not np.array_equal(got[0], two_step(tts, conv, reqs[0]))


def test_clone_batch_resamples_to_the_converter_rate(tmp_path_factory):
    tts, conv = models(tmp_path_factory, "f16x3", conv_sr=24000)
    reqs = requests(3)
    got = conv.clone_batch(tts, reqs)
    for r, q in enumerate(reqs):
        assert np.array_equal(got[r], two_step(tts, conv, q, sr=22050)), r
    with pytest.raises(ValueError, match="24000"):
        conv.clone_stream_batch(tts, reqs)


# ------------------------------------------------------------------------------------------------ clone_stream_batch
@pytest.mark.parametrize("window_frames,first_window_frames", [(64, 16), (256, 32)])
def test_clone_stream_batch_follows_clone_batch(pair, window_frames, first_window_frames):
    tts, conv = pair
    reqs = requests(5)
    whole = conv.clone_batch(tts, reqs)
    chunks = {r: [] for r in range(len(reqs))}
    order = []
    for r, c in conv.clone_stream_batch(tts, reqs, window_frames=window_frames, first_window_frames=first_window_frames):
        assert c.dtype == np.float32 and len(c) > 0
        chunks[r].append(c)
        order.append(r)
    for r, ref in enumerate(whole):
        got = np.concatenate(chunks[r])
        assert got.shape == ref.shape, (r, got.shape, ref.shape)
        err = rel_err(got, ref)
        print(f"W={window_frames} request {r}: {len(chunks[r])} chunks, max|d|/rms = {err:.2e}")
        assert err <= 1e-4, (r, err)
    # every step yields one chunk per unfinished request: a request that has finished stops yielding
    counts = [len(chunks[r]) for r in range(len(reqs))]
    print(f"W={window_frames} chunks per request: {counts}")
    steps, live, pos = max(counts), list(range(len(reqs))), 0
    for step in range(steps):
        live = [r for r in live if counts[r] > step]
        assert order[pos:pos + len(live)] == live, step
        pos += len(live)
    assert pos == len(order)
