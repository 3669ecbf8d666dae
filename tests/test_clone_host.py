"""CPU checks of the text-to-cloned-voice join: the ovc_splice element rules (openvoice_b200/csrc/ovc_splice.h, compiled
with g++ through tests/hostcheck/splice_host.cpp) against a NumPy model, the PCM16 round trip against a real 16-bit
wav, the host-side planning against ``audio_numpy_concat``, the request checks of ``clone_batch`` /
``clone_stream_batch`` with stand-in models, and the ptxas report of the splice kernel."""
import copy
import ctypes as C
import os
import re
import shutil
import subprocess
import types

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LL = C.c_longlong


@pytest.fixture(scope="module")
def sp(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("hostcheck") / "splice_host.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, os.path.join(HERE, "hostcheck", "splice_host.cpp")])
    return C.CDLL(so)


# ------------------------------------------------------------------------------------------------ NumPy model
def q16(x):
    """include/ovc.h OVC_SPLICE_PCM16: rint_even(fl32(x * 32767)) saturated to int16, / 32768 (NaN: 0)."""
    y = np.asarray(x, np.float32) * np.float32(32767.0)
    y = np.where(np.isnan(y), np.float32(0), y)
    q = np.clip(np.rint(y), -32768, 32767).astype(np.int16)
    return q.astype(np.float32) / np.float32(32768.0), q


def clamp_seg(v, src_rows, src_pitch, dst_rows, dst_cap):
    sr, so, n, dr, do = (int(a) for a in v)
    dr = min(max(dr, 0), dst_rows - 1)
    do = do % dst_cap
    n = min(max(n, 0), dst_cap)
    if sr < 0 or src_rows < 1:
        sr, so = -1, 0
    else:
        sr, so = min(sr, src_rows - 1), min(max(so, 0), src_pitch)
        n = min(n, src_pitch - so)
    return sr, so, n, dr, do


def np_splice(src, dst, seg, pcm16=False):
    src_rows, src_pitch = src.shape
    dst_rows, cap = dst.shape
    out = dst.copy()
    for v in seg:
        sr, so, n, dr, do = clamp_seg(v, src_rows, src_pitch, dst_rows, cap)
        vals = np.zeros(n, np.float32) if sr < 0 else src[sr, so:so + n]
        out[dr, (do + np.arange(n)) % cap] = q16(vals)[0] if pcm16 and sr >= 0 else vals
    return out


def run(sp, src, dst, seg, pcm16=False):
    src = np.ascontiguousarray(src, np.float32)
    out = np.ascontiguousarray(dst, np.float32).copy()
    seg = np.ascontiguousarray(seg, np.int64).reshape(-1, 5)
    sp.sp_run(src.ctypes.data_as(C.c_void_p), LL(src.shape[0]), LL(src.shape[1]), out.ctypes.data_as(C.c_void_p),
              LL(out.shape[0]), LL(out.shape[1]), seg.ctypes.data_as(C.c_void_p), len(seg), 1 if pcm16 else 0)
    return out


def random_segments(rng, S, src_rows, src_pitch, dst_rows, cap, gap_share=0.3):
    """In-range segments, some gaps, some wrapping past the ring's end; destinations do not overlap (one per row)."""
    seg = []
    for s in range(S):
        n = int(rng.integers(0, min(src_pitch, cap) + 1))
        r = -1 if rng.random() < gap_share else int(rng.integers(0, src_rows))
        seg.append((r, int(rng.integers(0, src_pitch - n + 1)), n, s % dst_rows, int(rng.integers(0, 4 * cap))))
    return np.asarray(seg, np.int64)


# ------------------------------------------------------------------------------------------------ splice rules
@pytest.mark.parametrize("pcm16", [False, True])
def test_segments_gaps_and_ring_wrap_match_the_model(sp, pcm16):
    rng = np.random.default_rng(3)
    src = rng.uniform(-1.2, 1.2, (7, 300)).astype(np.float32)
    for dst_rows, cap in ((5, 64), (3, 301), (9, 1000)):
        dst = np.full((dst_rows, cap), np.nan, np.float32)
        seg = random_segments(rng, dst_rows, 7, 300, dst_rows, cap)
        got, ref = run(sp, src, dst, seg, pcm16), np_splice(src, dst, seg, pcm16)
        assert np.array_equal(got, ref, equal_nan=True), (dst_rows, cap)
    # a wrapped write: 50 samples from slot 40 of a 64-slot ring land in slots 40..63 then 0..25
    dst = np.zeros((1, 64), np.float32)
    got = run(sp, src, dst, [(2, 10, 50, 0, 64 * 7 + 40)])
    assert np.array_equal(got[0, 40:], src[2, 10:34]) and np.array_equal(got[0, :26], src[2, 34:60])
    assert not got[0, 26:40].any()


def test_clamping_keeps_every_access_in_bounds(sp):
    rng = np.random.default_rng(5)
    src = rng.standard_normal((4, 50)).astype(np.float32)
    big = 2 ** 62
    cases = [(9, 0, 10, 0, 0), (-5, 99, 10, 1, 3), (1, -7, 10, 0, 0), (1, 45, 10, 2, 0), (1, 60, 10, 0, 0),
             (0, 0, -3, 0, 0), (0, 0, 10 ** 9, 0, 0), (0, 0, 20, -4, -5), (0, 0, 20, 99, 2 ** 40 + 3),
             (big, big, big, big, big), (-big, -big, -big, -big, -big), (3, 0, 50, 1, -1)]
    for v in cases:
        o5 = (LL * 5)()
        sp.sp_seg(np.asarray(v, np.int64).ctypes.data_as(C.c_void_p), 0, LL(4), LL(50), LL(3), LL(40), o5)
        assert tuple(o5) == clamp_seg(v, 4, 50, 3, 40), v
        sr, so, n, dr, do = tuple(o5)
        assert 0 <= n <= 40 and 0 <= dr < 3 and 0 <= do < 40
        assert sr == -1 or (0 <= sr < 4 and 0 <= so and so + n <= 50)
    dst = np.full((3, 40), 7.0, np.float32)
    assert np.array_equal(run(sp, src, dst, cases), np_splice(src, dst, np.asarray(cases)))
    # no source rows: every segment is a gap
    none = np.zeros((0, 1), np.float32)
    assert np.array_equal(run(sp, none, dst, [(2, 0, 5, 1, 0)]), np_splice(none, dst, [(2, 0, 5, 1, 0)]))


def test_pcm16_values_ties_and_saturation(sp):
    ties = []
    for k in list(range(-32768, -32700)) + list(range(-300, 300)) + list(range(32700, 32767)):
        x = np.float32((k + 0.5) / 32767.0)
        if np.float32(x) * np.float32(32767.0) == np.float32(k + 0.5):      # fl32(x * 32767) is exactly k + 1/2
            ties.append(x)
    ties = np.asarray(ties, np.float32)
    assert len(ties) > 50
    specials = np.asarray([1.0, -1.0, 0.0, -0.0, 1.5, -1.5, 1e30, -1e30, np.inf, -np.inf, np.nan, 1e-9, -1e-9,
                           0.5 / 32767, 32767.5 / 32767], np.float32)
    x = np.concatenate([ties, specials, np.random.default_rng(1).uniform(-1.1, 1.1, 5000).astype(np.float32)])
    y = np.empty_like(x)
    sp.sp_pcm16(x.ctypes.data_as(C.c_void_p), LL(len(x)), y.ctypes.data_as(C.c_void_p))
    ref, q = q16(x)
    assert np.array_equal(y.view(np.int32), ref.view(np.int32))          # bit for bit, signed zeros included
    # ties round to the even integer
    t = q[: len(ties)].astype(np.int64)
    assert (t % 2 == 0).all() and (np.abs(t - (ties * np.float32(32767.0)).astype(np.float64)) == 0.5).all()
    assert y[len(ties)] == np.float32(32767 / 32768) and y[len(ties) + 1] == np.float32(-32767 / 32768)
    assert y[len(ties) + 4] == np.float32(32767 / 32768) and y[len(ties) + 5] == -1.0 and y[len(ties) + 10] == 0.0


def test_pcm16_equals_a_16_bit_wav_round_trip(tmp_path):
    from scipy.io import wavfile
    from openvoice_b200.api import _load_audio
    x = np.random.default_rng(2).uniform(-1.05, 1.05, 22050).astype(np.float32)
    x[:4] = [1.0, -1.0, 0.5 / 32767, 0.0]
    ref, q = q16(x)
    path = str(tmp_path / "tmp.wav")
    wavfile.write(path, 22050, q)
    back = _load_audio(path, 22050)
    assert back.dtype == np.float32 and np.array_equal(back, ref)


# ------------------------------------------------------------------------------------------------ planning
def test_plan_and_table_give_audio_numpy_concat(sp):
    from openvoice_b200.api import BaseSpeakerTTS, plan_clone, splice_table
    rng = np.random.default_rng(11)
    hop, sr = 256, 22050
    for trial in range(20):
        n_req = int(rng.integers(1, 6))
        owner = sorted(int(v) for v in rng.integers(0, n_req, int(rng.integers(n_req, 3 * n_req + 1))))
        owner = sorted(set(range(n_req)) | set(owner)) if trial % 2 else list(range(n_req)) + owner
        speeds = [float(rng.choice([0.5, 0.9, 1.0, 1.3, 2.0, 3.7])) for _ in range(n_req)]
        frames = [int(v) for v in rng.integers(1, 40, len(owner))]
        o = rng.standard_normal((len(owner), hop * max(frames))).astype(np.float32)
        runs, lengths = plan_clone(frames, owner, speeds, hop, sr)
        ref = [BaseSpeakerTTS.audio_numpy_concat([o[i, : hop * frames[i]] for i, r in enumerate(owner) if r == q], sr,
                                                 speed=speeds[q]) for q in range(n_req)]
        assert lengths == [len(a) for a in ref]
        pitch = max(lengths) + int(rng.integers(0, 300))
        table = splice_table(runs, pitch)
        assert table.dtype == np.int64 and table.shape[1] == 5
        dst = np.full((n_req, pitch), np.nan, np.float32)
        got = run(sp, o, dst, table)
        assert np.array_equal(got, np_splice(o, dst, table))
        for q in range(n_req):
            assert np.array_equal(got[q, : lengths[q]], ref[q]) and not got[q, lengths[q]:].any(), (trial, q)


# ------------------------------------------------------------------------------------------------ request checks
def _stub_models(tts_sr=22050, device=0):
    """A BaseSpeakerTTS and a ToneColorConverter that never touched a device; their native objects record calls."""
    from oracle import tts_oracle as T
    from oracle import vc_oracle as O
    from openvoice_b200.api import BaseSpeakerTTS, ToneColorConverter
    from openvoice_b200.utils import HParams
    calls = []

    class Native:
        def __getattr__(self, name):
            return lambda *a, **k: calls.append(name)

    hp = copy.deepcopy(O.DEFAULT_HPARAMS)
    hp["data"]["n_speakers"] = T.TTS_HPARAMS["n_speakers"]
    hp["data"]["sampling_rate"] = tts_sr
    tts = BaseSpeakerTTS.__new__(BaseSpeakerTTS)
    tts.hps = HParams(**hp)
    tts.text_frontend = None

    def infer_ragged(x, lens, sid=None, **kw):                 # an encode whose sentences all come out 1 frame long
        calls.append("infer_ragged")
        return None, [1] * x.shape[0]

    def tts_encode(x, lens, sid=None, **kw):
        calls.append("tts_encode")
        return types.SimpleNamespace(frames=[1] * x.shape[0])
    tts.model = types.SimpleNamespace(device=torch.device("cuda", device), infer_ragged=infer_ragged,
                                      tts_encode=tts_encode, native=Native())
    conv = ToneColorConverter.__new__(ToneColorConverter)
    conv.hps = HParams(**O.DEFAULT_HPARAMS)
    conv.device = "cuda:0"
    conv.watermark_model = None
    conv.model = types.SimpleNamespace(device=torch.device("cuda", 0), native=Native())
    return tts, conv, calls


def _req(**kw):
    q = dict(ids=[[1, 2, 3, 4], [5, 6]], speaker=0, seed=1, src_se=torch.zeros(1, 256, 1), tgt_se=torch.zeros(1, 256, 1))
    q.update(kw)
    return q


def test_clone_request_refusals_before_any_launch(monkeypatch):
    import openvoice_b200.api as A
    monkeypatch.setattr(A.ToneColorConverter, "_resampled_len", lambda self, n, sr: n)
    tts, conv, calls = _stub_models()
    bad = [dict(src_se=None), dict(tgt_se=None), dict(src_se=torch.zeros(255)), dict(tgt_se=torch.zeros(1, 257, 1)),
           dict(tau=float("nan")), dict(tau=float("inf")), dict(convert_seed=-1), dict(convert_seed=2 ** 64),
           dict(convert_seed=1.5), dict(seed=-3), dict(speed=0.0), dict(ids=[])]
    for kw in bad:
        for call in (lambda r: conv.clone_batch(tts, r), lambda r: conv.clone_stream_batch(tts, r)):
            with pytest.raises(ValueError):
                call([_req(), _req(**kw)])
            assert calls == [], kw
    with pytest.raises(ValueError, match="window_frames"):
        conv.clone_stream_batch(tts, [_req()], window_frames=0)
    tts_other, _, calls_other = _stub_models(device=1)
    for call in (conv.clone_batch, conv.clone_stream_batch):
        with pytest.raises(ValueError, match="cuda:1"):
            call(tts_other, [_req()])
    assert calls == [] and calls_other == []
    assert conv.clone_batch(tts, []) == [] and list(conv.clone_stream_batch(tts, [])) == []
    assert calls == [] and "_dev_cache" not in conv.__dict__ and "_pin_cache" not in conv.__dict__


def test_clone_short_utterance_refused_before_the_conversion(monkeypatch):
    """Every sentence decodes to 1 frame (256 samples): at speed 9 the 1-sentence utterance has 256 + 122 samples, not
    past the STFT padding (384), so both calls stop after the encode, as ``convert`` refuses such audio."""
    import openvoice_b200.api as A
    monkeypatch.setattr(A.ToneColorConverter, "_resampled_len", lambda self, n, sr: n)
    tts, conv, calls = _stub_models()
    with pytest.raises(ValueError, match="request 1"):
        conv.clone_batch(tts, [_req(), _req(ids=[[1, 2]], speed=9.0)])
    assert calls == ["infer_ragged"]
    with pytest.raises(ValueError, match="request 1"):
        conv.clone_stream_batch(tts, [_req(), _req(ids=[[1, 2]], speed=9.0)])
    assert calls == ["infer_ragged", "tts_encode"]
    tts48, conv48, calls48 = _stub_models(tts_sr=48000)
    with pytest.raises(ValueError, match="48000"):
        conv48.clone_stream_batch(tts48, [_req()])
    assert calls48 == []


# ------------------------------------------------------------------------------------------------ ptxas
def test_splice_kernel_does_not_spill(tmp_path):
    """-Xptxas -v report of the library's translation unit: the splice kernel uses no stack and spills nothing."""
    log = os.path.join(ROOT, "openvoice_b200", "csrc", "build", "ovc_lib.ptxas.log")
    src = os.path.join(ROOT, "openvoice_b200", "csrc", "ovc_lib.cu")
    if os.path.exists(log) and os.path.getmtime(log) >= os.path.getmtime(os.path.join(ROOT, "openvoice_b200", "csrc",
                                                                                      "ovc_splice.h")):
        text = open(log).read()
    else:
        nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
        if not os.path.exists(nvcc):
            pytest.skip("no nvcc")
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                            "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "lib.o")],
                           capture_output=True, text=True, cwd=os.path.dirname(src))
        assert r.returncode == 0, r.stderr[-3000:]
        text = r.stderr
    m = re.search(r"Compiling entry function '(_ZN6ovc_sp13splice_kernel\w*)' for 'sm_90a'\n(?:ptxas info[^\n]*\n)*?"
                  r"\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", text)
    assert m, "splice_kernel not in the ptxas report"
    assert (int(m.group(2)), int(m.group(3)), int(m.group(4))) == (0, 0, 0), m.group(0)
