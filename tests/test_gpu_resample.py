"""On-device sample-rate conversion (ovc_resample, ovc_resample.cuh) and the ``sr=`` / ``input_sr`` / ``output_sr``
surface built on it.

The kernel is held to float32(scipy.signal.resample_poly(float64(x))) within one ulp on ragged batches with NaN in
the padding; a batch row, a windowed call and a stream equal the one-shot call bit for bit; every entry point with
``sr=`` equals the same entry point fed the one-shot device resample, bit for bit.  The resampler does not depend on
the conv precision, so these tests use the session converter directly instead of the two-mode ``native`` fixture."""
import numpy as np
import pytest
import torch
from scipy.signal import firwin, resample_poly

from conftest import get_native

pytestmark = pytest.mark.gpu

MODEL_SR = 22050
PAIRS = [(8000, MODEL_SR), (16000, MODEL_SR), (24000, MODEL_SR), (32000, MODEL_SR), (44100, MODEL_SR),
         (48000, MODEL_SR), (96000, MODEL_SR), (192000, MODEL_SR), (MODEL_SR, 44100), (MODEL_SR, 48000)]


def rel_err(got, ref):
    ref = np.asarray(ref, dtype=np.float64)
    got = np.asarray(got, dtype=np.float64)
    return float(np.abs(got - ref).max() / (np.sqrt((ref ** 2).mean()) + 1e-30))


def wave(seed, n):
    rng = np.random.default_rng(int(seed))
    return (0.5 * (2 * rng.random(int(n), dtype=np.float32) - 1)).astype(np.float32)


def updown(a, b):
    g = np.gcd(a, b)
    return b // g, a // g


def ref_poly(x, a, b):
    up, down = updown(a, b)
    return resample_poly(np.asarray(x, np.float64), up, down).astype(np.float32)


def device_resample(x, a, b):
    """One-shot whole-clip ovc_resample of a NumPy clip, back on the host."""
    nat = get_native(False).native
    d = torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()[None]
    y = nat.resample(d, torch.tensor([len(x)], dtype=torch.int64, device="cuda"), a, b)
    return y[0].cpu().numpy()


def within_ulp(got, ref):
    return np.abs(got - ref) <= np.spacing(np.maximum(np.abs(got), np.abs(ref)))


def run_batch(xs, a, b, pad_extra=5, out_extra=7):
    """Ragged batch: rows padded with NaN past each clip, output buffer pre-filled with NaN."""
    from openvoice_b200._native import resample_span
    nat = get_native(False).native
    Lmax = max(len(x) for x in xs) + pad_extra
    inp = np.full((len(xs), Lmax), np.nan, np.float32)
    for i, x in enumerate(xs):
        inp[i, : len(x)] = x
    pitch = resample_span(a, b, Lmax)[0] + out_extra
    out = torch.full((len(xs), pitch), float("nan"), device="cuda")
    lens = torch.tensor([len(x) for x in xs], dtype=torch.int64, device="cuda")
    nat.resample(torch.from_numpy(inp).cuda(), lens, a, b, out=out)
    return out.cpu().numpy()


@pytest.mark.parametrize("a,b", PAIRS + [(2048, 1)])
def test_kernel_matches_resample_poly(a, b):
    from openvoice_b200._native import resample_span
    up, down = updown(a, b)
    K = -(-(20 * max(up, down) + 1) // up)                      # input samples under one output: N / up
    lens = [1, 2, K - 1, K + 1, 1000, 10 * a] if (a, b) != (2048, 1) else [1, 5000, 50000]
    xs = [wave(a + 7 * i, n) for i, n in enumerate(lens)]
    y = run_batch(xs, a, b)
    assert not np.isnan(y).any()
    for i, x in enumerate(xs):
        n = resample_span(a, b, len(x))[0]
        ref = ref_poly(x, a, b)
        assert n == len(ref)
        assert within_ulp(y[i, :n], ref).all(), (a, b, len(x))
        assert not y[i, n:].any() and (np.signbit(y[i, n:]) == 0).all()     # +0 past n_out: zero-padded rows


@pytest.mark.parametrize("a,b", [(48000, MODEL_SR), (MODEL_SR, 48000), (16000, MODEL_SR), (192000, MODEL_SR)])
def test_batch_row_and_windows_equal_whole_clip(a, b):
    from openvoice_b200._native import resample_span
    nat = get_native(False).native
    xs = [wave(3 + i, n) for i, n in enumerate((a * 3 + 17, 999, a // 2))]
    y = run_batch(xs, a, b)
    for i, x in enumerate(xs):
        solo = device_resample(x, a, b)
        assert np.array_equal(y[i, : len(solo)], solo)
    x = xs[0]
    whole = device_resample(x, a, b)
    for m0, m1, extra in ((0, 1, 0), (0, 300, 3), (5, 6, 0), (1234, 5678, 11), (len(whole) - 50, len(whole), 0),
                          (len(whole) - 3, len(whole) + 4, 2)):
        _, _, lo, hi = resample_span(a, b, 0, m0, m1)
        lo, hi = max(0, lo - extra), min(len(x), hi + extra)
        seg = torch.from_numpy(x[lo:hi].copy()).cuda()[None]
        ln = torch.tensor([len(x)], dtype=torch.int64, device="cuda")
        got = nat.resample(seg, ln, a, b, out_pitch=m1 - m0, in_start=lo, out_start=m0)[0].cpu().numpy()
        ref = np.concatenate([whole, np.zeros(max(0, m1 - len(whole)), np.float32)])[m0:m1]
        assert np.array_equal(got, ref), (m0, m1)


@pytest.mark.parametrize("a,b", [(48000, MODEL_SR), (MODEL_SR, 48000), (16000, MODEL_SR), (44100, MODEL_SR)])
def test_streaming_resampler_equals_one_shot(a, b):
    from openvoice_b200.streaming import StreamingResampler
    x = wave(17, 2 * a + 333)
    whole = device_resample(x, a, b)
    up, down = updown(a, b)
    span = -(-(20 * max(up, down) + 1) // up)
    for sizes in ([1] * 200 + [span // 2, 3, span * 3, 4096], [span - 1, span + 1, 7, 10000]):
        rs = StreamingResampler(get_native(False), a, b)
        outs, pos, i, peak = [], 0, 0, 0
        while pos < len(x):
            n = min(sizes[i % len(sizes)], len(x) - pos)
            outs.append(rs.push(x[pos: pos + n]))
            pos, i = pos + n, i + 1
            peak = max(peak, rs.state_samples)
        outs.append(rs.flush())
        assert np.array_equal(np.concatenate(outs), whole)
        assert peak <= span + 2 * down // up + 4, peak          # the tail future outputs read, never the chunk backlog
    rs = StreamingResampler(get_native(False), a, b)             # nothing but a flush
    assert len(rs.flush()) == 0


@pytest.fixture(scope="module")
def conv(hps):
    """A ToneColorConverter around the session's converter on the synthetic checkpoint."""
    from openvoice_b200.api import ToneColorConverter
    c = ToneColorConverter.__new__(ToneColorConverter)
    c.hps, c.device, c.watermark_model, c.version = hps, "cuda:0", None, "v1"
    c.model = get_native(False)
    return c


@pytest.fixture(scope="module")
def ses():
    gen = torch.Generator().manual_seed(31)
    return 0.1 * torch.randn(1, 256, 1, generator=gen), 0.1 * torch.randn(1, 256, 1, generator=gen)


def test_convert_with_sr_equals_device_resample_then_convert(conv, ses):
    src, tgt = ses
    x = wave(41, 48000 * 3 + 555)
    y = device_resample(x, 48000, MODEL_SR)
    T = len(y) // 256
    noise = torch.randn(1, 192, T, generator=torch.Generator().manual_seed(2))
    got = conv.convert(x, src, tgt, tau=0.3, noise=noise, sr=48000)
    assert np.array_equal(got, conv.convert(y, src, tgt, tau=0.3, noise=noise))
    host = conv.convert(ref_poly(x, 48000, MODEL_SR), src, tgt, tau=0.3, noise=noise)
    assert rel_err(got, host) <= 1e-4
    assert np.array_equal(conv.convert(x, src, tgt, tau=0.3, noise=noise, sr=MODEL_SR),
                          conv.convert(x, src, tgt, tau=0.3, noise=noise))          # the model rate: no resampling
    # convert_batch: ragged batch of resampled items, each equal to its own convert
    xs = [x, wave(42, 48000 + 77), wave(43, 2000)]
    ys = [device_resample(v, 48000, MODEL_SR) for v in xs]
    for got, v in zip(conv.convert_batch(xs, src, tgt, tau=0.0, sr=48000), ys):
        assert np.array_equal(got, conv.convert(v, src, tgt, tau=0.0))


def test_other_entry_points_with_sr(conv, ses):
    src, tgt = ses
    xs = [wave(50 + i, n) for i, n in enumerate((16000 * 2 + 5, 16000 * 3, 9000))]
    ys = [device_resample(v, 16000, MODEL_SR) for v in xs]
    assert torch.equal(conv.extract_se(xs, sr=16000), conv.extract_se(ys))
    a = conv.extract_se_batch([xs[:2], xs[2]], sr=16000)
    b = conv.extract_se_batch([ys[:2], ys[2]])
    assert all(torch.equal(p, q) for p, q in zip(a, b))
    x = wave(60, 48000 * 4 + 1)
    y = device_resample(x, 48000, MODEL_SR)
    noise = torch.randn(192, len(y) // 256, generator=torch.Generator().manual_seed(3))
    assert np.array_equal(conv.convert_long(x, src, tgt, tau=0.3, noise=noise, window_frames=200, sr=48000),
                          conv.convert_long(y, src, tgt, tau=0.3, noise=noise, window_frames=200))
    w48 = [x, wave(61, 30000), wave(62, 48000)]
    w22 = [y] + [device_resample(v, 48000, MODEL_SR) for v in w48[1:]]
    for p, q in zip(conv.convert_concurrent(w48, src, tgt, tau=0.0, streams=2, sr=48000),
                    conv.convert_concurrent(w22, src, tgt, tau=0.0, streams=2)):
        assert np.array_equal(p, q)
    o, n = conv.convert_batch_device(w48, src, tgt, tau=0.0, slot=0, sr=48000)
    o = o.clone()
    o2, n2 = conv.convert_batch_device(w22, src, tgt, tau=0.0, slot=1)
    torch.cuda.synchronize()
    assert n == n2
    for i, k in enumerate(n):
        assert torch.equal(o[i, :k], o2[i, :k])


def test_streaming_converter_input_and_output_sr(conv, ses):
    from openvoice_b200.streaming import StreamingConverter, StreamingResampler
    src, tgt = ses
    x = wave(70, 48000 * 5 + 123)
    T = len(device_resample(x, 48000, MODEL_SR)) // 256
    noise = torch.randn(192, T, generator=torch.Generator().manual_seed(4))
    whole = conv.convert(x, src, tgt, tau=0.3, noise=noise[None], sr=48000)
    whole48 = device_resample(whole, MODEL_SR, 48000)
    # error gain of the 22.05 kHz -> 48 kHz filter: max over its phases of sum |h| = 2.24, so the model-rate stream's
    # 2e-6 * rms bound grows to at most 2e-6 * 2.24 * rms at 48 kHz
    h = firwin(20 * 320 + 1, 1.0 / 320, window=("kaiser", 5.0)) * 320
    gain = max(np.abs(h[p::320]).sum() for p in range(320))
    assert 2.2 < gain < 2.3
    for out_sr, ref, bound in ((None, whole, 2e-6), (48000, whole48, 2e-6 * gain)):
        sc = StreamingConverter(conv, src, tgt, tau=0.3, window_frames=200, noise_fn=lambda a, b: noise[:, a:b],
                                input_sr=48000, output_sr=out_sr)
        outs, pos, i = [], 0, 0
        sizes = [480, 1, 7000, 48000, 333, 96000]
        while pos < len(x):
            n = min(sizes[i % len(sizes)], len(x) - pos)
            outs.append(sc.push(x[pos: pos + n]))
            pos, i = pos + n, i + 1
        outs.append(sc.flush())
        stream = np.concatenate(outs)
        assert stream.shape == ref.shape, out_sr
        assert rel_err(stream, ref) <= bound, out_sr
    la = StreamingResampler(conv.model, 48000, MODEL_SR).lookahead_s + StreamingResampler(conv.model, MODEL_SR, 48000).lookahead_s
    assert 0 < la < 1e-3


class CallCounter:
    def __init__(self, monkeypatch, nat):
        self.n = {}
        for name in ("resample", "spectrogram", "convert_waveform", "reference_encoder"):
            fn = getattr(nat, name)
            self.n[name] = 0

            def wrapped(*a, _fn=fn, _name=name, **k):
                self.n[_name] += 1
                return _fn(*a, **k)
            monkeypatch.setattr(nat, name, wrapped)


def test_refusals_before_any_launch(conv, ses, monkeypatch, tmp_path):
    src, tgt = ses
    counter = CallCounter(monkeypatch, conv.model.native)
    x = wave(80, 48000)
    with pytest.raises(ValueError, match="44101"):
        conv.convert(x, src, tgt, sr=44101)
    with pytest.raises(ValueError, match="44101"):
        conv.extract_se([x], sr=44101)
    short = wave(81, 800)                        # 368 samples at 22.05 kHz: not longer than the reflect padding (384)
    with pytest.raises(ValueError, match="after resampling"):
        conv.convert_batch([x, short], src, tgt, sr=48000)
    with pytest.raises(ValueError, match="after resampling"):
        conv.convert_concurrent([short], src, tgt, sr=48000)
    with pytest.raises(ValueError, match="clip 1 .*after resampling"):
        conv.extract_se([x, short], sr=48000)
    path = tmp_path / "a.npy"
    np.save(path, x)
    with pytest.raises(ValueError, match="file path"):
        conv.convert(str(path), src, tgt, sr=48000)
    with pytest.raises(ValueError, match="file path"):
        conv.convert_long(str(path), src, tgt, sr=48000)
    assert counter.n == {"resample": 0, "spectrogram": 0, "convert_waveform": 0, "reference_encoder": 0}
