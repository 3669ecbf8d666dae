"""-m gpu: the ragged reference encoder (ovc_reference_encoder_ragged) and the batched extract_se /
extract_se_batch built on it.

The rule under test: every item of a ragged batch is encoded at its own length, so its row is bit-identical to a solo
call on that item alone, whatever the padding frames hold; and extract_se, which groups its clips into such batches,
returns bit for bit what encoding the clips one at a time returned.  Against the reference (golden vectors of
oracle/make_golden.py and oracle/make_golden_se.py) and the CPU oracle the gate is the parity suite's
max|cuda - ref| <= 1e-4 * rms(ref)."""
import os

import numpy as np
import pytest
import torch

from conftest import get_native
from oracle import vc_oracle as O

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
REL = 1e-4
LENS = [1, 2, 3, 63, 64, 65, 128, 129, 257]


def rel_err(got, ref):
    ref = np.asarray(ref, dtype=np.float64)
    got = np.asarray(got, dtype=np.float64)
    return float(np.abs(got - ref).max() / (np.sqrt((ref ** 2).mean()) + 1e-30))


def clips(seed, lengths):
    """The clip recipe of oracle/make_golden_se.py."""
    rng = np.random.default_rng(int(seed))
    return [(0.5 * (2 * rng.random(int(n), dtype=np.float32) - 1)).astype(np.float32) for n in lengths]


@pytest.fixture(scope="module")
def conv(hps):
    """A ToneColorConverter around the session's converter on the synthetic checkpoint."""
    from openvoice_b200.api import ToneColorConverter
    c = ToneColorConverter.__new__(ToneColorConverter)
    c.hps, c.device, c.watermark_model, c.version = hps, "cuda:0", None, "v1"
    c.model = get_native(False)
    return c


@pytest.fixture(scope="module")
def golden():
    d = np.load(os.path.join(GOLD, "extract_se.npz"))
    a = clips(d["a_seed"], d["a_lengths"])
    b = clips(d["b_seed"], d["b_lengths"])
    speakers, k = [], 0
    for n in d["b_counts"]:
        speakers.append(b[k: k + int(n)])
        k += int(n)
    return d, a, speakers


def old_loop(nat, waves):
    """extract_se as it was before the batched path: one spectrogram and one encoder pass per clip."""
    gs = []
    for w in waves:
        y = torch.from_numpy(w).cuda().unsqueeze(0).contiguous()
        n = torch.tensor([y.shape[1]], dtype=torch.int64, device="cuda")
        y, _ = nat.spectrogram(y, n)
        gs.append(nat.reference_encoder(y).unsqueeze(-1))
    return torch.stack(gs).mean(0)


class CallCounter:
    def __init__(self, monkeypatch, nat):
        self.n = {"spectrogram": 0, "reference_encoder": 0}
        for name in self.n:
            monkeypatch.setattr(nat, name, self._wrap(name, getattr(nat, name)))

    def _wrap(self, name, fn):
        def f(*a, **k):
            self.n[name] += 1
            return fn(*a, **k)
        return f


@pytest.mark.parametrize("fill", [float("nan"), 1e30])
def test_ragged_equals_solo_bitwise(fill):
    """Every row of a ragged batch equals a solo call at the item's length; padding frames (NaN / 1e30) and a
    workspace left dirty by a call on all-padding input are never read."""
    nat = get_native(False).native
    N, T = len(LENS), max(LENS)
    spec = O.synthetic_inputs(N, T, 21)[0]
    for n, L in enumerate(LENS):
        spec[n, :, L:] = fill
    spec = spec.cuda().contiguous()
    nat.reference_encoder(torch.full_like(spec, fill))            # stale workspace
    g = nat.reference_encoder(spec, torch.tensor(LENS, dtype=torch.int64, device="cuda"))
    assert g.shape == (N, 256) and torch.isfinite(g).all()
    for n, L in enumerate(LENS):
        solo = nat.reference_encoder(spec[n: n + 1, :, :L].contiguous())
        assert torch.equal(g[n], solo[0]), L


def test_ragged_full_lengths_equal_plain_call():
    nat = get_native(False).native
    d = np.load(os.path.join(GOLD, "ref_enc.npz"))
    spec = O.synthetic_inputs(2, 140, 7)[0].cuda().contiguous()
    g = nat.reference_encoder(spec, torch.tensor([140, 140], dtype=torch.int64, device="cuda"))
    assert torch.equal(g, nat.reference_encoder(spec))
    assert rel_err(g.cpu().numpy(), d["g"]) <= REL


def test_ragged_matches_oracle(synthetic_sd):
    nat = get_native(False).native
    N, T = len(LENS), max(LENS)
    spec = O.synthetic_inputs(N, T, 22)[0]
    g = nat.reference_encoder(spec.cuda().contiguous(), torch.tensor(LENS, dtype=torch.int64, device="cuda")).cpu()
    for n, L in enumerate(LENS):
        with torch.no_grad():
            ref = O.reference_encoder(synthetic_sd, spec[n: n + 1, :, :L].transpose(1, 2))
        assert rel_err(g[n].numpy(), ref[0].numpy()) <= REL, L


def test_extract_se_matches_reference_golden(conv, golden):
    d, a, speakers = golden
    for i, w in enumerate(a):
        assert rel_err(conv.extract_se([w]).cpu().numpy()[0, :, 0], d["a_clip"][i]) <= REL, i
    se = conv.extract_se(a)
    assert se.shape == (1, 256, 1)
    assert rel_err(se.cpu().numpy()[0, :, 0], d["a_mean"][0]) <= REL
    for j, se in enumerate(conv.extract_se_batch(speakers)):
        assert rel_err(se.cpu().numpy()[0, :, 0], d["b_mean"][j]) <= REL, j
    flat = [w for s in speakers for w in s]
    for i, w in enumerate(flat):
        assert rel_err(conv.extract_se(w).cpu().numpy()[0, :, 0], d["b_clip"][i]) <= REL, i


def test_extract_se_equals_per_clip_loop(conv, golden):
    _, a, speakers = golden
    for waves in (a, a[::-1], speakers[2], [a[3]]):
        assert torch.equal(conv.extract_se(waves), old_loop(conv.model.native, waves))


def test_extract_se_one_pass_and_chunking(conv, golden, monkeypatch):
    from openvoice_b200 import api
    _, a, _ = golden
    full = conv.extract_se(a)
    counter = CallCounter(monkeypatch, conv.model.native)
    assert torch.equal(conv.extract_se(a), full)
    assert counter.n == {"spectrogram": 1, "reference_encoder": 1}
    monkeypatch.setattr(api, "SE_CHUNK_FRAMES", 150)
    counter.n = {"spectrogram": 0, "reference_encoder": 0}
    chunks = api.plan_se_chunks([len(w) // 256 for w in a], 150)
    assert len(chunks) >= 3
    assert torch.equal(conv.extract_se(a), full)
    assert counter.n == {"spectrogram": len(chunks), "reference_encoder": len(chunks)}


def test_extract_se_batch_equals_extract_se(conv, golden, tmp_path):
    _, a, speakers = golden
    assert [len(s) for s in speakers] == [1, 2, 4]
    speakers = [speakers[0][0], speakers[1], speakers[2] + [a[0]], a[:3]]      # a bare clip is a speaker of one
    paths = [str(tmp_path / f"spk{i}" / "se.pth") for i in range(len(speakers))]
    got = conv.extract_se_batch(speakers, se_save_paths=paths)
    assert len(got) == len(speakers)
    for se, s, p in zip(got, speakers, paths):
        assert se.shape == (1, 256, 1)
        assert torch.equal(se, conv.extract_se(s))
        assert torch.equal(torch.load(p), se.cpu())


def test_extract_se_refuses_short_clip_before_launch(conv, golden, monkeypatch):
    _, a, _ = golden
    counter = CallCounter(monkeypatch, conv.model.native)
    with pytest.raises(ValueError, match="clip 1 "):
        conv.extract_se([a[0], np.zeros(300, np.float32)])
    with pytest.raises(ValueError, match="clip 0 "):
        conv.extract_se_batch([[np.zeros(200, np.float32)], a[:2]])
    assert counter.n == {"spectrogram": 0, "reference_encoder": 0}


def test_get_se_uses_batched_extract_se(conv, tmp_path):
    from openvoice_b200 import se_extractor
    sr = conv.hps.data.sampling_rate
    audio = clips(77, [35 * sr])[0]
    se, name = se_extractor.get_se(audio, conv, target_dir=str(tmp_path))
    segs = se_extractor.split_audio_fixed(audio, sr)
    assert len(segs) == 4
    assert torch.equal(se, conv.extract_se(segs))
    assert torch.equal(se, old_loop(conv.model.native, segs))
    assert os.path.isfile(os.path.join(str(tmp_path), name, "se.pth"))
