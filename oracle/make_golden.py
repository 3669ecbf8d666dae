"""Generate tests/golden/*.npz by running the REAL reference (a checkout of myshell-ai/OpenVoice).

Run on a machine that has the reference checked out:
``OPENVOICE_REFERENCE=<path to the checkout> python oracle/make_golden.py``.  The tests only read the
committed vectors, so nothing else in the project needs the reference.  The reference ships no tests or golden vectors (SURVEY.md section 8c),
so parity is pinned on outputs of the reference's own code -- ``SynthesizerTrn.voice_conversion``
(openvoice/models.py:492-499), ``ToneColorConverter.convert`` (openvoice/api.py:141-160),
``spectrogram_torch`` (openvoice/mel_processing.py:40-75) and ``ReferenceEncoder``
(openvoice/models.py:339-359) -- on the seeded synthetic checkpoint of ``vc_oracle``.

I/O-only third-party modules that are not installed (librosa, soundfile, wavmark, G2P
libs) are stubbed in sys.modules; none of them does arithmetic on this path
(the "audio files" are .npy arrays already at the model sampling rate; watermark off).
"""
from __future__ import annotations

import json
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.dont_write_bytecode = True  # the reference tree is read-only

import vc_oracle as O  # noqa: E402


def import_reference():
    ref = os.environ.get("OPENVOICE_REFERENCE")
    if not ref or not os.path.isdir(ref):
        raise SystemExit("set OPENVOICE_REFERENCE to a checkout of myshell-ai/OpenVoice")
    sys.path.insert(0, ref)
    lib = types.ModuleType("librosa")
    lib.filters = types.ModuleType("librosa.filters")
    lib.filters.mel = lambda *a, **k: None
    lib.load = lambda path, sr=None, mono=True: (np.load(path).astype(np.float32), sr)
    sys.modules["librosa"] = lib
    sys.modules["librosa.filters"] = lib.filters
    sf = types.ModuleType("soundfile")
    sf.write = lambda p, a, sr: np.save(p, a)
    sys.modules["soundfile"] = sf
    for n in ["inflect", "unidecode", "eng_to_ipa", "pypinyin", "jieba", "cn2an"]:
        sys.modules[n] = types.ModuleType(n)
    sys.modules["inflect"].engine = lambda: None
    sys.modules["unidecode"].unidecode = lambda s: s
    sys.modules["pypinyin"].lazy_pinyin = None
    sys.modules["pypinyin"].BOPOMOFO = None

    class _WM:
        def to(self, d):
            return self

    wm = types.ModuleType("wavmark")
    wm.load_model = lambda: _WM()
    sys.modules["wavmark"] = wm
    from openvoice import api, mel_processing, models  # noqa: F401
    return api, mel_processing, models


class injected_noise:
    """Make the one randn_like on the path (openvoice/models.py:220) return our noise."""

    def __init__(self, noise):
        self.noise = noise

    def __enter__(self):
        self.orig = torch.randn_like
        torch.randn_like = lambda x, **k: self.noise.to(x.dtype)

    def __exit__(self, *a):
        torch.randn_like = self.orig


def build_reference_converter(api, sd, zero_g=False):
    hp = json.loads(json.dumps(O.DEFAULT_HPARAMS))
    hp["model"]["zero_g"] = zero_g
    if zero_g:
        hp["_version_"] = "v2"
    with tempfile.NamedTemporaryFile("w", suffix=".json", delete=False) as f:
        json.dump(hp, f)
    conv = api.ToneColorConverter(f.name, device="cpu")
    conv.watermark_model = None
    missing, unexpected = conv.model.load_state_dict(sd, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    os.unlink(f.name)
    return conv


def maxdiff(a, b):
    return float((a - b).abs().max())


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    api, mel, models = import_reference()
    sd = O.synthetic_state_dict(1234)
    outdir = os.path.join(ROOT, "tests", "golden")
    os.makedirs(outdir, exist_ok=True)
    report = {}

    conv = build_reference_converter(api, sd, zero_g=False)
    conv2 = build_reference_converter(api, sd, zero_g=True)

    cases = [
        ("vc_b1_t24", dict(B=1, T=24, seed=1, lengths=None, zero_g=False, tau=0.3)),
        ("vc_b1_t67", dict(B=1, T=67, seed=2, lengths=None, zero_g=False, tau=0.3)),
        ("vc_b2_padded", dict(B=2, T=40, seed=3, lengths=[40, 29], zero_g=False, tau=0.3)),
        ("vc_b1_t24_v2", dict(B=1, T=24, seed=4, lengths=None, zero_g=True, tau=0.3)),
        ("vc_b1_t24_tau0", dict(B=1, T=24, seed=5, lengths=None, zero_g=False, tau=0.0)),
    ]
    for name, c in cases:
        spec, lengths, gs, gt, noise = O.synthetic_inputs(c["B"], c["T"], c["seed"], lengths=c["lengths"])
        model = (conv2 if c["zero_g"] else conv).model
        with torch.no_grad(), injected_noise(noise):
            o, mask, (z, zp, zh) = model.voice_conversion(spec, lengths, gs, gt, tau=c["tau"])
        with torch.no_grad():
            oo, omask, (oz, ozp, ozh) = O.voice_conversion(sd, spec, lengths, gs, gt, noise, c["tau"], c["zero_g"])
        d = dict(o=maxdiff(o, oo), z=maxdiff(z, oz), zp=maxdiff(zp, ozp), zh=maxdiff(zh, ozh))
        report[name] = d
        # fp64 twin of the oracle = the noise floor of the reference's own fp32 arithmetic
        with torch.no_grad():
            o64, _, (z64, zp64, zh64) = O.voice_conversion(
                {k: v.double() for k, v in sd.items()}, spec.double(), lengths, gs.double(), gt.double(),
                noise.double(), c["tau"], c["zero_g"])
        report[name]["floor_o"] = maxdiff(o.double(), o64)
        report[name]["floor_zh"] = maxdiff(zh.double(), zh64)
        np.savez_compressed(
            os.path.join(outdir, name + ".npz"),
            o_hat=o.numpy(), z=z.numpy(), z_p=zp.numpy(), z_hat=zh.numpy(), mask=mask.numpy(),
            meta=np.array(json.dumps(c)))

    # ToneColorConverter.convert end to end (spectrogram + VC), tau = 0 so no RNG is involved,
    # and once with injected noise.
    rng = np.random.default_rng(1000)
    L = 256 * 30 + 77
    wav = (0.5 * (2 * rng.random(L, dtype=np.float32) - 1)).astype(np.float32)
    gen = torch.Generator().manual_seed(2000)
    src_se = 0.1 * torch.randn(1, 256, 1, generator=gen)
    tgt_se = 0.1 * torch.randn(1, 256, 1, generator=gen)
    with tempfile.TemporaryDirectory() as td:
        p = os.path.join(td, "a.npy")
        np.save(p, wav)
        a0 = conv.convert(p, src_se, tgt_se, tau=0.0)
        T = L // 256
        noise = torch.randn(1, 192, T, generator=torch.Generator().manual_seed(4000))
        with injected_noise(noise):
            a1 = conv.convert(p, src_se, tgt_se, tau=0.3)
    with torch.no_grad():
        b0 = O.convert_waveform(sd, torch.from_numpy(wav), src_se, tgt_se, None, 0.0)
        b1 = O.convert_waveform(sd, torch.from_numpy(wav), src_se, tgt_se, noise, 0.3)
        spec_ref = mel.spectrogram_torch(torch.from_numpy(wav)[None], 1024, 22050, 256, 1024, center=False)
        spec_or = O.spectrogram(torch.from_numpy(wav)[None])
    report["convert"] = dict(tau0=maxdiff(torch.from_numpy(a0), b0), tau03=maxdiff(torch.from_numpy(a1), b1),
                             spec=maxdiff(spec_ref, spec_or))
    np.savez_compressed(os.path.join(outdir, "convert_wave.npz"), audio_tau0=a0, audio_tau03=a1,
                        spec=spec_ref.numpy(), L=np.array(L))

    # ReferenceEncoder (extract_se arithmetic, openvoice/api.py:123-133)
    spec_se = O.synthetic_inputs(2, 140, 7)[0]
    with torch.no_grad():
        g_ref = conv.model.ref_enc(spec_se.transpose(1, 2))
        g_or = O.reference_encoder(sd, spec_se.transpose(1, 2))
    report["ref_enc"] = dict(g=maxdiff(g_ref, g_or))
    np.savez_compressed(os.path.join(outdir, "ref_enc.npz"), g=g_ref.numpy())

    with open(os.path.join(outdir, "REPORT.json"), "w") as f:
        json.dump(report, f, indent=1, sort_keys=True)
    print(json.dumps(report, indent=1, sort_keys=True))


if __name__ == "__main__":
    main()
