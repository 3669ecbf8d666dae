"""Generate the per-frame embedding vectors tests/golden/vc_frames_*.npz and convert_frames.npz by running the REAL
reference (a checkout of myshell-ai/OpenVoice), as make_golden.py does for the per-item ones.

``OPENVOICE_REFERENCE=<path to the checkout> python oracle/make_golden_frames.py``.  It writes only its own files
(the vectors above and tests/golden/REPORT_frames.json); the other fixtures are left alone.

The reference's ``SynthesizerTrn.voice_conversion`` (openvoice/models.py:492-499) takes ``sid_src`` / ``sid_tgt`` of
shape [B, gin, T]: every conditioning layer (``WN.cond_layer``, modules.py:189-196; ``Generator.cond``,
models.py:274-275) is a 1x1 conv added to per-frame activations, so the per-frame embedding broadcasts with no change to
the reference, and ``ToneColorConverter.convert`` (api.py:141-160) passes the embeddings straight through.  Each case
stores its inputs (spectrogram or waveform, lengths, both embeddings, noise) next to the reference's outputs.
"""
from __future__ import annotations

import json
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.dont_write_bytecode = True  # the reference tree is read-only

import make_golden as M  # noqa: E402
import vc_oracle as O  # noqa: E402


def morph(a, b, T):
    w = torch.linspace(0, 1, T).view(1, 1, T)
    return (a + w * (b - a)).contiguous()


def switch(a, b, T, s):
    g = a.expand(a.shape[0], a.shape[1], T).clone()
    g[:, :, s:] = b
    return g


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    api, _, _ = M.import_reference()
    sd = O.synthetic_state_dict(1234)
    outdir = os.path.join(ROOT, "tests", "golden")
    report = {}
    convs = {False: M.build_reference_converter(api, sd, zero_g=False),
             True: M.build_reference_converter(api, sd, zero_g=True)}

    # source: a linear morph to a second voice over the clip; target: a hard switch at frame 30
    cases = [
        ("vc_frames_b1_t67", dict(B=1, T=67, seed=2, lengths=None, zero_g=False, tau=0.3)),
        ("vc_frames_b2_padded", dict(B=2, T=40, seed=3, lengths=[40, 29], zero_g=False, tau=0.3)),
        ("vc_frames_b1_t67_v2", dict(B=1, T=67, seed=4, lengths=None, zero_g=True, tau=0.3)),
    ]
    for name, c in cases:
        spec, lengths, gs, gt, noise = O.synthetic_inputs(c["B"], c["T"], c["seed"], lengths=c["lengths"])
        gen = torch.Generator().manual_seed(500 + c["seed"])
        a2, b2 = (0.1 * torch.randn(c["B"], 256, 1, generator=gen) for _ in range(2))
        g_src, g_tgt = morph(gs, a2, c["T"]), switch(gt, b2, c["T"], 30)
        with torch.no_grad(), M.injected_noise(noise):
            o, mask, (z, zp, zh) = convs[c["zero_g"]].model.voice_conversion(spec, lengths, g_src, g_tgt, tau=c["tau"])
            oc, _, _ = convs[c["zero_g"]].model.voice_conversion(spec, lengths, gs, gt, tau=c["tau"])
        with torch.no_grad():
            oo, _, (oz, ozp, ozh) = O.voice_conversion(sd, spec, lengths, g_src, g_tgt, noise, c["tau"], c["zero_g"])
        rms = float(o.pow(2).mean().sqrt())
        report[name] = dict(o=M.maxdiff(o, oo), z=M.maxdiff(z, oz), zp=M.maxdiff(zp, ozp), zh=M.maxdiff(zh, ozh),
                            vs_constant_over_rms=M.maxdiff(o, oc) / rms)
        np.savez_compressed(os.path.join(outdir, name + ".npz"), spec=spec.numpy(), lengths=lengths.numpy(),
                            g_src=g_src.numpy(), g_tgt=g_tgt.numpy(), noise=noise.numpy(), o_hat=o.numpy(),
                            z=z.numpy(), z_p=zp.numpy(), z_hat=zh.numpy(), meta=np.array(json.dumps(c)))

    # ToneColorConverter.convert on a waveform with [1, 256, T] embeddings, T = L // 256 (what the broadcast needs)
    rng = np.random.default_rng(1001)
    L = 256 * 30 + 77
    T = L // 256
    wav = (0.5 * (2 * rng.random(L, dtype=np.float32) - 1)).astype(np.float32)
    gen = torch.Generator().manual_seed(2001)
    s0, s1, t0, t1 = (0.1 * torch.randn(1, 256, 1, generator=gen) for _ in range(4))
    g_src, g_tgt = morph(s0, s1, T), switch(t0, t1, T, 12)
    noise = torch.randn(1, 192, T, generator=torch.Generator().manual_seed(4001))
    with tempfile.TemporaryDirectory() as td:
        p = os.path.join(td, "a.npy")
        np.save(p, wav)
        with M.injected_noise(noise):
            a = convs[False].convert(p, g_src, g_tgt, tau=0.3)
    with torch.no_grad():
        b = O.convert_waveform(sd, torch.from_numpy(wav), g_src, g_tgt, noise, 0.3)
    report["convert_frames"] = dict(audio=M.maxdiff(torch.from_numpy(a), b))
    np.savez_compressed(os.path.join(outdir, "convert_frames.npz"), wav=wav, g_src=g_src.numpy(), g_tgt=g_tgt.numpy(),
                        noise=noise.numpy(), audio=a)

    with open(os.path.join(outdir, "REPORT_frames.json"), "w") as f:
        json.dump(report, f, indent=1, sort_keys=True)
    print(json.dumps(report, indent=1, sort_keys=True))


if __name__ == "__main__":
    main()
