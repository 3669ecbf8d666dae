"""Generate tests/golden/tts_fit_*.npz by running the REAL reference modules with fitted length scales.

Run in the build container only (``python oracle/make_golden_tts_fit.py``).  Same checkpoint, inputs and injected
RNG as ``make_golden_tts.py``.  Per case: ``enc_p``, ``sdp`` (reverse) and ``dp`` of the reference give
logw = sdp * sdp_ratio + dp * (1 - sdp_ratio) (openvoice/models.py:474-476); the float32 NumPy statement of the rule
(``tts_fit_oracle``) gives each fit group's scale s*; then ``SynthesizerTrn.infer(..., length_scale=s)`` gives each
row's audio at its own scale (rows outside every group at the case's unfitted scale).  Every row runs alone at its own
length (batch 1), as ``tts_batch`` promises each sentence: a padded reference batch decodes every row to the longest
row's frames, and the generator's activations past a row's end reach back into its last samples.  Writes only
tests/golden/tts_fit_*.npz and REPORT_tts_fit.json.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.dont_write_bytecode = True

import vc_oracle as V  # noqa: E402
import tts_oracle as T  # noqa: E402
import tts_fit_oracle as FO  # noqa: E402
from make_golden import import_reference  # noqa: E402
from make_golden_tts import injected_rng  # noqa: E402

# name, inputs, groups as (row0, row1, target as a multiple of the group's frames at scale 1 -- or "clamp": past F(hi))
CASES = [
    ("tts_fit_b1_one", dict(B=1, T=37, seed=41, lengths=None), [(0, 1, 1.37)]),
    ("tts_fit_b3_joint", dict(B=3, T=60, seed=42, lengths=[60, 45, 52]), [(0, 3, 0.81)]),
    ("tts_fit_b2_mixed", dict(B=2, T=50, seed=43, lengths=[50, 31]), [(0, 1, 1.9)]),
    ("tts_fit_b1_clamp", dict(B=1, T=40, seed=44, lengths=None), [(0, 1, "clamp")]),
]
PARAMS = dict(noise_scale=0.667, noise_scale_w=0.6, sdp_ratio=0.2)
UNFITTED_SCALE = 1.0


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    api, mel, models = import_reference()
    hp = V.DEFAULT_HPARAMS
    tts = T.TTS_HPARAMS
    hop = hp["data"]["hop_length"]
    sd = T.synthetic_tts_state_dict()
    model = models.SynthesizerTrn(tts["n_vocab"], hp["data"]["filter_length"] // 2 + 1,
                                  n_speakers=tts["n_speakers"], **hp["model"]).eval()
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not unexpected and all(k.startswith("sdp.post_") for k in missing), (missing, unexpected)

    outdir = os.path.join(ROOT, "tests", "golden")
    report = {}
    for name, c, groups in CASES:
        tokens, lengths, sid, noise_w = T.synthetic_tts_inputs(c["B"], c["T"], c["seed"], c["lengths"])
        noise = torch.randn(c["B"], 192, 40 * c["T"] + 64, generator=torch.Generator().manual_seed(30_000 + c["seed"]))
        lens = lengths.numpy()
        rows = [(tokens[b:b + 1, :lens[b]], lengths[b:b + 1], sid[b:b + 1], noise_w[b:b + 1, :, :lens[b]], noise[b:b + 1])
                for b in range(c["B"])]
        logw = np.zeros((c["B"], c["T"]), np.float32)
        for b, (tk, ln, sp, nw, nz) in enumerate(rows):
            with torch.no_grad(), injected_rng(nw, nz):
                x, m_p, logs_p, x_mask = model.enc_p(tk, ln)
                g = model.emb_g(sp).unsqueeze(-1)
                lw = (model.sdp(x, x_mask, g=g, reverse=True, noise_scale=PARAMS["noise_scale_w"]) * PARAMS["sdp_ratio"]
                      + model.dp(x, x_mask, g=g) * (1 - PARAMS["sdp_ratio"]))
            logw[b, : lens[b]] = lw[0, 0].numpy()
        e = np.exp(logw)
        scale = np.full(c["B"], UNFITTED_SCALE, np.float32)
        fit = []
        for r0, r1, k in groups:
            if k == "clamp":
                target = FO.group_frames(e[r0:r1], lens[r0:r1], FO.SCALE_HI) + 50
            else:
                target = int(round(FO.group_frames(e[r0:r1], lens[r0:r1], 1.0) * k))
            s = FO.fit_scale(e[r0:r1], lens[r0:r1], target)
            scale[r0:r1] = s
            fit.append((r0, r1, target))
        o_rows = {}
        w_ceil = np.zeros_like(logw)
        y_lengths = np.zeros(c["B"], np.int64)
        for b, (tk, ln, sp, nw, nz) in enumerate(rows):
            with torch.no_grad(), injected_rng(nw, nz):
                o, attn, y_mask, _ = model.infer(tk, ln, sid=sp, length_scale=float(scale[b]), **PARAMS)
            y_lengths[b] = int(y_mask[0, 0].sum())
            w_ceil[b, : lens[b]] = attn[0, 0].sum(0).numpy()
            o_rows[b] = o[0, 0, : y_lengths[b] * hop].numpy()
        o_out = np.zeros((c["B"], int(y_lengths.max()) * hop), np.float32)
        for b, a in o_rows.items():
            o_out[b, : len(a)] = a
        frames = [FO.group_frames(e[r0:r1], lens[r0:r1], scale[r0]) for r0, r1, _ in fit]
        report[name] = dict(fit=fit, scale=[float(v) for v in scale], y_lengths=y_lengths.tolist(), group_frames=frames,
                            reference_frames=[int(y_lengths[r0:r1].sum()) for r0, r1, _ in fit])
        assert report[name]["reference_frames"] == frames, report[name]
        np.savez_compressed(os.path.join(outdir, name + ".npz"), logw=logw, scale=scale,
                            fit=np.asarray(fit, np.int64).reshape(-1, 3), w_ceil=w_ceil, y_lengths=y_lengths, o=o_out,
                            meta=np.array(json.dumps(dict(c, unfitted_scale=UNFITTED_SCALE, **PARAMS))))
    with open(os.path.join(outdir, "REPORT_tts_fit.json"), "w") as f:
        json.dump(report, f, indent=1, sort_keys=True)
    print(json.dumps(report, indent=1, sort_keys=True))


if __name__ == "__main__":
    main()
