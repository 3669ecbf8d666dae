"""Generate tests/golden/tts_style_*.npz by running the REAL reference modules with per-token speaker vectors.

Run in the build container only (``python oracle/make_golden_tts_style.py``, OPENVOICE_REFERENCE set).  The reference's
``infer`` derives g from ``sid``; every module it calls takes g [B, gin, T], so sentence inputs are run through
``model.enc_p``, ``model.sdp(..., g=g_tok, reverse=True)``, ``model.dp(..., g=g_tok)``, ``commons.generate_path``,
then ``model.flow(..., g=g_frames, reverse=True)`` and ``model.dec(..., g=g_frames)``, with g_frames = g_tok expanded
along the path by the same matmul that expands m_p (models.py:482-483).  Cases: B = 1 with a style ramp and a hard
switch; a padded B = 2 mixing a track row with a plain sid row; a per-row blend ([1, gin, 1], not expanded).  The
two RNG draws are injected as in make_golden_tts.py.  Writes new fixtures only.
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
import tts_style_oracle as S  # noqa: E402
from make_golden import import_reference, maxdiff  # noqa: E402
from make_golden_tts import injected_rng  # noqa: E402


def track(keys, n):
    """ToneTrack.dense arithmetic (openvoice_b200.api) over token positions 0..n-1: [gin, n]."""
    kf = np.asarray([f for f, _ in keys], dtype=np.int64)
    kse = torch.stack([e for _, e in keys]).numpy()
    t = np.arange(n, dtype=np.int64)
    hi = np.searchsorted(kf, t, side="right")
    lo, nx = np.clip(hi - 1, 0, len(kf) - 1), np.clip(hi, 0, len(kf) - 1)
    inner = (hi > 0) & (hi < len(kf))
    span = np.where(inner, kf[nx] - kf[lo], 1).astype(np.float32)
    u = np.where(inner, (t - kf[lo]).astype(np.float32) / span, np.float32(0)).astype(np.float32)
    a, b = kse[lo], kse[nx]
    return torch.from_numpy(np.ascontiguousarray(np.where(inner[:, None], a + u[:, None] * (b - a), a).astype(np.float32).T))


def cases(emb):
    e = lambda i: emb[i]  # noqa: E731
    g1 = track([(4, e(1)), (30, e(2)), (41, e(2)), (41, e(0))], 60)[None]
    g2 = torch.zeros(2, emb.shape[1], 50)
    g2[0] = track([(0, e(0)), (18, e(3)), (35, e(3)), (35, e(1))], 50)
    g2[1, :, :31] = e(2)[:, None]
    g3 = (0.7 * e(1) + 0.3 * e(3))[None, :, None]
    return [("tts_style_b1_t60", dict(B=1, T=60, seed=11, lengths=None), g1),
            ("tts_style_b2_padded", dict(B=2, T=50, seed=12, lengths=[50, 31]), g2),
            ("tts_style_b1_blend", dict(B=1, T=45, seed=13, lengths=None), g3)]


KW = dict(noise_scale=0.667, length_scale=1.0, noise_scale_w=0.6, sdp_ratio=0.2)


def inputs(c):
    tokens, lengths, _, noise_w = T.synthetic_tts_inputs(c["B"], c["T"], c["seed"], c["lengths"])
    noise = torch.randn(c["B"], 192, 40 * c["T"] + 64, generator=torch.Generator().manual_seed(30_000 + c["seed"]))
    return tokens, lengths, noise_w, noise


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    api, mel, models = import_reference()
    from openvoice import commons
    hp = V.DEFAULT_HPARAMS
    tts = T.TTS_HPARAMS
    sd = T.synthetic_tts_state_dict()
    model = models.SynthesizerTrn(tts["n_vocab"], hp["data"]["filter_length"] // 2 + 1,
                                  n_speakers=tts["n_speakers"], **hp["model"]).eval()
    model.load_state_dict(sd, strict=False)
    outdir = os.path.join(ROOT, "tests", "golden")
    report = {}
    for name, c, g in cases(sd["emb_g.weight"].float()):
        tokens, lengths, noise_w, noise = inputs(c)
        with torch.no_grad(), injected_rng(noise_w, noise):
            x, m_p, logs_p, x_mask = model.enc_p(tokens, lengths)
            logw_s = model.sdp(x, x_mask, g=g, reverse=True, noise_scale=KW["noise_scale_w"])
            logw_d = model.dp(x, x_mask, g=g)
            logw = logw_s * KW["sdp_ratio"] + logw_d * (1 - KW["sdp_ratio"])
            w_ceil = torch.ceil(torch.exp(logw) * x_mask * KW["length_scale"])
            y_lengths = torch.clamp_min(torch.sum(w_ceil, [1, 2]), 1).long()
            y_mask = torch.unsqueeze(commons.sequence_mask(y_lengths, None), 1).to(x_mask.dtype)
            attn = commons.generate_path(w_ceil, torch.unsqueeze(x_mask, 2) * torch.unsqueeze(y_mask, -1))
            expand = lambda t: torch.matmul(attn.squeeze(1), t.transpose(1, 2)).transpose(1, 2)  # noqa: E731
            m_y, logs_y = expand(m_p), expand(logs_p)
            g_frames = g if g.shape[-1] == 1 else expand(g)
            z_p = m_y + torch.randn_like(m_y) * torch.exp(logs_y) * KW["noise_scale"]
            z = model.flow(z_p, y_mask, g=g_frames, reverse=True)
            o = model.dec(z * y_mask, g=g_frames)
            r = S.tts_infer_g(sd, tokens, lengths, g, noise_w, noise, **KW)
        w = w_ceil[:, 0]
        report[name] = dict(logw_sdp=maxdiff(logw_s, r["logw_sdp"]), logw_dp=maxdiff(logw_d, r["logw_dp"]),
                            w_ceil=maxdiff(w, r["w_ceil"]), z_p=maxdiff(z_p, r["z_p"]), z=maxdiff(z, r["z"]),
                            o=maxdiff(o, r["o"]), frames=[int(v) for v in y_lengths])
        np.savez_compressed(os.path.join(outdir, name + ".npz"), g=g.numpy(), logw_sdp=logw_s.numpy(),
                            logw_dp=logw_d.numpy(), w_ceil=w.numpy(), y_lengths=y_lengths.numpy(), z_p=z_p.numpy(),
                            z=z.numpy(), o=o.numpy(), meta=np.array(json.dumps(dict(c, **KW))))
    with open(os.path.join(outdir, "REPORT_tts_style.json"), "w") as f:
        json.dump(report, f, indent=1, sort_keys=True)
    print(json.dumps(report, indent=1, sort_keys=True))


if __name__ == "__main__":
    main()
